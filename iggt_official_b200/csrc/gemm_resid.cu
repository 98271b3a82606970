// C-ABI launchers: residual (TMA reduce-add) and fused qkv + q/k-LayerNorm + RoPE epilogues.
#include <stdlib.h>
#include "gemm_launch.cuh"
#include "../../include/iggt_b200.h"

using namespace iggt;

namespace {
// the residual and qkv epilogues always run 128-wide tiles (plan_gemm)
template <int EPI, bool BF16>
int dispatch_bn(int /*bn*/, const CUtensorMap& tA, const CUtensorMap& tB, const CUtensorMap& tC, const GemmParams& p,
                cudaStream_t s) {
  return launch_gemm_kernel<128, EPI, BF16, false>(tA, tB, tC, p, s);
}
}  // namespace

extern "C" int iggt_gemm_resid32(const void* A, int64_t lda, const void* W, int64_t ldw, float* x,
                                 int64_t ldx, int M, int N, int K, int dtype, const float* bias,
                                 const float* gamma, int round_out16, iggt_stream_t stream) {
  if (M <= 0 || N <= 0 || K <= 0) return -1;
  if ((lda % 8) || (ldw % 8) || (K % 8) || (ldx % 4) || (N % 4)) return -2;
  if (dtype != 0 && dtype != 1) return -3;
  GemmParams p{};
  p.M = M; p.N = N; p.K = K; p.bias = bias; p.gamma = gamma; p.round_out16 = round_out16;
  const GemmPlan plan = plan_gemm(EPI_RESID32, M, N, K);
  const int bn = plan.bn;
  p.stream_k = plan.stream_k;
  p.num_m_tiles = plan.m_tiles; p.num_n_tiles = plan.n_tiles; p.num_k_blocks = plan.k_blocks;
  const TmDtype dt = dtype ? TM_BF16 : TM_F16;
  CUtensorMap tA, tB, tC;
  if (make_tmap_2d(&tA, dt, A, M, K, lda, GEMM_BK, GEMM_BM)) return -4;
  if (make_tmap_2d(&tB, dt, W, N, K, ldw, GEMM_BK, bn)) return -4;
  if (make_tmap_2d(&tC, TM_F32, x, M, N, ldx, 32, GEMM_BM)) return -4;
  return dtype ? dispatch_bn<EPI_RESID32, true>(bn, tA, tB, tC, p, (cudaStream_t)stream)
               : dispatch_bn<EPI_RESID32, false>(bn, tA, tB, tC, p, (cudaStream_t)stream);
}

extern "C" int iggt_gemm_qkv(const void* A, int64_t lda, const void* W, int64_t ldw, void* qkv,
                             int64_t ldo, int M, int C, int K, int dtype, const float* bias,
                             int qk_norm, const float* qn_w, const float* qn_b, const float* kn_w,
                             const float* kn_b, const float* rope_cos, const float* rope_sin,
                             const int* pos_yx, int T, const void* gather_maps, int n_gather, int gather_rows,
                             iggt_stream_t stream) {
  if (M <= 0 || C <= 0 || K <= 0 || (C % 64)) return -1;
  if ((lda % 8) || (ldw % 8) || (K % 8) || (ldo % 8)) return -2;
  if (dtype != 0 && dtype != 1) return -3;
  if (qk_norm && (!qn_w || !qn_b || !kn_w || !kn_b || !rope_cos || !rope_sin || !pos_yx || T <= 0))
    return -5;
  const int N = 3 * C;
  GemmParams p{};
  p.M = M; p.N = N; p.K = K; p.bias = bias;
  p.qk_norm = qk_norm; p.C = C;
  p.qn_w = qn_w; p.qn_b = qn_b; p.kn_w = kn_w; p.kn_b = kn_b;
  p.rope_cos = rope_cos; p.rope_sin = rope_sin; p.pos_yx = pos_yx; p.T = T > 0 ? T : 1;
  if (n_gather < 0 || n_gather > 16 || (n_gather > 0 && (!gather_maps || gather_rows <= 0 || M % gather_rows))) return -1;
  p.gather_maps = static_cast<const CUtensorMap*>(gather_maps); p.n_gather = n_gather; p.gather_col0 = C;
  p.gather_rows = gather_rows > 0 ? gather_rows : M;
  const GemmPlan plan = plan_gemm(EPI_QKV, M, N, K);
  const int bn = plan.bn;
  p.num_m_tiles = plan.m_tiles; p.num_n_tiles = plan.n_tiles; p.num_k_blocks = plan.k_blocks;
  const TmDtype dt = dtype ? TM_BF16 : TM_F16;
  CUtensorMap tA, tB, tC;
  if (make_tmap_2d(&tA, dt, A, M, K, lda, GEMM_BK, GEMM_BM)) return -4;
  if (make_tmap_2d(&tB, dt, W, N, K, ldw, GEMM_BK, bn)) return -4;
  if (make_tmap_2d(&tC, dt, qkv, M, N, ldo, 64, GEMM_BM)) return -4;
  if (n_gather > 0)
    return dtype ? dispatch_bn<EPI_QKV_GATHER, true>(bn, tA, tB, tC, p, (cudaStream_t)stream)
                 : dispatch_bn<EPI_QKV_GATHER, false>(bn, tA, tB, tC, p, (cudaStream_t)stream);
  return dtype ? dispatch_bn<EPI_QKV, true>(bn, tA, tB, tC, p, (cudaStream_t)stream)
               : dispatch_bn<EPI_QKV, false>(bn, tA, tB, tC, p, (cudaStream_t)stream);
}

// Tensor maps for the fused K|V gather: dst[i] = address of THIS rank's first row inside rank i's gathered K|V buffer
// ([scenes][world * rows][cols] 16-bit, row pitch ld elements; peer-mapped pointers); the map is 3-D {cols, rows, scenes}
// with scene pitch `scene_ld` elements.  Writes n maps (128 bytes each) to `dev_maps` (device memory, 64-byte aligned)
// followed by the n raw pointers and (ld, scene_ld) as int64 (for the rows the epilogue stores directly, gemm.cuh), with a
// synchronous copy - call once at setup, not inside a graph capture.  dev_maps: n * 136 + 16 bytes.
extern "C" int iggt_kv_gather_maps(void* const* dst, int n, int64_t rows, int64_t cols, int64_t ld, int64_t scenes,
                                   int64_t scene_ld, int dtype, void* dev_maps) {
  if (!dst || !dev_maps || n <= 0 || n > 16 || rows <= 0 || cols <= 0 || scenes <= 0 || (ld % 8) || (scene_ld % 8) ||
      (dtype != 0 && dtype != 1))
    return -1;
  CUtensorMap maps[16];
  for (int i = 0; i < n; ++i) {
    uint64_t dims[3] = {(uint64_t)cols, (uint64_t)rows, (uint64_t)scenes};
    uint64_t str[2] = {(uint64_t)ld * 2, (uint64_t)scene_ld * 2};
    uint32_t box[3] = {64, (uint32_t)GEMM_BM, 1};
    if (make_tmap(&maps[i], dtype ? TM_BF16 : TM_F16, 3, dst[i], dims, str, box)) return -4;
  }
  cudaError_t e = cudaMemcpy(dev_maps, maps, sizeof(CUtensorMap) * n, cudaMemcpyHostToDevice);
  if (e != cudaSuccess) return (int)e;
  int64_t tail[18];
  for (int i = 0; i < n; ++i) tail[i] = reinterpret_cast<int64_t>(dst[i]);
  tail[n] = ld; tail[n + 1] = scene_ld;
  return (int)cudaMemcpy(static_cast<uint8_t*>(dev_maps) + sizeof(CUtensorMap) * n, tail, sizeof(int64_t) * (n + 2),
                         cudaMemcpyHostToDevice);
}
