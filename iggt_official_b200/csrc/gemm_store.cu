// C-ABI launchers: 16-bit and 32-bit store epilogues (see include/iggt_b200.h).
#include "gemm_launch.cuh"
#include "../../include/iggt_b200.h"

using namespace iggt;

namespace {

template <int EPI, bool BF16>
int dispatch_bn(int bn, const CUtensorMap& tA, const CUtensorMap& tB, const CUtensorMap& tC, const GemmParams& p,
                cudaStream_t s) {
  if (bn == 64) return launch_gemm_kernel<64, EPI, BF16, false>(tA, tB, tC, p, s);
  return launch_gemm_kernel<128, EPI, BF16, false>(tA, tB, tC, p, s);
}

int gemm_common(int epi, const void* A, int64_t lda, const void* W, int64_t ldw, void* out,
                int64_t ldo, int M, int N, int K, int dtype, GemmParams p, cudaStream_t stream) {
  if (M <= 0 || N <= 0 || K <= 0) return -1;
  if ((lda % 8) || (ldw % 8) || (K % 8)) return -2;  // TMA needs 16-byte row pitch
  if (dtype != 0 && dtype != 1) return -3;
  const bool out32 = (epi == EPI_STORE32);
  if (out32 ? (ldo % 4) : (ldo % 8)) return -2;
  p.M = M; p.N = N; p.K = K;
  const GemmPlan plan = plan_gemm(epi, M, N, K);
  const int bn = plan.bn;
  p.num_m_tiles = plan.m_tiles; p.num_n_tiles = plan.n_tiles; p.num_k_blocks = plan.k_blocks;
  const TmDtype dt = dtype ? TM_BF16 : TM_F16;
  CUtensorMap tA, tB, tC;
  if (make_tmap_2d(&tA, dt, A, M, K, lda, GEMM_BK, GEMM_BM)) return -4;
  if (make_tmap_2d(&tB, dt, W, N, K, ldw, GEMM_BK, bn)) return -4;
  if (out32) {
    if (make_tmap_2d(&tC, TM_F32, out, M, N, ldo, 32, GEMM_BM)) return -4;
  } else {
    if (make_tmap_2d(&tC, dt, out, M, N, ldo, 64, GEMM_BM)) return -4;
  }
  if (epi == EPI_STORE16) {
    return dtype ? dispatch_bn<EPI_STORE16, true>(bn, tA, tB, tC, p, stream)
                 : dispatch_bn<EPI_STORE16, false>(bn, tA, tB, tC, p, stream);
  }
  return dtype ? dispatch_bn<EPI_STORE32, true>(bn, tA, tB, tC, p, stream)
               : dispatch_bn<EPI_STORE32, false>(bn, tA, tB, tC, p, stream);
}

}  // namespace

// Host-only: the schedule the launchers would use for an (epilogue, M, N, K) problem on this device (132 SMs assumed
// when no GPU is visible).  epi: 0 store16, 1 resid32, 2 qkv (N = 3C), 3 store32.
// out = {bn, pair, stream_k, m_tiles, n_tiles, k_blocks, grid}.
extern "C" int iggt_gemm_plan(int epi, int M, int N, int K, int* out) {
  if (epi < 0 || epi > 3 || M <= 0 || N <= 0 || K <= 0 || !out) return -1;
  const GemmPlan g = plan_gemm(epi, M, N, K);
  out[0] = g.bn; out[1] = g.pair; out[2] = g.stream_k; out[3] = g.m_tiles; out[4] = g.n_tiles; out[5] = g.k_blocks;
  out[6] = g.grid;
  return 0;
}

extern "C" int iggt_gemm_store16(const void* A, int64_t lda, const void* W, int64_t ldw, void* out,
                                 int64_t ldo, int M, int N, int K, int dtype, const float* bias,
                                 int act, const void* addend, int add_rows, int64_t add_ld,
                                 iggt_stream_t stream) {
  GemmParams p{};
  p.bias = bias; p.act = act;
  p.addend = addend; p.add_rows = add_rows > 0 ? add_rows : 1; p.add_ld = (int)add_ld;
  if (addend && (add_ld % 8)) return -2;
  return gemm_common(EPI_STORE16, A, lda, W, ldw, out, ldo, M, N, K, dtype, p, (cudaStream_t)stream);
}

extern "C" int iggt_gemm_store32(const void* A, int64_t lda, const void* W, int64_t ldw, float* out,
                                 int64_t ldo, int M, int N, int K, int dtype, const float* bias,
                                 int act, iggt_stream_t stream) {
  GemmParams p{};
  p.bias = bias; p.act = act;
  return gemm_common(EPI_STORE32, A, lda, W, ldw, out, ldo, M, N, K, dtype, p, (cudaStream_t)stream);
}
