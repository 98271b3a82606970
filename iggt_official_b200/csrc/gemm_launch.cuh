// Host-side launch helpers shared by the GEMM / conv translation units.
#pragma once
#include "gemm.cuh"
#include "tmap.cuh"

namespace iggt {

// Pick the N tile: 128 wherever N allows it (a 128 x 128 tile reads 2 x 16 KB of operands per 64-deep k-block for
// 2 x 64 x 128 x 64 MACs; the 64-wide tile needs the same A bytes for half the work).  Wider tiles do not fit: each
// ping-pong consumer warpgroup holds the whole 128 x BN fp32 accumulator, BN registers per thread out of the 232 it
// gets from setmaxnreg, and the epilogue needs its 64-value row chunk next to it; 128 x 256 would need 256.
inline int choose_bn(int N) { return N <= 64 ? 64 : 128; }

// The host-side schedule of one GEMM launch, shared by the launchers and by iggt_gemm_plan (unit-tested without a GPU).
struct GemmPlan {
  int bn;          // N tile
  int pair;        // CTA pairs (a 256-row tile shared by two CTAs): not used on sm_90, always 0
  int stream_k;    // residual epilogue only
  int m_tiles, n_tiles, k_blocks;
  int grid;        // CTAs launched
};

inline GemmPlan plan_gemm(int epi, int M, int N, int K) {
  static const int sk_env = [] { const char* e = getenv("IGGT_STREAMK"); return e ? atoi(e) : 1; }();
  GemmPlan g{};
  const int m_sub = (M + GEMM_BM - 1) / GEMM_BM;
  g.k_blocks = (K + GEMM_BK - 1) / GEMM_BK;
  g.m_tiles = m_sub;
  const int sms = device_sm_count();
  g.bn = choose_bn(N);
  if ((epi == EPI_RESID32 || epi == EPI_QKV) && g.bn < 128) g.bn = 128;
  if (epi == EPI_RESID32) {
    // Stream-K: cutting the (tile, k-block) space into equal ranges removes the wave-quantisation loss (N = 1024 gives
    // 5.2 waves of 128 x 128 tiles at M = 10992 on 132 SMs).  IGGT_STREAMK=0 restores whole-tile scheduling
    // (bit-reproducible accumulation order).
    const int tiles = m_sub * ((N + 127) / 128);
    const bool quantised = tiles % sms != 0 && tiles > sms / 2;
    g.stream_k = (sk_env && N >= 128 && quantised && (long)tiles * g.k_blocks >= 4L * sms) ? 1 : 0;
  }
  g.n_tiles = (N + g.bn - 1) / g.bn;
  const int tiles = g.m_tiles * g.n_tiles;
  g.grid = g.stream_k ? sms : (tiles < sms ? tiles : sms);
  return g;
}

template <int BN, int EPI, bool BF16, bool CONV>
inline int launch_gemm_kernel(const CUtensorMap& tA, const CUtensorMap& tB, const CUtensorMap& tC,
                              const GemmParams& p, cudaStream_t stream) {
  constexpr int smem = GemmSmem<BN>::TOTAL;
  static_assert(smem <= 232448, "shared memory budget");
  const cudaError_t e = opt_in_smem<gemm_wgmma_kernel<BN, EPI, BF16, CONV>>(smem);
  if (e != cudaSuccess) return (int)e;
  const int sms = device_sm_count();
  const int tiles = p.num_m_tiles * p.num_n_tiles;
  int workers = tiles < sms ? tiles : sms;
  if (p.stream_k) workers = sms;
  if (workers <= 0) return 0;
  return (int)launch_pdl(gemm_wgmma_kernel<BN, EPI, BF16, CONV>, dim3(workers), dim3(GEMM_THREADS), smem, stream, tA, tB,
                         tC, p);
}

// The launch of epilogue EPI with the plan's N tile.  Only the store epilogues (the conv stores 16-bit) are built with
// 64-wide tiles: plan_gemm gives the residual and qkv epilogues 128.
template <int EPI, bool BF16, bool CONV = false>
inline int launch_gemm(int bn, const CUtensorMap& tA, const CUtensorMap& tB, const CUtensorMap& tC, const GemmParams& p,
                       cudaStream_t stream) {
  if constexpr (EPI == EPI_STORE16 || EPI == EPI_STORE32) {
    if (bn == 64) return launch_gemm_kernel<64, EPI, BF16, CONV>(tA, tB, tC, p, stream);
  }
  return launch_gemm_kernel<128, EPI, BF16, CONV>(tA, tB, tC, p, stream);
}

// What the matrix (non-conv) GEMM launchers share: the A [M, K] / W [N, K] operand checks, the schedule (problem size
// and tile counts into p, the N tile into bn) and the A / W tensor maps.
inline int gemm_operands(int epi, TmDtype dt, const void* A, int64_t lda, const void* W, int64_t ldw, int M, int N,
                         int K, GemmParams& p, CUtensorMap& tA, CUtensorMap& tB, int& bn) {
  if (M <= 0 || N <= 0 || K <= 0) return -1;
  if ((lda % 8) || (ldw % 8) || (K % 8)) return -2;  // TMA needs 16-byte row pitch
  const GemmPlan plan = plan_gemm(epi, M, N, K);
  p.M = M; p.N = N; p.K = K;
  p.stream_k = plan.stream_k;
  p.num_m_tiles = plan.m_tiles; p.num_n_tiles = plan.n_tiles; p.num_k_blocks = plan.k_blocks;
  bn = plan.bn;
  if (make_tmap_2d(&tA, dt, A, M, K, lda, GEMM_BK, GEMM_BM)) return -4;
  if (make_tmap_2d(&tB, dt, W, N, K, ldw, GEMM_BK, bn)) return -4;
  return 0;
}

}  // namespace iggt
