// Host-side launch helpers shared by the GEMM / conv translation units.
#pragma once
#include "gemm.cuh"
#include "tmap.cuh"

namespace iggt {

// Pick the N tile: 128 wherever N allows it (a 128 x 128 tile reads 2 x 16 KB of operands per 64-deep k-block for
// 2 x 64 x 128 x 64 MACs; the 64-wide tile needs the same A bytes for half the work).  Wider tiles do not fit: each
// ping-pong consumer warpgroup holds the whole 128 x BN fp32 accumulator, BN registers per thread out of the 232 it
// gets from setmaxnreg, and the epilogue needs its 64-value row chunk next to it; 128 x 256 would need 256.
inline int choose_bn(int /*m_tiles*/, int N) { return N <= 64 ? 64 : 128; }

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
  g.bn = choose_bn(m_sub, N);
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
  auto kern = gemm_wgmma_kernel<BN, EPI, BF16, CONV>;
  static DeviceOnce once;
  constexpr int smem = GemmSmem<BN>::TOTAL;
  static_assert(smem <= 232448, "shared memory budget");
  if (once.first()) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) { once.reset_current(); return (int)e; }
  }
  const int sms = device_sm_count();
  const int tiles = p.num_m_tiles * p.num_n_tiles;
  int workers = tiles < sms ? tiles : sms;
  if (p.stream_k) workers = sms;
  if (workers <= 0) return 0;
  return (int)launch_pdl(kern, dim3(workers), dim3(GEMM_THREADS), smem, stream, tA, tB, tC, p);
}

}  // namespace iggt
