// C-ABI launchers: 16-bit and 32-bit store epilogues (see include/iggt_b200.h).
#include "gemm_launch.cuh"
#include "../../include/iggt_b200.h"

using namespace iggt;

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
  return dispatch_dtype(dtype, [&](auto bf16) {
    if ((ldo % 8) || (addend && (add_ld % 8))) return -2;
    GemmParams p{};
    p.bias = bias; p.act = act;
    p.addend = addend; p.add_rows = add_rows > 0 ? add_rows : 1; p.add_ld = (int)add_ld;
    CUtensorMap tA, tB, tC;
    int bn;
    if (const int st = gemm_operands(EPI_STORE16, tm16(bf16), A, lda, W, ldw, M, N, K, p, tA, tB, bn)) return st;
    if (make_tmap_2d(&tC, tm16(bf16), out, M, N, ldo, 64, GEMM_BM)) return -4;
    return launch_gemm<EPI_STORE16, bf16>(bn, tA, tB, tC, p, (cudaStream_t)stream);
  });
}

extern "C" int iggt_gemm_store32(const void* A, int64_t lda, const void* W, int64_t ldw, float* out,
                                 int64_t ldo, int M, int N, int K, int dtype, const float* bias,
                                 int act, iggt_stream_t stream) {
  return dispatch_dtype(dtype, [&](auto bf16) {
    if (ldo % 4) return -2;
    GemmParams p{};
    p.bias = bias; p.act = act;
    CUtensorMap tA, tB, tC;
    int bn;
    if (const int st = gemm_operands(EPI_STORE32, tm16(bf16), A, lda, W, ldw, M, N, K, p, tA, tB, bn)) return st;
    if (make_tmap_2d(&tC, TM_F32, out, M, N, ldo, 32, GEMM_BM)) return -4;
    return launch_gemm<EPI_STORE32, bf16>(bn, tA, tB, tC, p, (cudaStream_t)stream);
  });
}
