// C-ABI launcher: NHWC implicit-GEMM convolution (3x3 pad 1 / 1x1) on the wgmma GEMM main loop.
// The A operand of tap (ky,kx) is the 4-D TMA box {64 ch, 16 px, 8 rows, 1 image} shifted by
// (kx-1, ky-1); TMA zero-fills the halo, so no im2col buffer is ever materialised.
#include "gemm_launch.cuh"
#include "../../include/iggt_b200.h"

using namespace iggt;

extern "C" int iggt_conv_nhwc(const void* x, const void* Wp, void* out, int NB, int H, int W,
                              int Cin, int Cout, int taps, int dtype, const float* bias, int act,
                              const void* resid, const void* resid2, int act_post,
                              iggt_stream_t stream) {
  return dispatch_dtype(dtype, [&](auto bf16) {
    if (NB <= 0 || H <= 0 || W <= 0 || Cin <= 0 || Cout <= 0) return -1;
    if ((Cin % 64) || (Cout % 8)) return -2;
    if (taps != 1 && taps != 9) return -1;
    GemmParams p{};
    p.bias = bias; p.act = act; p.resid = resid; p.resid2 = resid2; p.act_post = act_post;
    p.conv_taps = taps; p.conv_C = Cin; p.H = H; p.W = W; p.NB = NB;
    p.tiles_x = (W + CONV_TW - 1) / CONV_TW;
    p.tiles_y = (H + CONV_TH - 1) / CONV_TH;
    p.M = NB * H * W; p.N = Cout; p.K = taps * Cin;
    p.num_m_tiles = NB * p.tiles_x * p.tiles_y;
    const int bn = choose_bn(Cout);
    p.num_n_tiles = (Cout + bn - 1) / bn;
    p.num_k_blocks = taps * (Cin / GEMM_BK);
    p.add_rows = 1;
    CUtensorMap tA, tB, tC;
    {
      uint64_t dims[4] = {(uint64_t)Cin, (uint64_t)W, (uint64_t)H, (uint64_t)NB};
      uint64_t str[3] = {(uint64_t)Cin * 2, (uint64_t)W * Cin * 2, (uint64_t)H * W * Cin * 2};
      uint32_t box[4] = {64, CONV_TW, CONV_TH, 1};
      if (make_tmap(&tA, tm16(bf16), 4, x, dims, str, box)) return -4;
    }
    if (make_tmap_2d(&tB, tm16(bf16), Wp, Cout, (uint64_t)taps * Cin, (uint64_t)taps * Cin, GEMM_BK, bn)) return -4;
    {
      uint64_t dims[4] = {(uint64_t)Cout, (uint64_t)W, (uint64_t)H, (uint64_t)NB};
      uint64_t str[3] = {(uint64_t)Cout * 2, (uint64_t)W * Cout * 2, (uint64_t)H * W * Cout * 2};
      uint32_t box[4] = {64, CONV_TW, CONV_TH, 1};
      if (make_tmap(&tC, tm16(bf16), 4, out, dims, str, box)) return -4;
    }
    return launch_gemm<EPI_STORE16, bf16, true>(bn, tA, tB, tC, p, (cudaStream_t)stream);
  });
}
