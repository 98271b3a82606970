// The dense heads' last stage in ONE kernel: 3x3 conv (128 -> 32, pad 1) + bias + ReLU + 1x1 conv (32 -> OC, fp32)
// + head activation, at full image resolution.  Replaces `output_conv2` and `activate_head`
// (iggt/heads/dpt_head.py:120-126,264-265, iggt/heads/head_act.py:61-125) and the part head's tail
// (iggt/heads/part_head.py:240-243).
//
// Why a dedicated kernel: the generic implicit-GEMM convolution (gemm.cuh) loads one TMA box per tap, i.e. re-reads
// this 550 MB input (8 x 518 x 518 x 128, 16-bit) nine times through L2 for 0.16 TFLOP of work, then writes a 32-channel 16-bit map that a second kernel reads back.  Here:
//   * tall boxes: an output tile is 8 (x) x 16 (y) pixels = 128 GEMM rows.  For each x-shift dx in {-1,0,1} and each
//     64-channel block ONE box {64 ch, 8 px, 18 rows} is loaded (TMA zero-fills the halo).  A box row (8 px x 128 B)
//     is exactly one 128B-swizzle atom, so the A operand of tap (dy, dx) is the same box at a (dy+1)*1024-byte
//     offset - an ordinary atom-aligned wgmma descriptor.  6 boxes (108 KB) per tile instead of 18 taps (288 KB);
//   * the 9 x 2 weight tiles (32 couts x 64 ch, 72 KB) stay resident in shared memory for the whole persistent CTA;
//   * two consumer warpgroups issue the wgmma of 64 pixels each; the 32 fp32 accumulators of a pixel go through a small
//     shared-memory tile to the thread that owns the pixel: + bias, ReLU, the 32 -> OC 1x1 product in fp32 and
//     exp / sign*expm1 / 1+exp are applied there and the fp32 outputs written directly (no 16-bit rounding of the
//     32-channel map, no second pass).
// Bound: HBM (input read once, 2 B x 128 per pixel in, <= 32 B per pixel out); algorithmic bytes per pixel 256 + 4*OC.
#include <stdlib.h>
#include "ptx.cuh"
#include "tmap.cuh"
#include "launch.cuh"
#include "../../include/iggt_b200.h"

namespace iggt {

constexpr int TC_TW = 8, TC_TH = 16;                 // output tile (pixels)
constexpr int TC_CIN = 128, TC_N = 32;               // input channels, conv output channels
constexpr int TC_BOX_ROWS = TC_TH + 2;               // 18 y-rows per box
constexpr int TC_A_BYTES = TC_BOX_ROWS * TC_TW * 128;     // 18 KB
constexpr int TC_B_BYTES = TC_N * 128;               // 4 KB per (tap, channel block)
constexpr int TC_STAGES = 7;
constexpr int TC_MAXOC = 8;
constexpr int TC_VEC_BYTES = (TC_N + TC_MAXOC * TC_N + TC_MAXOC) * 4;     // bias32 | w2[OC][32] | b2[OC]
constexpr int TC_ACC_LD = TC_N + 8;                  // fp32 accumulator tile row pitch (conflict-free fragment stores)
constexpr int TC_ACC_BYTES = 128 * TC_ACC_LD * 4;
constexpr int TC_THREADS = 384;                       // producer warpgroup + 2 consumer warpgroups
constexpr int TC_SMEM = 18 * TC_B_BYTES + TC_STAGES * TC_A_BYTES + TC_ACC_BYTES + 256 + ((TC_VEC_BYTES + 127) / 128) * 128;
static_assert(TC_SMEM <= 232448, "shared memory budget");
static_assert(TC_A_BYTES % 1024 == 0 && TC_B_BYTES % 1024 == 0, "128B-swizzle atoms need 1024-byte aligned tiles");

struct TailConvParams {
  int NB, H, W;
  int tiles_x, tiles_y, total_tiles;
  const float* bias;     // [32] conv bias
  const float* w2;       // [OC][32] fp32 1x1 weights (nullptr: store the 32-channel ReLU map as 16-bit NHWC)
  const float* b2;       // [OC]
  int OC;                // 2, 4 or 8
  int mode;              // 0 depth (exp | 1+exp), 1 points (sign*expm1|.| | 1+exp), 2 raw channels-first
  float* out_main;       // mode 0/1: [NB,H,W,OC-1]; mode 2: [NB,OC,H,W]
  float* out_conf;       // mode 0/1: [NB,H,W]
  void* out16;           // w2 == nullptr: NHWC [NB,H,W,32] 16-bit
};

template <bool BF16>
__global__ void __launch_bounds__(TC_THREADS, 1)
tailconv_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const TailConvParams p) {
  extern __shared__ __align__(1024) uint8_t smem[];
  if ((smem_u32(smem) & 1023u) != 0) __trap();
  uint8_t* smem_b = smem;                                  // [tap 0..8][cb 0..1] weight tiles
  uint8_t* smem_a = smem + 18 * TC_B_BYTES;                // ring of tall boxes
  float* acc_tile = reinterpret_cast<float*>(smem_a + TC_STAGES * TC_A_BYTES);   // [128 pixels][TC_ACC_LD]
  uint64_t* bars = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(acc_tile) + TC_ACC_BYTES);
  uint64_t* a_full = bars;
  uint64_t* a_empty = bars + TC_STAGES;
  uint64_t* b_full = bars + 2 * TC_STAGES;
  float* vec = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(bars) + 256);
  float* s_bias = vec;                                     // [32]
  float* s_w2 = vec + TC_N;                                // [OC][32]
  float* s_b2 = s_w2 + TC_MAXOC * TC_N;                    // [OC]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (warp == 0 && lane == 0) { tma_prefetch_desc(&tmA); tma_prefetch_desc(&tmB); }
  if (warp == 1 && lane == 0) {
    for (int i = 0; i < TC_STAGES; ++i) { mbar_init(&a_full[i], 1); mbar_init(&a_empty[i], 2); }   // 2 consumers
    mbar_init(b_full, 1);
    fence_barrier_init();
  }
  __syncthreads();
  griddep_wait();
  griddep_launch();

  auto decode = [&](int tile, int& img, int& y0, int& x0) {
    const int per_img = p.tiles_x * p.tiles_y;
    img = tile / per_img;
    const int r = tile % per_img;
    y0 = (r / p.tiles_x) * TC_TH;
    x0 = (r % p.tiles_x) * TC_TW;
  };

  if (warp < 4) {
    if (warp == 0 && lane == 0) {
      // weights once: 18 boxes of {64 ch, 32 couts} on one barrier
      mbar_expect_tx(b_full, 18 * TC_B_BYTES);
      for (int tap = 0; tap < 9; ++tap)
        for (int cb = 0; cb < 2; ++cb)
          tma_load_2d(smem_b + (tap * 2 + cb) * TC_B_BYTES, &tmB, b_full, tap * TC_CIN + cb * 64, 0);
      int st = 0; uint32_t ph = 0;
      for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
        int img, y0, x0;
        decode(tile, img, y0, x0);
        for (int dx = -1; dx <= 1; ++dx)
          for (int cb = 0; cb < 2; ++cb) {
            mbar_wait(&a_empty[st], ph ^ 1);
            mbar_expect_tx(&a_full[st], TC_A_BYTES);
            tma_load_4d(smem_a + st * TC_A_BYTES, &tmA, &a_full[st], cb * 64, x0 + dx, y0 - 1, img);
            if (++st == TC_STAGES) { st = 0; ph ^= 1; }
          }
      }
    }
  } else {
    // ---------------------------------------------------------------- consumers: warpgroup cw = GEMM rows [64 cw, +64)
    const int cw = (warp - 4) >> 2;
    const int gtid = threadIdx.x & 127;
    const int ew = (warp - 4) & 3;
    for (int i = threadIdx.x - 128; i < TC_N; i += 256) s_bias[i] = p.bias ? p.bias[i] : 0.f;
    if (p.w2) {
      for (int i = threadIdx.x - 128; i < p.OC * TC_N; i += 256) s_w2[i] = p.w2[i];
      for (int i = threadIdx.x - 128; i < p.OC; i += 256) s_b2[i] = p.b2[i];
    }
    named_bar_sync(1, 256);
    const int row = cw * 64 + gtid;                        // epilogue (gtid < 64): GEMM row = pixel (yl, xl) of the tile
    const int xl = row % TC_TW, yl = row / TC_TW;
    const int64_t hw = static_cast<int64_t>(p.H) * p.W;
    const uint32_t bar_id = 2 + cw;
    mbar_wait(b_full, 0);
    int st = 0; uint32_t ph = 0;
    for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
      int img, y0, x0;
      decode(tile, img, y0, x0);
      float acc[TC_N / 2];
#pragma unroll
      for (int i = 0; i < TC_N / 2; ++i) acc[i] = 0.f;
      bool first = true;
      int prev = -1;
      for (int dx = -1; dx <= 1; ++dx)
        for (int cb = 0; cb < 2; ++cb) {
          mbar_wait(&a_full[st], ph);
          const uint32_t a_base = smem_u32(smem_a + st * TC_A_BYTES) + cw * (8 * TC_TW * 128);   // 8 box rows down
          wgmma_fence();
#pragma unroll
          for (int dy = -1; dy <= 1; ++dy) {
            const int tap = (dy + 1) * 3 + (dx + 1);
            const uint32_t a_addr = a_base + (dy + 1) * (TC_TW * 128);      // (dy + 1) box rows down: 1024 B each
            const uint32_t b_addr = smem_u32(smem_b + (tap * 2 + cb) * TC_B_BYTES);
#pragma unroll
            for (int k = 0; k < 4; ++k) {
              wgmma_m64n32k16_ss<BF16>(acc, make_desc_sw128(a_addr + k * 32, 1024), make_desc_sw128(b_addr + k * 32, 1024),
                                       first ? 0u : 1u);
              first = false;
            }
          }
          wgmma_commit();
          wgmma_wait<1>();                                 // the previous box's MMAs have retired: free its slot
          if (prev >= 0 && gtid == 0) mbar_arrive(&a_empty[prev]);
          prev = st;
          if (++st == TC_STAGES) { st = 0; ph ^= 1; }
        }
      wgmma_wait<0>();
      reg_fence(acc);
      if (gtid == 0) mbar_arrive(&a_empty[prev]);
      // accumulator fragments -> this warpgroup's 64 rows of the fp32 tile
      named_bar_sync(bar_id, 128);                         // the previous tile's rows have been read
      {
        float* const d0 = acc_tile + (cw * 64 + ew * 16 + (lane >> 2)) * TC_ACC_LD + 2 * (lane & 3);
#pragma unroll
        for (int j = 0; j < TC_N / 8; ++j) {
          *reinterpret_cast<float2*>(d0 + 8 * j) = make_float2(acc[4 * j], acc[4 * j + 1]);
          *reinterpret_cast<float2*>(d0 + 8 * TC_ACC_LD + 8 * j) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
        }
      }
      named_bar_sync(bar_id, 128);
      if (gtid >= 64) continue;
      float r[TC_N];
#pragma unroll
      for (int i = 0; i < TC_N; i += 4) {
        const float4 a = *reinterpret_cast<const float4*>(acc_tile + row * TC_ACC_LD + i);
        r[i] = a.x; r[i + 1] = a.y; r[i + 2] = a.z; r[i + 3] = a.w;
      }
      const int y = y0 + yl, x = x0 + xl;
      if (y < p.H && x < p.W) {
        float f[TC_N];
#pragma unroll
        for (int i = 0; i < TC_N; ++i) f[i] = relu_nan(r[i] + s_bias[i]);     // conv bias + ReLU
        const int64_t pix = (static_cast<int64_t>(img) * p.H + y) * p.W + x;
        if (!p.w2) {
          uint16_t* dst = reinterpret_cast<uint16_t*>(p.out16) + pix * TC_N;
#pragma unroll
          for (int c = 0; c < TC_N; c += 8) {
            uint4 u;
            u.x = pack16x2<BF16>(f[c], f[c + 1]); u.y = pack16x2<BF16>(f[c + 2], f[c + 3]);
            u.z = pack16x2<BF16>(f[c + 4], f[c + 5]); u.w = pack16x2<BF16>(f[c + 6], f[c + 7]);
            *reinterpret_cast<uint4*>(dst + c) = u;
          }
        } else {
          float o[TC_MAXOC];
#pragma unroll
          for (int c = 0; c < TC_MAXOC; ++c) {
            if (c < p.OC) {
              float s = s_b2[c];
#pragma unroll
              for (int k = 0; k < TC_N; ++k) s = fmaf(f[k], s_w2[c * TC_N + k], s);
              o[c] = s;
            }
          }
          if (p.mode == 2) {
            float* dst = p.out_main + static_cast<int64_t>(img) * p.OC * hw + static_cast<int64_t>(y) * p.W + x;
#pragma unroll
            for (int c = 0; c < TC_MAXOC; ++c)
              if (c < p.OC) dst[c * hw] = o[c];
          } else {
            float* dst = p.out_main + pix * (p.OC - 1);
#pragma unroll
            for (int c = 0; c < TC_MAXOC - 1; ++c)
              if (c < p.OC - 1) dst[c] = p.mode == 0 ? expf(o[c]) : copysignf(expm1f(fabsf(o[c])), o[c]);
            float last = o[0];
#pragma unroll
            for (int c = 1; c < TC_MAXOC; ++c)
              if (c == p.OC - 1) last = o[c];
            p.out_conf[pix] = 1.0f + expf(last);
          }
        }
      }
    }
  }
}

template <bool BF16>
int launch_tailconv(const CUtensorMap& tA, const CUtensorMap& tB, const TailConvParams& p, cudaStream_t stream) {
  auto kern = tailconv_kernel<BF16>;
  static DeviceOnce once;
  if (once.first()) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_SMEM);
    if (e != cudaSuccess) { once.reset_current(); return (int)e; }
  }
  const int sms = device_sm_count();
  const int grid = p.total_tiles < sms ? p.total_tiles : sms;
  return (int)launch_pdl(kern, dim3(grid), dim3(TC_THREADS), TC_SMEM, stream, tA, tB, p);
}

}  // namespace iggt

using namespace iggt;

extern "C" int iggt_dpt_tail_fused(const void* x, const void* Wp, const float* bias, const float* w2, const float* b2,
                                   float* out_main, float* out_conf, void* out16, int NB, int H, int W, int OC, int mode,
                                   int dtype, iggt_stream_t stream) {
  if (!x || !Wp || NB <= 0 || H <= 0 || W <= 0) return -1;
  if (dtype != 0 && dtype != 1) return -3;
  if (w2) {
    if (!b2 || !out_main || (OC != 2 && OC != 4 && OC != 8) || mode < 0 || mode > 2) return -1;
    if (mode != 2 && !out_conf) return -1;
  } else if (!out16) {
    return -1;
  }
  const TmDtype dt = dtype ? TM_BF16 : TM_F16;
  CUtensorMap tA, tB;
  {
    uint64_t dims[4] = {(uint64_t)TC_CIN, (uint64_t)W, (uint64_t)H, (uint64_t)NB};
    uint64_t str[3] = {(uint64_t)TC_CIN * 2, (uint64_t)W * TC_CIN * 2, (uint64_t)H * W * TC_CIN * 2};
    uint32_t box[4] = {64, TC_TW, TC_BOX_ROWS, 1};
    if (make_tmap(&tA, dt, 4, x, dims, str, box)) return -4;
  }
  if (make_tmap_2d(&tB, dt, Wp, (uint64_t)TC_N, (uint64_t)9 * TC_CIN, (uint64_t)9 * TC_CIN, 64, TC_N)) return -4;
  TailConvParams p;
  p.NB = NB; p.H = H; p.W = W;
  p.tiles_x = (W + TC_TW - 1) / TC_TW;
  p.tiles_y = (H + TC_TH - 1) / TC_TH;
  p.total_tiles = NB * p.tiles_x * p.tiles_y;
  p.bias = bias; p.w2 = w2; p.b2 = b2; p.OC = OC; p.mode = mode;
  p.out_main = out_main; p.out_conf = out_conf; p.out16 = out16;
  return dtype ? launch_tailconv<true>(tA, tB, p, (cudaStream_t)stream) : launch_tailconv<false>(tA, tB, p, (cudaStream_t)stream);
}
