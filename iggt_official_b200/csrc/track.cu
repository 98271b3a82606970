// Kernels of the track head (SURVEY.md 8f row 4; iggt/heads/track_modules/*): everything around the update
// transformer that is not a GEMM or an attention call.
//   avgpool2_nhwc        one level of the correlation pyramid (blocks.py:166-176)
//   sample_bilinear_nhwc feature rows at sub-pixel positions, border padding (utils.py:199-226)
//   corr_sample          the 7-level, 9x9 correlation lookup WITHOUT the correlation volume: bilinear sampling is linear,
//                        so <target, fmap> is evaluated on the 10x10 integer pixels under the window and interpolated
//                        afterwards (blocks.py:187-246 builds the whole [N, H*W] volume per level and samples it)
//   track_input          flow embedding + concatenation + positional / reference tokens + LayerNorm(388) in one pass
//                        (base_track_predictor.py:139-165 + blocks.py:103-104)
//   layernorm_rows       LayerNorm over any width <= 2048 of fp32 rows, fp32 and / or 16-bit result
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include "../../include/iggt_b200.h"

namespace iggt {

template <bool BF16>
__device__ __forceinline__ float ld16(const uint16_t* p) {
  if constexpr (BF16) return __uint_as_float(static_cast<uint32_t>(*p) << 16);
  else return __half2float(__ushort_as_half(*p));
}
template <bool BF16>
__device__ __forceinline__ uint16_t st16(float v) {
  if constexpr (BF16) return __bfloat16_as_ushort(__float2bfloat16_rn(v));
  else return __half_as_ushort(__float2half_rn(v));
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// [NB, H, W, C] -> [NB, H/2, W/2, C] (floor), fp32 mean of the 2x2 window, one thread per 2 channels
template <bool BF16>
__global__ void __launch_bounds__(256)
avgpool2_kernel(const uint16_t* __restrict__ x, uint16_t* __restrict__ y, int NB, int H, int W, int C) {
  const int Ho = H / 2, Wo = W / 2, C2 = C / 2;
  const int64_t total = static_cast<int64_t>(NB) * Ho * Wo * C2;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(i % C2) * 2;
    int64_t r = i / C2;
    const int xo = static_cast<int>(r % Wo); r /= Wo;
    const int yo = static_cast<int>(r % Ho);
    const int n = static_cast<int>(r / Ho);
    const uint16_t* p = x + ((static_cast<int64_t>(n) * H + 2 * yo) * W + 2 * xo) * C + c;
    const int64_t row = static_cast<int64_t>(W) * C;
    float a0 = 0.f, a1 = 0.f;
#pragma unroll
    for (int dy = 0; dy < 2; ++dy)
#pragma unroll
      for (int dx = 0; dx < 2; ++dx) {
        a0 += ld16<BF16>(p + dy * row + dx * C);
        a1 += ld16<BF16>(p + dy * row + dx * C + 1);
      }
    uint16_t* q = y + ((static_cast<int64_t>(n) * Ho + yo) * Wo + xo) * C + c;
    q[0] = st16<BF16>(a0 * 0.25f);
    q[1] = st16<BF16>(a1 * 0.25f);
  }
}

// out[n, r, :] = bilinear(x[n], coords[n, r]) with align_corners=True and BORDER padding (coordinates clamped to the
// image), C = 128: one warp per point, 4 channels per lane
template <bool BF16>
__global__ void __launch_bounds__(256)
sample_bilinear_kernel(const uint16_t* __restrict__ x, const float* __restrict__ coords, float* __restrict__ out, int NB,
                       int R, int H, int W, int C) {
  const int64_t pt = static_cast<int64_t>(blockIdx.x) * 8 + (threadIdx.x >> 5);
  if (pt >= static_cast<int64_t>(NB) * R) return;
  const int lane = threadIdx.x & 31;
  const int n = static_cast<int>(pt / R);
  const float cx = fminf(fmaxf(coords[pt * 2], 0.f), static_cast<float>(W - 1));
  const float cy = fminf(fmaxf(coords[pt * 2 + 1], 0.f), static_cast<float>(H - 1));
  const int x0 = static_cast<int>(floorf(cx)), y0 = static_cast<int>(floorf(cy));
  const int x1 = min(x0 + 1, W - 1), y1 = min(y0 + 1, H - 1);
  const float fx = cx - x0, fy = cy - y0;
  const uint16_t* base = x + static_cast<int64_t>(n) * H * W * C;
  for (int c = lane; c < C; c += 32) {
    const float v00 = ld16<BF16>(base + (static_cast<int64_t>(y0) * W + x0) * C + c);
    const float v01 = ld16<BF16>(base + (static_cast<int64_t>(y0) * W + x1) * C + c);
    const float v10 = ld16<BF16>(base + (static_cast<int64_t>(y1) * W + x0) * C + c);
    const float v11 = ld16<BF16>(base + (static_cast<int64_t>(y1) * W + x1) * C + c);
    out[pt * C + c] = (v00 * (1.f - fx) + v01 * fx) * (1.f - fy) + (v10 * (1.f - fx) + v11 * fx) * fy;
  }
}

constexpr int CORR_LEVELS = 7;
constexpr int CORR_R = 4;
constexpr int CORR_WIN = 2 * CORR_R + 1;      // 9
constexpr int CORR_PATCH = CORR_WIN + 1;      // 10 integer pixels per axis under a 9-wide unit-spaced window

struct CorrParams {
  const uint16_t* level[CORR_LEVELS];         // NHWC [B*S, H_l, W_l, 128]
  int H[CORR_LEVELS], W[CORR_LEVELS];
  const float* targets;                       // [rows, 128]   rows ordered (b, n, s)
  const float* coords;                        // [rows, 2]     level-0 pixels (x, y)
  void* out;                                  // [rows, ldo] 16-bit: 7 x 81 values, then zero padding up to ldo
  int rows, N, S, ldo;
};

// One warp per (row, level).  out[(i, j)] = corr(cx + i - 4, cy + j - 4): the reference adds its (dy, dx) grid to (x, y)
// as is (blocks.py:183-185, 224), so the FIRST window index moves along x.  Zero padding outside the level.
template <bool BF16>
__global__ void __launch_bounds__(256)
corr_sample_kernel(const CorrParams p) {
  __shared__ float patch[8][CORR_PATCH * CORR_PATCH];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t item = static_cast<int64_t>(blockIdx.x) * 8 + warp;
  const bool live = item < static_cast<int64_t>(p.rows) * CORR_LEVELS;
  const int lvl = live ? static_cast<int>(item % CORR_LEVELS) : 0;
  const int row = live ? static_cast<int>(item / CORR_LEVELS) : 0;
  // row = (b * N + n) * S + s  ->  image index b * S + s
  const int s = row % p.S, b = row / (p.S * p.N);
  const int H = p.H[lvl], W = p.W[lvl];
  const float inv = 1.0f / static_cast<float>(1 << lvl);
  // A level that has shrunk to ONE pixel along an axis is degenerate in the reference: its sampler normalises with
  // 2 / max(size - 1, 1) and grid_sample(align_corners=True) maps every coordinate of a size-1 axis to pixel 0
  // (utils.py:176-196), so all window positions read that pixel.  Reproduced by pinning the centre to 0 and freezing
  // the window index along that axis (only small inputs get here: 518 x 518 images end at a 4 x 4 level).
  const bool flat_x = p.W[lvl] == 1, flat_y = p.H[lvl] == 1;
  const float cx = flat_x ? 0.f : p.coords[static_cast<int64_t>(row) * 2] * inv;
  const float cy = flat_y ? 0.f : p.coords[static_cast<int64_t>(row) * 2 + 1] * inv;
  const float fx0 = floorf(cx), fy0 = floorf(cy);
  const int x0 = static_cast<int>(fx0) - CORR_R, y0 = static_cast<int>(fy0) - CORR_R;
  const float fx = cx - fx0, fy = cy - fy0;
  const float4 t = *reinterpret_cast<const float4*>(p.targets + static_cast<int64_t>(row) * 128 + lane * 4);
  const uint16_t* img = p.level[lvl] + static_cast<int64_t>(b * p.S + s) * H * W * 128;
  const float scale = 0.08838834764831845f;                    // 1 / sqrt(128)
  if (live) {
    for (int k = 0; k < CORR_PATCH * CORR_PATCH; ++k) {
      const int px = x0 + k % CORR_PATCH, py = y0 + k / CORR_PATCH;
      float d = 0.f;
      if (px >= 0 && px < W && py >= 0 && py < H) {              // warp-uniform
        const uint2 u = *reinterpret_cast<const uint2*>(img + (static_cast<int64_t>(py) * W + px) * 128 + lane * 4);
        const uint16_t* h = reinterpret_cast<const uint16_t*>(&u);
        d = t.x * ld16<BF16>(h) + t.y * ld16<BF16>(h + 1) + t.z * ld16<BF16>(h + 2) + t.w * ld16<BF16>(h + 3);
        d = warp_sum(d) * scale;
      }
      if (lane == 0) patch[warp][k] = d;
    }
  }
  __syncwarp();
  if (!live) return;
  uint16_t* o = reinterpret_cast<uint16_t*>(p.out) + static_cast<int64_t>(row) * p.ldo + lvl * CORR_WIN * CORR_WIN;
  for (int k = lane; k < CORR_WIN * CORR_WIN; k += 32) {
    const int i = flat_x ? CORR_R : k / CORR_WIN, j = flat_y ? CORR_R : k % CORR_WIN;   // i: x offset, j: y offset
    const float* q = &patch[warp][j * CORR_PATCH + i];
    const float v = (q[0] * (1.f - fx) + q[1] * fx) * (1.f - fy) + (q[CORR_PATCH] * (1.f - fx) + q[CORR_PATCH + 1] * fx) * fy;
    o[k] = st16<BF16>(v);
  }
  if (lvl == CORR_LEVELS - 1)
    for (int k = CORR_LEVELS * CORR_WIN * CORR_WIN + lane; k < p.ldo; k += 32)
      reinterpret_cast<uint16_t*>(p.out)[static_cast<int64_t>(row) * p.ldo + k] = 0;
}

// One warp per row (b, n, s): x = [flow embedding 128 | flow / 518 (x2) 4 | corr feature 128 | track feature 128]
//                                + pos[(b, n)] + ref_token[s > 0], then LayerNorm(388) -> 16-bit [rows, ldo] (zero padded).
// `raw` (optional, fp32 [rows, 388]) receives x before the LayerNorm (what the reference feeds its update transformer).
template <bool BF16>
__global__ void __launch_bounds__(256)
track_input_kernel(const float* __restrict__ coords, const float* __restrict__ fcorr, const float* __restrict__ tfeat,
                   const float* __restrict__ pos, const float* __restrict__ ref_tok, const float* __restrict__ ln_w,
                   const float* __restrict__ ln_b, uint16_t* __restrict__ out, float* __restrict__ raw, int rows, int S,
                   int ldo, float eps) {
  constexpr int D = 388, PER = 13;                               // 13 x 32 = 416 >= 388
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  const int s = row % S, bn = row / S;
  const float fx = coords[static_cast<int64_t>(row) * 2] - coords[static_cast<int64_t>(bn) * S * 2];
  const float fy = coords[static_cast<int64_t>(row) * 2 + 1] - coords[static_cast<int64_t>(bn) * S * 2 + 1];
  float v[PER];
  float sum = 0.f;
#pragma unroll
  for (int k = 0; k < PER; ++k) {
    const int c = lane + 32 * k;
    float x = 0.f;
    if (c < 128) {                                               // utils.py:91-127: [sin, cos] interleaved, x then y
      const int cc = c & 63;
      const float arg = (c < 64 ? fx : fy) * (static_cast<float>(cc & ~1) * (1000.0f / 64.0f));
      x = (cc & 1) ? cosf(arg) : sinf(arg);
    } else if (c < 132) {
      x = ((c & 1) ? fy : fx) / 518.0f;
    } else if (c < 260) {
      x = fcorr[static_cast<int64_t>(row) * 128 + (c - 132)];
    } else if (c < D) {
      x = tfeat[static_cast<int64_t>(row) * 128 + (c - 260)];
    }
    // (x + pos) + ref in the reference's order (base_track_predictor.py:154, 160), so these fp32 sums match it bit for bit
    if (c < D) x = (x + pos[static_cast<int64_t>(bn) * D + c]) + ref_tok[(s > 0 ? D : 0) + c];
    v[k] = x;
    sum += (c < D) ? x : 0.f;
    if (raw && c < D) raw[static_cast<int64_t>(row) * D + c] = x;
  }
  const float mean = warp_sum(sum) * (1.0f / D);
  float var = 0.f;
#pragma unroll
  for (int k = 0; k < PER; ++k) {
    const float d = v[k] - mean;
    var += (lane + 32 * k < D) ? d * d : 0.f;
  }
  const float rstd = rsqrtf(warp_sum(var) * (1.0f / D) + eps);
#pragma unroll
  for (int k = 0; k < PER; ++k) {
    const int c = lane + 32 * k;
    if (c < ldo) out[static_cast<int64_t>(row) * ldo + c] = c < D ? st16<BF16>((v[k] - mean) * rstd * ln_w[c] + ln_b[c]) : 0;
  }
}

// LayerNorm over C <= 2048 of fp32 rows (row pitch ldx): y32 (pitch C) and / or y16 (pitch ld16, zero padded) may be NULL
template <bool BF16>
__global__ void __launch_bounds__(256)
layernorm_rows_kernel(const float* __restrict__ x, int64_t ldx, int C, const float* __restrict__ w,
                      const float* __restrict__ b, float eps, int64_t rows, float* __restrict__ y32,
                      uint16_t* __restrict__ y16, int ld16) {
  const int64_t row = static_cast<int64_t>(blockIdx.x) * 8 + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  const float* xr = x + row * ldx;
  float sum = 0.f;
  for (int c = lane; c < C; c += 32) sum += xr[c];
  const float mean = warp_sum(sum) / C;
  float var = 0.f;
  for (int c = lane; c < C; c += 32) { const float d = xr[c] - mean; var += d * d; }
  const float rstd = rsqrtf(warp_sum(var) / C + eps);
  for (int c = lane; c < (y16 ? ld16 : C); c += 32) {
    const float v = c < C ? (xr[c] - mean) * rstd * w[c] + b[c] : 0.f;
    if (y32 && c < C) y32[row * C + c] = v;
    if (y16) y16[row * ld16 + c] = c < C ? st16<BF16>(v) : 0;
  }
}

inline unsigned cap_grid(int64_t work, int per_block) {
  const int64_t g = (work + per_block - 1) / per_block;
  return static_cast<unsigned>(g < 1 ? 1 : (g > 132 * 16 ? 132 * 16 : g));
}

}  // namespace iggt

using namespace iggt;

extern "C" int iggt_avgpool2_nhwc(const void* x, void* y, int NB, int H, int W, int C, int dtype, iggt_stream_t stream) {
  if (!x || !y || NB <= 0 || H < 2 || W < 2 || C <= 0 || (C & 1)) return -1;
  const int64_t total = static_cast<int64_t>(NB) * (H / 2) * (W / 2) * (C / 2);
  cudaStream_t s = (cudaStream_t)stream;
  if (dtype) avgpool2_kernel<true><<<cap_grid(total, 256), 256, 0, s>>>((const uint16_t*)x, (uint16_t*)y, NB, H, W, C);
  else avgpool2_kernel<false><<<cap_grid(total, 256), 256, 0, s>>>((const uint16_t*)x, (uint16_t*)y, NB, H, W, C);
  return (int)cudaGetLastError();
}

extern "C" int iggt_sample_bilinear_nhwc(const void* x, const float* coords, float* out, int NB, int R, int H, int W, int C,
                                         int dtype, iggt_stream_t stream) {
  if (!x || !coords || !out || NB <= 0 || R <= 0 || H <= 0 || W <= 0 || C <= 0) return -1;
  const unsigned grid = static_cast<unsigned>((static_cast<int64_t>(NB) * R + 7) / 8);
  cudaStream_t s = (cudaStream_t)stream;
  if (dtype) sample_bilinear_kernel<true><<<grid, 256, 0, s>>>((const uint16_t*)x, coords, out, NB, R, H, W, C);
  else sample_bilinear_kernel<false><<<grid, 256, 0, s>>>((const uint16_t*)x, coords, out, NB, R, H, W, C);
  return (int)cudaGetLastError();
}

extern "C" int iggt_corr_sample(const void* const* levels, const int* Hs, const int* Ws, const float* targets,
                                const float* coords, void* out, int B, int N, int S, int ldo, int dtype,
                                iggt_stream_t stream) {
  if (!levels || !Hs || !Ws || !targets || !coords || !out || B <= 0 || N <= 0 || S <= 0) return -1;
  if (ldo < CORR_LEVELS * CORR_WIN * CORR_WIN) return -2;
  CorrParams p;
  for (int l = 0; l < CORR_LEVELS; ++l) {
    if (!levels[l] || Hs[l] <= 0 || Ws[l] <= 0) return -1;
    p.level[l] = static_cast<const uint16_t*>(levels[l]); p.H[l] = Hs[l]; p.W[l] = Ws[l];
  }
  p.targets = targets; p.coords = coords; p.out = out;
  p.rows = B * N * S; p.N = N; p.S = S; p.ldo = ldo;
  const unsigned grid = static_cast<unsigned>((static_cast<int64_t>(p.rows) * CORR_LEVELS + 7) / 8);
  if (dtype) corr_sample_kernel<true><<<grid, 256, 0, (cudaStream_t)stream>>>(p);
  else corr_sample_kernel<false><<<grid, 256, 0, (cudaStream_t)stream>>>(p);
  return (int)cudaGetLastError();
}

extern "C" int iggt_track_input(const float* coords, const float* fcorr, const float* tfeat, const float* pos,
                                const float* ref_tok, const float* ln_w, const float* ln_b, void* out, float* raw,
                                int rows, int S, int ldo, float eps, int dtype, iggt_stream_t stream) {
  if (!coords || !fcorr || !tfeat || !pos || !ref_tok || !ln_w || !ln_b || !out || rows <= 0 || S <= 0) return -1;
  if (ldo < 388 || ldo > 416) return -2;
  const unsigned grid = static_cast<unsigned>((rows + 7) / 8);
  cudaStream_t s = (cudaStream_t)stream;
  if (dtype) track_input_kernel<true><<<grid, 256, 0, s>>>(coords, fcorr, tfeat, pos, ref_tok, ln_w, ln_b, (uint16_t*)out, raw, rows, S, ldo, eps);
  else track_input_kernel<false><<<grid, 256, 0, s>>>(coords, fcorr, tfeat, pos, ref_tok, ln_w, ln_b, (uint16_t*)out, raw, rows, S, ldo, eps);
  return (int)cudaGetLastError();
}

extern "C" int iggt_layernorm_rows(const float* x, int64_t ldx, int C, const float* w, const float* b, float eps,
                                   int64_t rows, float* y32, void* y16, int ld16, int dtype, iggt_stream_t stream) {
  if (!x || !w || !b || C <= 0 || C > 2048 || rows <= 0 || (!y32 && !y16) || (y16 && ld16 < C)) return -1;
  const unsigned grid = static_cast<unsigned>((rows + 7) / 8);
  cudaStream_t s = (cudaStream_t)stream;
  if (dtype) layernorm_rows_kernel<true><<<grid, 256, 0, s>>>(x, ldx, C, w, b, eps, rows, y32, (uint16_t*)y16, ld16);
  else layernorm_rows_kernel<false><<<grid, 256, 0, s>>>(x, ldx, C, w, b, eps, rows, y32, (uint16_t*)y16, ld16);
  return (int)cudaGetLastError();
}
