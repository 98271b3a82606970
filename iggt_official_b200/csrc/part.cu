// Kernels of the part (instance-feature) path that are not GEMM-shaped enough for the wgmma main loop:
// small-C LayerNorm on 16-bit NHWC rows, the k4/s2/p1 ConvTranspose gather, the two 8x8-window attentions
// (OCAB with 12x12 overlapping keys + relative-position bias and the reference's scrambled query windows;
// HAB plain window self-attention), and the CAB channel-attention (squeeze-excite) pieces.
// Reference: iggt/heads/adaptor.py:140-226, iggt/heads/part_head.py:148-243, iggt/heads/window_sa.py.
#include <stdlib.h>
#include "ptx.cuh"
#include "launch.cuh"
#include "winattn.cuh"
#include "../../include/iggt_b200.h"

namespace iggt {

template <bool BF16>
__device__ __forceinline__ float ld16(const uint16_t* p) {
  if constexpr (BF16) return __uint_as_float(static_cast<uint32_t>(*p) << 16);
  else return __half2float(__ushort_as_half(*p));
}
template <bool BF16>
__device__ __forceinline__ uint16_t st16(float v) {
  if constexpr (BF16) { __nv_bfloat16 t = __float2bfloat16_rn(v); return *reinterpret_cast<uint16_t*>(&t); }
  else { __half t = __float2half_rn(v); return *reinterpret_cast<uint16_t*>(&t); }
}

// LayerNorm over C in {64,128,256} channels of 16-bit rows (nn.LayerNorm eps 1e-5 of window_sa.py's
// patch_embed.norm / norm1 / norm2 / norm), fp32 statistics, one warp per row.
template <bool BF16, int C>
__global__ void __launch_bounds__(256)
layernorm16_kernel(const uint16_t* __restrict__ x, uint16_t* __restrict__ y, const float* __restrict__ w,
                   const float* __restrict__ b, float eps, int64_t rows) {
  constexpr int PER = C / 32;
  const int64_t r = static_cast<int64_t>(blockIdx.x) * 8 + (threadIdx.x >> 5);
  if (r >= rows) return;
  const int lane = threadIdx.x & 31;
  float v[PER];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < PER; ++i) { v[i] = ld16<BF16>(x + r * C + lane * PER + i); s += v[i]; }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  const float mean = s / C;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < PER; ++i) { const float d = v[i] - mean; q += d * d; }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
  const float rstd = rsqrtf(q / C + eps);
#pragma unroll
  for (int i = 0; i < PER; ++i) {
    const int c = lane * PER + i;
    y[r * C + c] = st16<BF16>((v[i] - mean) * rstd * __ldg(w + c) + __ldg(b + c));
  }
}

// ConvTranspose2d(k=4, s=2, p=1) gather (iggt/heads/adaptor.py:152-157): the GEMM produced
// Y[(n,iy,ix), (ky*4+kx)*C + co]; out[n,oy,ox,co] = bias + sum over the (<=4) taps with oy = 2*iy - 1 + ky.
template <bool BF16>
__global__ void __launch_bounds__(256)
col2im_k4s2p1_kernel(const uint16_t* __restrict__ Y, const float* __restrict__ bias, uint16_t* __restrict__ out,
                     int NB, int h, int w, int C) {
  const int cv = C / 8;
  const int H = 2 * h, W = 2 * w;
  const int64_t total = static_cast<int64_t>(NB) * H * W * cv;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int c8 = static_cast<int>(i % cv);
    int64_t r = i / cv;
    const int ox = static_cast<int>(r % W); r /= W;
    const int oy = static_cast<int>(r % H);
    const int n = static_cast<int>(r / H);
    float acc[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) acc[k] = __ldg(bias + c8 * 8 + k);
#pragma unroll
    for (int a = 0; a < 2; ++a) {
      const int ky = ((oy + 1) & 1) + 2 * a;       // ky == (oy+1) mod 2
      const int iy = (oy + 1 - ky) / 2;
      if (iy < 0 || iy >= h) continue;
#pragma unroll
      for (int bq = 0; bq < 2; ++bq) {
        const int kx = ((ox + 1) & 1) + 2 * bq;
        const int ix = (ox + 1 - kx) / 2;
        if (ix < 0 || ix >= w) continue;
        const uint16_t* src = Y + ((static_cast<int64_t>(n) * h + iy) * w + ix) * (16 * C) + (ky * 4 + kx) * C + c8 * 8;
        const uint4 u = __ldg(reinterpret_cast<const uint4*>(src));
        const uint32_t ww[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          uint16_t lo = static_cast<uint16_t>(ww[j] & 0xFFFF), hi = static_cast<uint16_t>(ww[j] >> 16);
          acc[2 * j] += ld16<BF16>(&lo);
          acc[2 * j + 1] += ld16<BF16>(&hi);
        }
      }
    }
    uint4 o;
    o.x = pack16x2<BF16>(acc[0], acc[1]); o.y = pack16x2<BF16>(acc[2], acc[3]);
    o.z = pack16x2<BF16>(acc[4], acc[5]); o.w = pack16x2<BF16>(acc[6], acc[7]);
    *reinterpret_cast<uint4*>(out + ((static_cast<int64_t>(n) * H + oy) * W + ox) * C + c8 * 8) = o;
  }
}

// OCAB attention (iggt/heads/window_sa.py:271-319), one CTA per (image, window, head), 256 threads.
//   q windows: the reference partitions the (b, c, h, w)-permuted Q with a (b, h, w, c) partition, so
//     q_win[n, t, f] = Q[b, yb*8+yi, x, cb*8+ci] with L = (n*64+t)*256+f decoded little-endian with radices
//     (x:w, yi:8, ci:8, yb:h/8, cb:32)                                               (SURVEY F5 / E-15)
//   k/v windows: 12x12 pixels around window (wy,wx) (rows 8wy-2 .. 8wy+9), zeros outside the map
//   scores = (q * d^-0.5) k^T + table[rpi[t, j]][head]; softmax; out written to pixel (8wy+ty, 8wx+tx).
constexpr int OC_WS = 8, OC_OWS = 12, OC_NQ = 64, OC_NK = 144, OC_D = 64, OC_C = 256;

template <bool BF16>
__global__ void __launch_bounds__(256)
ocab_attention_kernel(const uint16_t* __restrict__ Q, const uint16_t* __restrict__ K, const uint16_t* __restrict__ V,
                      const float* __restrict__ table, const int* __restrict__ rpi, uint16_t* __restrict__ out,
                      int h, int w) {
  extern __shared__ float sm[];
  float* sq = sm;                              // [64][65]
  float* sk = sq + OC_NQ * 65;                 // [144][65]
  float* sv = sk + OC_NK * 65;                 // [144][64]
  float* ss = sv + OC_NK * 64;                 // [64][145]
  const int nwx = w / OC_WS, nwy = h / OC_WS;
  const int head = blockIdx.x % 4;
  const int win = (blockIdx.x / 4) % (nwx * nwy);
  const int b = blockIdx.x / (4 * nwx * nwy);
  const int wy = win / nwx, wx = win % nwx;
  const int tid = threadIdx.x;
  const float scale = 0.125f;                  // 64^-0.5
  // scrambled query gather
  for (int i = tid; i < OC_NQ * OC_D; i += 256) {
    const int t = i / OC_D, d = i % OC_D;
    int64_t L = (static_cast<int64_t>(win) * 64 + t) * OC_C + head * OC_D + d;
    const int x = static_cast<int>(L % w); L /= w;
    const int yi = static_cast<int>(L % 8); L /= 8;
    const int ci = static_cast<int>(L % 8); L /= 8;
    const int yb = static_cast<int>(L % nwy); L /= nwy;
    const int cb = static_cast<int>(L);
    sq[t * 65 + d] = ld16<BF16>(Q + ((static_cast<int64_t>(b) * h + yb * 8 + yi) * w + x) * OC_C + cb * 8 + ci) * scale;
  }
  for (int i = tid; i < OC_NK * OC_D; i += 256) {
    const int j = i / OC_D, d = i % OC_D;
    const int yy = wy * OC_WS - 2 + j / OC_OWS, xx = wx * OC_WS - 2 + j % OC_OWS;
    float kv = 0.f, vv = 0.f;
    if (yy >= 0 && yy < h && xx >= 0 && xx < w) {
      const int64_t off = ((static_cast<int64_t>(b) * h + yy) * w + xx) * OC_C + head * OC_D + d;
      kv = ld16<BF16>(K + off);
      vv = ld16<BF16>(V + off);
    }
    sk[j * 65 + d] = kv;
    sv[j * 64 + d] = vv;
  }
  __syncthreads();
  {  // scores: thread -> 4 queries x 9 keys
    const int tq = tid / 16, tk = tid % 16;
    float acc[4][9];
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
      for (int c = 0; c < 9; ++c) acc[a][c] = 0.f;
    for (int d = 0; d < OC_D; ++d) {
      float qa[4], kb[9];
#pragma unroll
      for (int a = 0; a < 4; ++a) qa[a] = sq[(tq * 4 + a) * 65 + d];
#pragma unroll
      for (int c = 0; c < 9; ++c) kb[c] = sk[(tk * 9 + c) * 65 + d];
#pragma unroll
      for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int c = 0; c < 9; ++c) acc[a][c] = fmaf(qa[a], kb[c], acc[a][c]);
    }
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
      for (int c = 0; c < 9; ++c) {
        const int t = tq * 4 + a, j = tk * 9 + c;
        ss[t * 145 + j] = acc[a][c] + __ldg(table + __ldg(rpi + t * OC_NK + j) * 4 + head);
      }
  }
  __syncthreads();
  {  // softmax per row: warp handles 8 rows
    const int warp = tid >> 5, lane = tid & 31;
    for (int r = warp * 8; r < warp * 8 + 8; ++r) {
      float mx = -INFINITY;
      for (int j = lane; j < OC_NK; j += 32) mx = fmaxf(mx, ss[r * 145 + j]);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
      float sum = 0.f;
      for (int j = lane; j < OC_NK; j += 32) { const float e = expf(ss[r * 145 + j] - mx); ss[r * 145 + j] = e; sum += e; }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
      const float inv = 1.0f / sum;
      for (int j = lane; j < OC_NK; j += 32) ss[r * 145 + j] *= inv;
    }
  }
  __syncthreads();
  {  // P V: thread -> 4 queries x 4 dims
    const int tq = tid / 16, td = tid % 16;
    float acc[4][4];
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
      for (int c = 0; c < 4; ++c) acc[a][c] = 0.f;
    for (int j = 0; j < OC_NK; ++j) {
      float pa[4], vb[4];
#pragma unroll
      for (int a = 0; a < 4; ++a) pa[a] = ss[(tq * 4 + a) * 145 + j];
#pragma unroll
      for (int c = 0; c < 4; ++c) vb[c] = sv[j * 64 + td * 4 + c];
#pragma unroll
      for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int c = 0; c < 4; ++c) acc[a][c] = fmaf(pa[a], vb[c], acc[a][c]);
    }
#pragma unroll
    for (int a = 0; a < 4; ++a) {
      const int t = tq * 4 + a;
      const int yy = wy * OC_WS + t / OC_WS, xx = wx * OC_WS + t % OC_WS;
      uint16_t* dst = out + ((static_cast<int64_t>(b) * h + yy) * w + xx) * OC_C + head * OC_D + td * 4;
      uint2 u;
      u.x = pack16x2<BF16>(acc[a][0], acc[a][1]);
      u.y = pack16x2<BF16>(acc[a][2], acc[a][3]);
      *reinterpret_cast<uint2*>(dst) = u;
    }
  }
}
constexpr int OCAB_SMEM = (OC_NQ * 65 + OC_NK * 65 + OC_NK * 64 + OC_NQ * 145) * 4;

// HAB window self-attention (iggt/heads/window_sa.py:201-227 + iggt/heads/block.py:113-130): 8x8 windows,
// 4 heads x 32, scale 32^-0.5, no bias / mask.  qkv [NB,h,w,384] = [q | k | v], head-major inside each.
// One CTA per (image, window, head), 128 threads.
template <bool BF16>
__global__ void __launch_bounds__(128)
window_attention_kernel(const uint16_t* __restrict__ qkv, uint16_t* __restrict__ out, int h, int w) {
  __shared__ float sq[64 * 33], sk[64 * 33], sv[64 * 32], ss[64 * 65];
  const int nwx = w / 8, nwy = h / 8;
  const int head = blockIdx.x % 4;
  const int win = (blockIdx.x / 4) % (nwx * nwy);
  const int b = blockIdx.x / (4 * nwx * nwy);
  const int wy = win / nwx, wx = win % nwx;
  const int tid = threadIdx.x;
  const float scale = 0.17677669529663687f;    // 32^-0.5
  for (int i = tid; i < 64 * 32; i += 128) {
    const int t = i / 32, d = i % 32;
    const int64_t pix = (static_cast<int64_t>(b) * h + wy * 8 + t / 8) * w + wx * 8 + t % 8;
    const uint16_t* p = qkv + pix * 384 + head * 32 + d;
    sq[t * 33 + d] = ld16<BF16>(p) * scale;
    sk[t * 33 + d] = ld16<BF16>(p + 128);
    sv[t * 32 + d] = ld16<BF16>(p + 256);
  }
  __syncthreads();
  {  // scores: thread -> 4 q x 8 k
    const int tq = tid / 8, tk = tid % 8;
    float acc[4][8];
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
      for (int c = 0; c < 8; ++c) acc[a][c] = 0.f;
    for (int d = 0; d < 32; ++d) {
      float qa[4], kb[8];
#pragma unroll
      for (int a = 0; a < 4; ++a) qa[a] = sq[(tq * 4 + a) * 33 + d];
#pragma unroll
      for (int c = 0; c < 8; ++c) kb[c] = sk[(tk * 8 + c) * 33 + d];
#pragma unroll
      for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int c = 0; c < 8; ++c) acc[a][c] = fmaf(qa[a], kb[c], acc[a][c]);
    }
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
      for (int c = 0; c < 8; ++c) ss[(tq * 4 + a) * 65 + tk * 8 + c] = acc[a][c];
  }
  __syncthreads();
  {
    const int warp = tid >> 5, lane = tid & 31;
    for (int r = warp * 16; r < warp * 16 + 16; ++r) {
      const float a0 = ss[r * 65 + lane], a1 = ss[r * 65 + lane + 32];
      float mx = fmaxf(a0, a1);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
      const float e0 = expf(a0 - mx), e1 = expf(a1 - mx);
      float sum = e0 + e1;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
      const float inv = 1.0f / sum;
      ss[r * 65 + lane] = e0 * inv;
      ss[r * 65 + lane + 32] = e1 * inv;
    }
  }
  __syncthreads();
  {  // P V: thread -> 4 q x 4 d
    const int tq = tid / 8, td = tid % 8;
    float acc[4][4];
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
      for (int c = 0; c < 4; ++c) acc[a][c] = 0.f;
    for (int j = 0; j < 64; ++j) {
      float pa[4], vb[4];
#pragma unroll
      for (int a = 0; a < 4; ++a) pa[a] = ss[(tq * 4 + a) * 65 + j];
#pragma unroll
      for (int c = 0; c < 4; ++c) vb[c] = sv[j * 32 + td * 4 + c];
#pragma unroll
      for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int c = 0; c < 4; ++c) acc[a][c] = fmaf(pa[a], vb[c], acc[a][c]);
    }
#pragma unroll
    for (int a = 0; a < 4; ++a) {
      const int t = tq * 4 + a;
      const int64_t pix = (static_cast<int64_t>(b) * h + wy * 8 + t / 8) * w + wx * 8 + t % 8;
      uint2 u;
      u.x = pack16x2<BF16>(acc[a][0], acc[a][1]);
      u.y = pack16x2<BF16>(acc[a][2], acc[a][3]);
      *reinterpret_cast<uint2*>(out + pix * 128 + head * 32 + td * 4) = u;
    }
  }
}

// CAB channel attention, part 1: per-image channel means of x[NB, HW, C] (16-bit) -> mean[NB, C] fp32
// (nn.AdaptiveAvgPool2d(1), iggt/heads/window_sa.py:26-38).  Grid (NB, chunks); atomics on a zeroed buffer.
template <bool BF16>
__global__ void __launch_bounds__(256)
channel_mean_kernel(const uint16_t* __restrict__ x, float* __restrict__ mean, int64_t hw, int C, float inv_hw) {
  const int n = blockIdx.y;
  const int c = threadIdx.x % C;               // C <= 256 and 256 % C == 0
  const int lanes = 256 / C;
  const int sub = threadIdx.x / C;
  float acc = 0.f;
  for (int64_t p = static_cast<int64_t>(blockIdx.x) * lanes + sub; p < hw; p += static_cast<int64_t>(gridDim.x) * lanes)
    acc += ld16<BF16>(x + (static_cast<int64_t>(n) * hw + p) * C + c);
  atomicAdd(mean + static_cast<int64_t>(n) * C + c, acc * inv_hw);
}

// CAB part 2 + HAB combine: y[pix, c] = y0[pix, c] + alpha * cx[pix, c] * sigmoid(W2 relu(W1 mean_n + b1) + b2)[c]
// (ChannelAttention + `shortcut + attn + conv_x * conv_scale`, window_sa.py:26-38,225).  C = 128, squeeze R.
template <bool BF16>
__global__ void __launch_bounds__(256)
se_scale_add_kernel(const uint16_t* __restrict__ y0, const uint16_t* __restrict__ cx, const float* __restrict__ mean,
                    const float* __restrict__ w1, const float* __restrict__ b1, const float* __restrict__ w2,
                    const float* __restrict__ b2, uint16_t* __restrict__ y, int64_t hw, int C, int R, float alpha) {
  __shared__ float s_scale[256];
  __shared__ float s_hid[16];
  const int n = blockIdx.y;
  if (threadIdx.x < R) {
    float a = b1[threadIdx.x];
    for (int c = 0; c < C; ++c) a = fmaf(w1[threadIdx.x * C + c], mean[static_cast<int64_t>(n) * C + c], a);
    s_hid[threadIdx.x] = relu_nan(a);
  }
  __syncthreads();
  if (threadIdx.x < C) {
    float a = b2[threadIdx.x];
    for (int r = 0; r < R; ++r) a = fmaf(w2[threadIdx.x * R + r], s_hid[r], a);
    s_scale[threadIdx.x] = alpha / (1.0f + expf(-a));
  }
  __syncthreads();
  const int cv = C / 8;
  const int64_t total = hw * cv;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int c8 = static_cast<int>(i % cv);
    const int64_t off = (static_cast<int64_t>(n) * hw + i / cv) * C + c8 * 8;
    const uint4 a = __ldg(reinterpret_cast<const uint4*>(y0 + off));
    const uint4 c = __ldg(reinterpret_cast<const uint4*>(cx + off));
    const uint32_t aw[4] = {a.x, a.y, a.z, a.w}, cw[4] = {c.x, c.y, c.z, c.w};
    float o[8];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      uint16_t al = aw[j] & 0xFFFF, ah = aw[j] >> 16, cl = cw[j] & 0xFFFF, ch = cw[j] >> 16;
      o[2 * j] = ld16<BF16>(&al) + ld16<BF16>(&cl) * s_scale[c8 * 8 + 2 * j];
      o[2 * j + 1] = ld16<BF16>(&ah) + ld16<BF16>(&ch) * s_scale[c8 * 8 + 2 * j + 1];
    }
    uint4 u;
    u.x = pack16x2<BF16>(o[0], o[1]); u.y = pack16x2<BF16>(o[2], o[3]);
    u.z = pack16x2<BF16>(o[4], o[5]); u.w = pack16x2<BF16>(o[6], o[7]);
    *reinterpret_cast<uint4*>(y + off) = u;
  }
}

inline unsigned grid_cap(int64_t total, int threads = 256) {
  int64_t g = (total + threads - 1) / threads;
  const int64_t cap = 132 * 16;
  return static_cast<unsigned>(g < cap ? (g > 0 ? g : 1) : cap);
}

}  // namespace iggt

using namespace iggt;

namespace {
int winattn_tc() {
  static const int v = [] { const char* e = getenv("IGGT_WINATTN_TC"); return e ? atoi(e) : 1; }();
  return v;
}
}  // namespace

extern "C" int iggt_layernorm16(const void* x, void* y, int64_t rows, int C, const float* w, const float* b,
                                float eps, int dtype, iggt_stream_t stream) {
  if (rows <= 0) return 0;
  if (!w || !b) return -1;
  const unsigned grid = static_cast<unsigned>((rows + 7) / 8);
  cudaStream_t s = (cudaStream_t)stream;
#define L16(BF, CC) layernorm16_kernel<BF, CC><<<grid, 256, 0, s>>>((const uint16_t*)x, (uint16_t*)y, w, b, eps, rows)
  if (C == 256) { if (dtype) L16(true, 256); else L16(false, 256); }
  else if (C == 128) { if (dtype) L16(true, 128); else L16(false, 128); }
  else if (C == 64) { if (dtype) L16(true, 64); else L16(false, 64); }
  else return -1;
#undef L16
  return (int)cudaGetLastError();
}

extern "C" int iggt_col2im_k4s2p1(const void* Y, const float* bias, void* out, int NB, int h, int w, int C,
                                  int dtype, iggt_stream_t stream) {
  if (NB <= 0 || (C % 8) || !bias) return -1;
  const int64_t total = static_cast<int64_t>(NB) * 4 * h * w * (C / 8);
  if (dtype) col2im_k4s2p1_kernel<true><<<grid_cap(total), 256, 0, (cudaStream_t)stream>>>((const uint16_t*)Y, bias, (uint16_t*)out, NB, h, w, C);
  else col2im_k4s2p1_kernel<false><<<grid_cap(total), 256, 0, (cudaStream_t)stream>>>((const uint16_t*)Y, bias, (uint16_t*)out, NB, h, w, C);
  return (int)cudaGetLastError();
}

extern "C" int iggt_ocab_attention(const void* q, const void* k, const void* v, const float* table, const int* rpi,
                                   void* out, int NB, int h, int w, int dtype, iggt_stream_t stream) {
  if (NB <= 0 || (h % 8) || (w % 8)) return -1;
  static DeviceOnce once;
  if (once.first()) {
    cudaFuncSetAttribute(ocab_attention_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, OCAB_SMEM);
    cudaFuncSetAttribute(ocab_attention_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, OCAB_SMEM);
    cudaFuncSetAttribute(ocab_attention_tc_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, OA_SMEM);
    cudaFuncSetAttribute(ocab_attention_tc_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, OA_SMEM);
  }
  const unsigned grid = static_cast<unsigned>(NB) * (h / 8) * (w / 8) * 4;
  if (winattn_tc()) {      // tensor-core kernel (winattn.cuh); IGGT_WINATTN_TC=0 selects the scalar fp32 kernel below
    if (dtype) ocab_attention_tc_kernel<true><<<grid, 128, OA_SMEM, (cudaStream_t)stream>>>((const uint16_t*)q, (const uint16_t*)k, (const uint16_t*)v, table, rpi, (uint16_t*)out, h, w);
    else ocab_attention_tc_kernel<false><<<grid, 128, OA_SMEM, (cudaStream_t)stream>>>((const uint16_t*)q, (const uint16_t*)k, (const uint16_t*)v, table, rpi, (uint16_t*)out, h, w);
    return (int)cudaGetLastError();
  }
  if (dtype) ocab_attention_kernel<true><<<grid, 256, OCAB_SMEM, (cudaStream_t)stream>>>((const uint16_t*)q, (const uint16_t*)k, (const uint16_t*)v, table, rpi, (uint16_t*)out, h, w);
  else ocab_attention_kernel<false><<<grid, 256, OCAB_SMEM, (cudaStream_t)stream>>>((const uint16_t*)q, (const uint16_t*)k, (const uint16_t*)v, table, rpi, (uint16_t*)out, h, w);
  return (int)cudaGetLastError();
}

extern "C" int iggt_window_attention(const void* qkv, void* out, int NB, int h, int w, int dtype,
                                     iggt_stream_t stream) {
  if (NB <= 0 || (h % 8) || (w % 8)) return -1;
  const unsigned grid = static_cast<unsigned>(NB) * (h / 8) * (w / 8) * 4;
  if (winattn_tc()) {
    if (dtype) window_attention_tc_kernel<true><<<grid, 128, 0, (cudaStream_t)stream>>>((const uint16_t*)qkv, (uint16_t*)out, h, w);
    else window_attention_tc_kernel<false><<<grid, 128, 0, (cudaStream_t)stream>>>((const uint16_t*)qkv, (uint16_t*)out, h, w);
    return (int)cudaGetLastError();
  }
  if (dtype) window_attention_kernel<true><<<grid, 128, 0, (cudaStream_t)stream>>>((const uint16_t*)qkv, (uint16_t*)out, h, w);
  else window_attention_kernel<false><<<grid, 128, 0, (cudaStream_t)stream>>>((const uint16_t*)qkv, (uint16_t*)out, h, w);
  return (int)cudaGetLastError();
}

extern "C" int iggt_channel_mean(const void* x, float* mean, int NB, int64_t hw, int C, int dtype,
                                 iggt_stream_t stream) {
  if (NB <= 0 || C <= 0 || C > 256 || (256 % C)) return -1;
  cudaError_t e = cudaMemsetAsync(mean, 0, sizeof(float) * NB * C, (cudaStream_t)stream);
  if (e != cudaSuccess) return (int)e;
  dim3 grid(static_cast<unsigned>(hw / 64 > 0 ? (hw / 64 < 296 ? hw / 64 : 296) : 1), NB);
  if (dtype) channel_mean_kernel<true><<<grid, 256, 0, (cudaStream_t)stream>>>((const uint16_t*)x, mean, hw, C, 1.0f / hw);
  else channel_mean_kernel<false><<<grid, 256, 0, (cudaStream_t)stream>>>((const uint16_t*)x, mean, hw, C, 1.0f / hw);
  return (int)cudaGetLastError();
}

extern "C" int iggt_se_scale_add(const void* y0, const void* cx, const float* mean, const float* w1, const float* b1,
                                 const float* w2, const float* b2, void* y, int NB, int64_t hw, int C, int R,
                                 float alpha, int dtype, iggt_stream_t stream) {
  if (NB <= 0 || C > 256 || (C % 8) || R > 16) return -1;
  dim3 grid(grid_cap(hw * (C / 8)) / 2 + 1, NB);
  if (dtype) se_scale_add_kernel<true><<<grid, 256, 0, (cudaStream_t)stream>>>((const uint16_t*)y0, (const uint16_t*)cx, mean, w1, b1, w2, b2, (uint16_t*)y, hw, C, R, alpha);
  else se_scale_add_kernel<false><<<grid, 256, 0, (cudaStream_t)stream>>>((const uint16_t*)y0, (const uint16_t*)cx, mean, w1, b1, w2, b2, (uint16_t*)y, hw, C, R, alpha);
  return (int)cudaGetLastError();
}
