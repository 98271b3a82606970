// HBM-bound kernels of the dense heads and the camera head (all NHWC 16-bit activations unless noted):
// bilinear(align_corners) upsample fused with the UV sinusoid pos-embed, deconv pixel-shuffle, stride-2
// im2col, the per-pixel 1x1 + activation tail, a skinny (M <= 32) weight-streaming GEMM and a tiny
// attention for the S camera tokens.  Coalesced 16-byte accesses, grid-stride loops.
#include "ptx.cuh"
#include "tmap.cuh"
#include "launch.cuh"
#include "../../include/iggt_b200.h"

namespace iggt {

template <bool BF16>
__device__ __forceinline__ void unpack8(const uint4& u, float (&f)[8]) {
  const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    if constexpr (BF16) {
      f[2 * j] = __uint_as_float(w[j] << 16);
      f[2 * j + 1] = __uint_as_float(w[j] & 0xFFFF0000u);
    } else {
      const __half2 h = *reinterpret_cast<const __half2*>(&w[j]);
      f[2 * j] = __low2float(h);
      f[2 * j + 1] = __high2float(h);
    }
  }
}
template <bool BF16>
__device__ __forceinline__ uint4 pack8(const float (&f)[8]) {
  uint4 u;
  u.x = pack16x2<BF16>(f[0], f[1]); u.y = pack16x2<BF16>(f[2], f[3]);
  u.z = pack16x2<BF16>(f[4], f[5]); u.w = pack16x2<BF16>(f[6], f[7]);
  return u;
}

// F.interpolate(mode="bilinear", align_corners=True) on NHWC (iggt/heads/dpt_head.py:251-256,478,484-509)
// + optional pos-embed: channels [0,C/2) get tabx[x][c], [C/2,C) get taby[y][c-C/2]
// (iggt/heads/dpt_head.py:274-284, iggt/heads/utils.py:11-108; tables are built on the host in float64).
template <bool BF16>
__device__ __forceinline__ float2 cvt16x2(uint32_t u) {
  if constexpr (BF16) return make_float2(__uint_as_float(u << 16), __uint_as_float(u & 0xFFFF0000u));
  else return __half22float2(*reinterpret_cast<const __half2*>(&u));
}
// One CTA per output row (n, oy): the vertical taps / weights are row constants, a thread walks (ox, 8-channel group)
// items of the row.  Index arithmetic stays 32-bit; the four-tap blend runs on fp32 pairs (same IEEE results as scalar
// code).
template <bool BF16>
__global__ void __launch_bounds__(256)
upsample_bilinear_kernel(const uint16_t* __restrict__ x, uint16_t* __restrict__ out, int NB, int h, int w,
                         int H, int W, int C, const float* __restrict__ tabx, const float* __restrict__ taby) {
  const int cv = C / 8;
  const int row = blockIdx.x;                                   // n * H + oy
  const int n = row / H, oy = row - n * H;
  const float sy = H > 1 ? static_cast<float>(h - 1) / static_cast<float>(H - 1) : 0.f;
  const float sx = W > 1 ? static_cast<float>(w - 1) / static_cast<float>(W - 1) : 0.f;
  const float fy = sy * oy;
  const int y0 = static_cast<int>(fy);
  const int y1 = min(y0 + 1, h - 1);
  const float ly = fy - y0, hy = 1.f - ly;
  const uint16_t* r0 = x + (static_cast<int64_t>(n) * h + y0) * w * C;
  const uint16_t* r1 = x + (static_cast<int64_t>(n) * h + y1) * w * C;
  uint16_t* orow = out + static_cast<int64_t>(row) * W * C;
  const int half = C / 2;
  const int items = W * cv;
  for (int i = threadIdx.x; i < items; i += blockDim.x) {
    const int ox = i / cv, c8 = i - ox * cv;
    const float fx = sx * ox;
    const int x0 = static_cast<int>(fx);
    const int x1 = min(x0 + 1, w - 1);
    const float lx = fx - x0, hx = 1.f - lx;
    const uint4 ua = __ldg(reinterpret_cast<const uint4*>(r0 + x0 * C + c8 * 8));
    const uint4 ub = __ldg(reinterpret_cast<const uint4*>(r0 + x1 * C + c8 * 8));
    const uint4 uc = __ldg(reinterpret_cast<const uint4*>(r1 + x0 * C + c8 * 8));
    const uint4 ud = __ldg(reinterpret_cast<const uint4*>(r1 + x1 * C + c8 * 8));
    const uint32_t wa[4] = {ua.x, ua.y, ua.z, ua.w}, wb[4] = {ub.x, ub.y, ub.z, ub.w};
    const uint32_t wc[4] = {uc.x, uc.y, uc.z, uc.w}, wd[4] = {ud.x, ud.y, ud.z, ud.w};
    const float2 hx2 = make_float2(hx, hx), lx2 = make_float2(lx, lx), hy2 = make_float2(hy, hy), ly2 = make_float2(ly, ly);
    float2 o[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      // hy * (hx * a + lx * b) + ly * (hx * c + lx * d), operation for operation as the scalar form
      const float2 top = ffma2(lx2, cvt16x2<BF16>(wb[k]), fmul2(hx2, cvt16x2<BF16>(wa[k])));
      const float2 bot = ffma2(lx2, cvt16x2<BF16>(wd[k]), fmul2(hx2, cvt16x2<BF16>(wc[k])));
      o[k] = ffma2(ly2, bot, fmul2(hy2, top));
    }
    if (tabx) {
      const int ch = c8 * 8;
      const float* t = ch < half ? tabx + ox * half + ch : taby + oy * half + (ch - half);
      const float4 t0 = __ldg(reinterpret_cast<const float4*>(t)), t1 = __ldg(reinterpret_cast<const float4*>(t) + 1);
      o[0] = fadd2(o[0], make_float2(t0.x, t0.y)); o[1] = fadd2(o[1], make_float2(t0.z, t0.w));
      o[2] = fadd2(o[2], make_float2(t1.x, t1.y)); o[3] = fadd2(o[3], make_float2(t1.z, t1.w));
    }
    uint4 u;
    u.x = pack16x2<BF16>(o[0].x, o[0].y); u.y = pack16x2<BF16>(o[1].x, o[1].y);
    u.z = pack16x2<BF16>(o[2].x, o[2].y); u.w = pack16x2<BF16>(o[3].x, o[3].y);
    *reinterpret_cast<uint4*>(orow + ox * C + c8 * 8) = u;
  }
}

// ConvTranspose2d with kernel == stride (iggt/heads/dpt_head.py:85-92): the GEMM produced
// y[pixel, (dy*k+dx)*C + co]; scatter to NHWC out[n, k*yy+dy, k*xx+dx, co].
__global__ void __launch_bounds__(256)
deconv_shuffle_kernel(const uint4* __restrict__ y, uint4* __restrict__ out, int NB, int h, int w, int C, int k) {
  const int cv = C / 8;
  const int64_t total = static_cast<int64_t>(NB) * h * w * k * k * cv;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int c8 = static_cast<int>(i % cv);
    int64_t r = i / cv;
    const int tap = static_cast<int>(r % (k * k)); r /= (k * k);
    const int xx = static_cast<int>(r % w); r /= w;
    const int yy = static_cast<int>(r % h);
    const int n = static_cast<int>(r / h);
    const int dy = tap / k, dx = tap % k;
    const int64_t dst = ((static_cast<int64_t>(n) * h * k + yy * k + dy) * (w * k) + xx * k + dx) * cv + c8;
    out[dst] = __ldg(y + i);
  }
}

// im2col for the one stride-2 3x3 conv (pad 1) of each head (iggt/heads/dpt_head.py:94-97):
// A[(n,oy,ox), tap*C + c] = x[n, 2oy+ky-1, 2ox+kx-1, c] (zero outside).
__global__ void __launch_bounds__(256)
im2col_s2_kernel(const uint4* __restrict__ x, uint4* __restrict__ A, int NB, int h, int w, int C, int ho, int wo) {
  const int cv = C / 8;
  const int64_t total = static_cast<int64_t>(NB) * ho * wo * 9 * cv;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int c8 = static_cast<int>(i % cv);
    int64_t r = i / cv;
    const int tap = static_cast<int>(r % 9); r /= 9;
    const int ox = static_cast<int>(r % wo); r /= wo;
    const int oy = static_cast<int>(r % ho);
    const int n = static_cast<int>(r / ho);
    const int iy = 2 * oy + tap / 3 - 1, ix = 2 * ox + tap % 3 - 1;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (iy >= 0 && iy < h && ix >= 0 && ix < w) v = __ldg(x + ((static_cast<int64_t>(n) * h + iy) * w + ix) * cv + c8);
    A[i] = v;
  }
}

// Per-pixel tail: 1x1 conv 32 -> OC (fp32 weights) + head activation (iggt/heads/dpt_head.py:264-265,
// iggt/heads/head_act.py:61-125).  mode 0: xyz=exp, conf=1+exp (depth); 1: xyz=sign*expm1|.|, conf=1+exp
// (points); 2: raw, channels-first [NB,OC,H,W] (part_feat, iggt/heads/part_head.py:240-243).
template <bool BF16, int OC>
__global__ void __launch_bounds__(256)
dpt_tail_kernel(const uint16_t* __restrict__ x, const float* __restrict__ w, const float* __restrict__ b,
                float* __restrict__ out_main, float* __restrict__ out_conf, int64_t npix, int64_t hw, int mode) {
  __shared__ float sw[OC * 32 + OC];
  for (int i = threadIdx.x; i < OC * 32 + OC; i += blockDim.x) sw[i] = i < OC * 32 ? w[i] : b[i - OC * 32];
  __syncthreads();
  for (int64_t pix = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; pix < npix;
       pix += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    float f[32];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      float t[8];
      unpack8<BF16>(__ldg(reinterpret_cast<const uint4*>(x + pix * 32) + q), t);
#pragma unroll
      for (int k = 0; k < 8; ++k) f[q * 8 + k] = t[k];
    }
    float o[OC];
#pragma unroll
    for (int c = 0; c < OC; ++c) {
      float s = sw[OC * 32 + c];
#pragma unroll
      for (int k = 0; k < 32; ++k) s = fmaf(f[k], sw[c * 32 + k], s);
      o[c] = s;
    }
    if (mode == 2) {
      const int64_t n = pix / hw, r = pix % hw;
#pragma unroll
      for (int c = 0; c < OC; ++c) out_main[(n * OC + c) * hw + r] = o[c];
    } else {
#pragma unroll
      for (int c = 0; c < OC - 1; ++c) {
        const float v = o[c];
        out_main[pix * (OC - 1) + c] = mode == 0 ? expf(v) : copysignf(expm1f(fabsf(v)), v);
      }
      out_conf[pix] = 1.0f + expf(o[OC - 1]);
    }
  }
}

// out[m, n] = (resid ? resid[m,n] : 0) + gamma[n] * act(x[m,:] . W[n,:] + bias[n]),  M <= 8 rows per launch
// (the host loops over row chunks), fp32 activations, 16-bit weights streamed once.  Camera-head Linear layers
// (iggt/heads/camera_head.py:83-154): 8 rows against up to 33 MB of weights -> purely weight-bandwidth bound, so
// no tensor cores; the job is to keep ~100 KB of loads in flight per SM.  A producer thread streams
// {32 columns x 256 k} weight boxes and the matching {8 rows x 256 k} activation box through a 6-stage TMA /
// mbarrier ring; consumer warp w owns columns 4w..4w+3 (lane = 8 consecutive k), accumulates 4 x 8 dot products
// in registers and reduces them with shuffles at the end.
constexpr int SK_COLS = 32;     // columns per CTA
constexpr int SK_KC = 256;      // k per stage
constexpr int SK_STAGES = 6;
constexpr int SK_W_BYTES = SK_COLS * SK_KC * 2;   // 16 KB
constexpr int SK_X_BYTES = 8 * SK_KC * 4;         // 8 KB
constexpr int SK_SMEM = SK_STAGES * (SK_W_BYTES + SK_X_BYTES) + 256;
template <bool BF16>
__global__ void __launch_bounds__(288)
skinny_gemm_kernel(const __grid_constant__ CUtensorMap tmW, const __grid_constant__ CUtensorMap tmX,
                   const float* __restrict__ bias, const float* __restrict__ gamma, const float* resid,
                   int64_t ldr, float* out, int64_t ldo, int M, int N, int K, int act) {
  extern __shared__ __align__(128) uint8_t sk_smem[];
  uint8_t* sW = sk_smem;
  uint8_t* sX = sk_smem + SK_STAGES * SK_W_BYTES;
  uint64_t* full = reinterpret_cast<uint64_t*>(sX + SK_STAGES * SK_X_BYTES);
  uint64_t* empty = full + SK_STAGES;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n0 = blockIdx.x * SK_COLS;
  const int nk = (K + SK_KC - 1) / SK_KC;
  if (threadIdx.x == 0) {
    for (int i = 0; i < SK_STAGES; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], 8); }
    fence_barrier_init();
  }
  __syncthreads();
  griddep_wait();
  griddep_launch();
  if (warp == 8) {
    if (lane == 0) {
      int st = 0; uint32_t ph = 0;
      for (int kb = 0; kb < nk; ++kb) {
        mbar_wait(&empty[st], ph ^ 1);
        mbar_expect_tx(&full[st], SK_W_BYTES + SK_X_BYTES);
        tma_load_2d(sW + st * SK_W_BYTES, &tmW, &full[st], kb * SK_KC, n0);
        tma_load_2d(sX + st * SK_X_BYTES, &tmX, &full[st], kb * SK_KC, 0);
        if (++st == SK_STAGES) { st = 0; ph ^= 1; }
      }
    }
    return;
  }
  float acc[4][8];
#pragma unroll
  for (int c = 0; c < 4; ++c)
#pragma unroll
    for (int m = 0; m < 8; ++m) acc[c][m] = 0.f;
  int st = 0; uint32_t ph = 0;
  for (int kb = 0; kb < nk; ++kb) {
    mbar_wait(&full[st], ph);
    const uint16_t* w = reinterpret_cast<const uint16_t*>(sW + st * SK_W_BYTES) + (warp * 4) * SK_KC + lane * 8;
    const float* xs = reinterpret_cast<const float*>(sX + st * SK_X_BYTES) + lane * 8;
    float xr[8][8];
#pragma unroll
    for (int m = 0; m < 8; ++m) {
      const float4 a = *reinterpret_cast<const float4*>(xs + m * SK_KC);
      const float4 b = *reinterpret_cast<const float4*>(xs + m * SK_KC + 4);
      xr[m][0] = a.x; xr[m][1] = a.y; xr[m][2] = a.z; xr[m][3] = a.w;
      xr[m][4] = b.x; xr[m][5] = b.y; xr[m][6] = b.z; xr[m][7] = b.w;
    }
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      float wf[8];
      unpack8<BF16>(*reinterpret_cast<const uint4*>(w + c * SK_KC), wf);
#pragma unroll
      for (int m = 0; m < 8; ++m)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[c][m] = fmaf(xr[m][j], wf[j], acc[c][m]);
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[st]);
    if (++st == SK_STAGES) { st = 0; ph ^= 1; }
  }
#pragma unroll
  for (int c = 0; c < 4; ++c)
#pragma unroll
    for (int m = 0; m < 8; ++m) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) acc[c][m] += __shfl_xor_sync(0xffffffffu, acc[c][m], o);
    }
  {
    const int c = lane / 8, m = lane % 8;
    const int n = n0 + warp * 4 + c;
    float v = 0.f;
#pragma unroll
    for (int cc = 0; cc < 4; ++cc)
#pragma unroll
      for (int mm = 0; mm < 8; ++mm) if (cc * 8 + mm == lane) v = acc[cc][mm];
    if (n < N && m < M) {
      v += bias ? bias[n] : 0.f;
      if (act == 1) v = gelu_erf(v);
      else if (act == 2) v = relu_nan(v);
      else if (act == 4) v = v / (1.0f + expf(-v));  // SiLU
      v *= gamma ? gamma[n] : 1.f;
      if (resid) v += resid[m * ldr + n];
      out[m * ldo + n] = v;
    }
  }
}

// softmax(q k^T / sqrt(d)) v for tiny sequences (camera tokens: N <= 64 views, d <= 128), fp32.
// qkv [B*N, 3*H*d] (q | k | v, head-major inside each), out [B*N, H*d]. One CTA per (b, head).
__global__ void __launch_bounds__(128)
small_attention_kernel(const float* __restrict__ qkv, float* __restrict__ out, int N, int H, int d, float scale) {
  extern __shared__ float sm[];
  float* sk = sm;                 // [N][d]
  float* sv = sm + N * d;         // [N][d]
  float* sp = sv + N * d;         // [4 warps][N]
  const int b = blockIdx.x / H, hh = blockIdx.x % H;
  const int C = H * d;
  for (int i = threadIdx.x; i < N * d; i += blockDim.x) {
    const int r = i / d, c = i % d;
    const float* row = qkv + static_cast<int64_t>(b * N + r) * 3 * C + hh * d + c;
    sk[i] = row[C];
    sv[i] = row[2 * C];
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* p = sp + warp * N;
  for (int qi = warp; qi < N; qi += 4) {
    const float* q = qkv + static_cast<int64_t>(b * N + qi) * 3 * C + hh * d;
    float mx = -INFINITY;
    for (int j = lane; j < N; j += 32) {
      float s = 0.f;
      for (int c = 0; c < d; ++c) s = fmaf(q[c], sk[j * d + c], s);
      s *= scale;
      p[j] = s;
      mx = fmaxf(mx, s);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    float sum = 0.f;
    for (int j = lane; j < N; j += 32) { const float e = expf(p[j] - mx); p[j] = e; sum += e; }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    __syncwarp();
    const float inv = 1.0f / sum;
    for (int c = lane; c < d; c += 32) {
      float acc = 0.f;
      for (int j = 0; j < N; ++j) acc = fmaf(p[j], sv[j * d + c], acc);
      out[static_cast<int64_t>(b * N + qi) * C + hh * d + c] = acc * inv;
    }
    __syncwarp();
  }
}

inline unsigned grid_for(int64_t total, int threads = 256) {
  int64_t g = (total + threads - 1) / threads;
  const int64_t cap = 132 * 16;
  return static_cast<unsigned>(g < cap ? (g > 0 ? g : 1) : cap);
}

}  // namespace iggt

using namespace iggt;

extern "C" int iggt_upsample_bilinear_nhwc(const void* x, void* out, int NB, int h, int w, int H, int W, int C,
                                           const float* tabx, const float* taby, int dtype, iggt_stream_t stream) {
  if (NB <= 0 || h <= 0 || w <= 0 || H <= 0 || W <= 0 || (C % 16)) return -1;
  if ((tabx == nullptr) != (taby == nullptr)) return -1;
  if (static_cast<int64_t>(NB) * H > 0x7fffffff || static_cast<int64_t>(w) * C > 0x7fffffff) return -1;
  const unsigned rows = static_cast<unsigned>(NB) * H;                 // one CTA per output row
  if (dtype) upsample_bilinear_kernel<true><<<rows, 256, 0, (cudaStream_t)stream>>>(
      (const uint16_t*)x, (uint16_t*)out, NB, h, w, H, W, C, tabx, taby);
  else upsample_bilinear_kernel<false><<<rows, 256, 0, (cudaStream_t)stream>>>(
      (const uint16_t*)x, (uint16_t*)out, NB, h, w, H, W, C, tabx, taby);
  return (int)cudaGetLastError();
}

extern "C" int iggt_deconv_shuffle(const void* y, void* out, int NB, int h, int w, int C, int k, iggt_stream_t stream) {
  if (NB <= 0 || (C % 8) || k <= 0) return -1;
  const int64_t total = static_cast<int64_t>(NB) * h * w * k * k * (C / 8);
  deconv_shuffle_kernel<<<grid_for(total), 256, 0, (cudaStream_t)stream>>>((const uint4*)y, (uint4*)out, NB, h, w, C, k);
  return (int)cudaGetLastError();
}

extern "C" int iggt_im2col3x3_s2(const void* x, void* A, int NB, int h, int w, int C, iggt_stream_t stream) {
  if (NB <= 0 || (C % 8)) return -1;
  const int ho = (h - 1) / 2 + 1, wo = (w - 1) / 2 + 1;
  const int64_t total = static_cast<int64_t>(NB) * ho * wo * 9 * (C / 8);
  im2col_s2_kernel<<<grid_for(total), 256, 0, (cudaStream_t)stream>>>((const uint4*)x, (uint4*)A, NB, h, w, C, ho, wo);
  return (int)cudaGetLastError();
}

extern "C" int iggt_dpt_tail(const void* x, const float* w, const float* b, float* out_main, float* out_conf,
                             int NB, int H, int W, int OC, int mode, int dtype, iggt_stream_t stream) {
  if (NB <= 0 || (OC != 2 && OC != 4 && OC != 8)) return -1;
  if (mode != 2 && !out_conf) return -1;
  const int64_t hw = static_cast<int64_t>(H) * W, npix = hw * NB;
  cudaStream_t s = (cudaStream_t)stream;
#define TAIL(BF, O) dpt_tail_kernel<BF, O><<<grid_for(npix), 256, 0, s>>>((const uint16_t*)x, w, b, out_main, out_conf, npix, hw, mode)
  if (dtype) { if (OC == 2) TAIL(true, 2); else if (OC == 4) TAIL(true, 4); else TAIL(true, 8); }
  else { if (OC == 2) TAIL(false, 2); else if (OC == 4) TAIL(false, 4); else TAIL(false, 8); }
#undef TAIL
  return (int)cudaGetLastError();
}

extern "C" int iggt_skinny_gemm(const float* x, int64_t ldx, const void* W, int64_t ldw, const float* bias,
                                const float* gamma, const float* resid, int64_t ldr, float* out, int64_t ldo,
                                int M, int N, int K, int act, int dtype, iggt_stream_t stream) {
  if (M <= 0 || M > 32 || N <= 0 || K <= 0 || (K % 8) || (ldx % 4) || (ldw % 8)) return -1;
  const unsigned grid = (N + SK_COLS - 1) / SK_COLS;
  cudaStream_t s = (cudaStream_t)stream;
  static DeviceOnce once;
  if (once.first()) {
    cudaFuncSetAttribute(skinny_gemm_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, SK_SMEM);
    cudaFuncSetAttribute(skinny_gemm_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, SK_SMEM);
  }
  CUtensorMap tW;
  {
    uint64_t dims[2] = {(uint64_t)K, (uint64_t)N};
    uint64_t str[1] = {(uint64_t)ldw * 2};
    uint32_t box[2] = {SK_KC, SK_COLS};
    if (make_tmap(&tW, dtype ? TM_BF16 : TM_F16, 2, W, dims, str, box, false)) return -4;
  }
  for (int m0 = 0; m0 < M; m0 += 8) {   // weights of the later chunks come from L2
    const int mm = M - m0 < 8 ? M - m0 : 8;
    const float* rp = resid ? resid + m0 * ldr : nullptr;
    CUtensorMap tX;
    uint64_t dims[2] = {(uint64_t)K, (uint64_t)mm};
    uint64_t str[1] = {(uint64_t)ldx * 4};
    uint32_t box[2] = {SK_KC, 8};
    if (make_tmap(&tX, TM_F32, 2, x + m0 * ldx, dims, str, box, false)) return -4;
    float* op = out + m0 * ldo;
    if (dtype) launch_pdl(skinny_gemm_kernel<true>, dim3(grid), dim3(288), SK_SMEM, s, tW, tX, bias, gamma, rp, ldr, op, ldo, mm, N, K, act);
    else launch_pdl(skinny_gemm_kernel<false>, dim3(grid), dim3(288), SK_SMEM, s, tW, tX, bias, gamma, rp, ldr, op, ldo, mm, N, K, act);
  }
  return (int)cudaGetLastError();
}

extern "C" int iggt_small_attention(const float* qkv, float* out, int B, int N, int H, int d, float scale,
                                    iggt_stream_t stream) {
  if (B <= 0 || N <= 0 || N > 256 || H <= 0 || d <= 0) return -1;
  const size_t smem = (2 * static_cast<size_t>(N) * d + 4 * N) * sizeof(float);
  if (smem > 200 * 1024) return -1;
  static DeviceOnce once;
  if (once.first()) {
    cudaFuncSetAttribute(small_attention_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
  }
  small_attention_kernel<<<B * H, 128, smem, (cudaStream_t)stream>>>(qkv, out, N, H, d, scale);
  return (int)cudaGetLastError();
}
