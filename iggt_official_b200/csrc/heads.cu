// HBM-bound kernels of the dense heads and the camera head (all NHWC 16-bit activations unless noted):
// bilinear(align_corners) upsample fused with the UV sinusoid pos-embed, deconv pixel-shuffle, stride-2
// im2col, the per-pixel 1x1 + activation tail, a skinny (M <= 32) weight-streaming GEMM and a tiny
// attention for the S camera tokens.  Coalesced 16-byte accesses, grid-stride loops.
#include "ptx.cuh"
#include "tmap.cuh"
#include "launch.cuh"
#include "../../include/iggt_b200.h"

namespace iggt {

// F.interpolate(mode="bilinear", align_corners=True) on NHWC (iggt/heads/dpt_head.py:251-256,478,484-509)
// + optional pos-embed: channels [0,C/2) get tabx[x][c], [C/2,C) get taby[y][c-C/2]
// (iggt/heads/dpt_head.py:274-284, iggt/heads/utils.py:11-108; tables are built on the host in float64).
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
    for (int m = 0; m < 8; ++m) acc[c][m] = warp_sum(acc[c][m]);
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
    sum = warp_sum(sum);
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

// softmax(q k^T / sqrt(d)) v over any number of keys (camera tokens of scenes with more views than small_attention's
// shared memory holds), fp32 on the CUDA cores.  Same layout as small_attention.  One CTA per (b, head, block of TA_QB
// query rows); the keys and values of the scene go through shared memory in tiles of TA_KT rows, in key order, so the
// shared memory is a constant independent of N.  Warp w owns query rows 4w..4w+3 of the block; lane l scores keys l and
// l + 32 of the tile (a sequential fmaf chain over d, then * scale, as small_attention) and owns output columns
// l + 32 i.  Online softmax per row: a running max m and sum l; when a tile raises the max, acc and l are rescaled by
// expf(m_old - m_new) (a factor of exactly 1 otherwise), p = expf(s - m_new), the tile's p are summed by the lanes
// (p0 + p1, then a butterfly) and added to l, and acc takes the tile's keys in key order with fmaf.  out = acc * (1/l).
// No atomics, a fixed tile order: repeated calls are bit-identical.
constexpr int TA_KT = 64;          // keys per tile
constexpr int TA_QB = 16;          // query rows per CTA (4 warps x 4 rows)
constexpr int TA_DMAX = 128;
constexpr int TA_LD_MAX = TA_DMAX + 4;   // row pitch d + 4: lanes reading float4s of 8 consecutive rows hit distinct banks
constexpr int TA_SMEM = (2 * TA_KT + TA_QB) * TA_LD_MAX * static_cast<int>(sizeof(float));   // 76032 B
template <int NC>                  // NC = d / 32 output columns per lane
__global__ void __launch_bounds__(128, 2)
token_attention_kernel(const float* __restrict__ qkv, float* __restrict__ out, int N, int H, float scale) {
  constexpr int d = NC * 32, ld = d + 4;
  extern __shared__ __align__(16) float ta_smem[];
  float* sk = ta_smem;                      // [TA_KT][ld]
  float* sv = sk + TA_KT * ld;              // [TA_KT][ld]
  float* sq = sv + TA_KT * ld;              // [TA_QB][ld]
  const int b = blockIdx.x / H, hh = blockIdx.x % H;
  const int q0 = blockIdx.y * TA_QB;
  const int64_t C = static_cast<int64_t>(H) * d;
  const float* base = qkv + static_cast<int64_t>(b) * N * 3 * C + hh * d;     // q of row 0 of scene b, head hh
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  constexpr int V4 = d / 4;                 // float4 per row
  for (int i = threadIdx.x; i < TA_QB * V4; i += blockDim.x) {
    const int r = i / V4, c4 = i - r * V4;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (q0 + r < N) v = __ldg(reinterpret_cast<const float4*>(base + static_cast<int64_t>(q0 + r) * 3 * C) + c4);
    *reinterpret_cast<float4*>(sq + r * ld + c4 * 4) = v;
  }
  float m[4], l[4], acc[4][NC];
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    m[r] = -INFINITY; l[r] = 0.f;
#pragma unroll
    for (int i = 0; i < NC; ++i) acc[r][i] = 0.f;
  }
  const int rows = min(4, max(0, N - q0 - warp * 4));          // valid query rows of this warp
  for (int t0 = 0; t0 < N; t0 += TA_KT) {
    const int nk = min(TA_KT, N - t0);
    __syncthreads();                        // the previous tile is consumed (and the q rows are stored)
    for (int i = threadIdx.x; i < TA_KT * V4; i += blockDim.x) {
      const int r = i / V4, c4 = i - r * V4;
      float4 kv = make_float4(0.f, 0.f, 0.f, 0.f), vv = kv;
      if (r < nk) {
        const float* row = base + static_cast<int64_t>(t0 + r) * 3 * C;
        kv = __ldg(reinterpret_cast<const float4*>(row + C) + c4);
        vv = __ldg(reinterpret_cast<const float4*>(row + 2 * C) + c4);
      }
      *reinterpret_cast<float4*>(sk + r * ld + c4 * 4) = kv;
      *reinterpret_cast<float4*>(sv + r * ld + c4 * 4) = vv;
    }
    __syncthreads();
    if (rows == 0) continue;
    float s[4][2];
#pragma unroll
    for (int r = 0; r < 4; ++r) s[r][0] = s[r][1] = 0.f;
    const float* k0 = sk + lane * ld;
    const float* k1 = sk + (lane + 32) * ld;
    const float* qw = sq + warp * 4 * ld;
#pragma unroll 4
    for (int c = 0; c < d; c += 4) {
      const float4 a = *reinterpret_cast<const float4*>(k0 + c);
      const float4 e = *reinterpret_cast<const float4*>(k1 + c);
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const float4 q = *reinterpret_cast<const float4*>(qw + r * ld + c);
        s[r][0] = fmaf(q.x, a.x, s[r][0]); s[r][0] = fmaf(q.y, a.y, s[r][0]);
        s[r][0] = fmaf(q.z, a.z, s[r][0]); s[r][0] = fmaf(q.w, a.w, s[r][0]);
        s[r][1] = fmaf(q.x, e.x, s[r][1]); s[r][1] = fmaf(q.y, e.y, s[r][1]);
        s[r][1] = fmaf(q.z, e.z, s[r][1]); s[r][1] = fmaf(q.w, e.w, s[r][1]);
      }
    }
    float p[4][2];
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const float s0 = lane < nk ? s[r][0] * scale : -INFINITY;
      const float s1 = lane + 32 < nk ? s[r][1] * scale : -INFINITY;
      float mt = fmaxf(s0, s1);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) mt = fmaxf(mt, __shfl_xor_sync(0xffffffffu, mt, o));
      const float mn = fmaxf(m[r], mt);
      const float alpha = expf(m[r] - mn);  // 0 at the first tile (m = -inf), 1 when the max did not grow
      m[r] = mn;
      p[r][0] = expf(s0 - mn);
      p[r][1] = expf(s1 - mn);
      l[r] = __fmaf_rn(l[r], alpha, warp_sum(p[r][0] + p[r][1]));
#pragma unroll
      for (int i = 0; i < NC; ++i) acc[r][i] *= alpha;
    }
    for (int j = 0; j < nk; ++j) {
      float vj[NC];
#pragma unroll
      for (int i = 0; i < NC; ++i) vj[i] = sv[j * ld + lane + 32 * i];
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const float pj = __shfl_sync(0xffffffffu, j < 32 ? p[r][0] : p[r][1], j & 31);
#pragma unroll
        for (int i = 0; i < NC; ++i) acc[r][i] = fmaf(pj, vj[i], acc[r][i]);
      }
    }
  }
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    if (r >= rows) break;
    const float inv = 1.0f / l[r];
    float* o = out + (static_cast<int64_t>(b) * N + q0 + warp * 4 + r) * C + hh * d;
#pragma unroll
    for (int i = 0; i < NC; ++i) o[lane + 32 * i] = acc[r][i] * inv;
  }
}

}  // namespace iggt

using namespace iggt;

extern "C" int iggt_upsample_bilinear_nhwc(const void* x, void* out, int NB, int h, int w, int H, int W, int C,
                                           const float* tabx, const float* taby, int dtype, iggt_stream_t stream) {
  return dispatch_dtype(dtype, [&](auto bf16) {
    if (NB <= 0 || h <= 0 || w <= 0 || H <= 0 || W <= 0 || (C % 16)) return -1;
    if ((tabx == nullptr) != (taby == nullptr)) return -1;
    if (static_cast<int64_t>(NB) * H > 0x7fffffff || static_cast<int64_t>(w) * C > 0x7fffffff) return -1;
    const unsigned rows = static_cast<unsigned>(NB) * H;                 // one CTA per output row
    upsample_bilinear_kernel<bf16><<<rows, 256, 0, (cudaStream_t)stream>>>((const uint16_t*)x, (uint16_t*)out, NB, h, w,
                                                                           H, W, C, tabx, taby);
    return (int)cudaGetLastError();
  });
}

extern "C" int iggt_deconv_shuffle(const void* y, void* out, int NB, int h, int w, int C, int k, iggt_stream_t stream) {
  if (NB <= 0 || (C % 8) || k <= 0) return -1;
  const int64_t total = static_cast<int64_t>(NB) * h * w * k * k * (C / 8);
  deconv_shuffle_kernel<<<grid_stride_blocks(total), 256, 0, (cudaStream_t)stream>>>((const uint4*)y, (uint4*)out, NB, h, w, C, k);
  return (int)cudaGetLastError();
}

extern "C" int iggt_im2col3x3_s2(const void* x, void* A, int NB, int h, int w, int C, iggt_stream_t stream) {
  if (NB <= 0 || (C % 8)) return -1;
  const int ho = (h - 1) / 2 + 1, wo = (w - 1) / 2 + 1;
  const int64_t total = static_cast<int64_t>(NB) * ho * wo * 9 * (C / 8);
  im2col_s2_kernel<<<grid_stride_blocks(total), 256, 0, (cudaStream_t)stream>>>((const uint4*)x, (uint4*)A, NB, h, w, C, ho, wo);
  return (int)cudaGetLastError();
}

extern "C" int iggt_skinny_gemm(const float* x, int64_t ldx, const void* W, int64_t ldw, const float* bias,
                                const float* gamma, const float* resid, int64_t ldr, float* out, int64_t ldo,
                                int M, int N, int K, int act, int dtype, iggt_stream_t stream) {
  return dispatch_dtype(dtype, [&](auto bf16) {
    if (M <= 0 || M > 32 || N <= 0 || K <= 0 || (K % 8) || (ldx % 4) || (ldw % 8)) return -1;
    const unsigned grid = (N + SK_COLS - 1) / SK_COLS;
    cudaStream_t s = (cudaStream_t)stream;
    const cudaError_t e = opt_in_smem<skinny_gemm_kernel<bf16>>(SK_SMEM);
    if (e != cudaSuccess) return (int)e;
    CUtensorMap tW;
    {
      uint64_t dims[2] = {(uint64_t)K, (uint64_t)N};
      uint64_t str[1] = {(uint64_t)ldw * 2};
      uint32_t box[2] = {SK_KC, SK_COLS};
      if (make_tmap(&tW, tm16(bf16), 2, W, dims, str, box, false)) return -4;
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
      launch_pdl(skinny_gemm_kernel<bf16>, dim3(grid), dim3(288), SK_SMEM, s, tW, tX, bias, gamma, rp, ldr, op, ldo, mm, N,
                 K, act);
    }
    return (int)cudaGetLastError();
  });
}

extern "C" int iggt_small_attention(const float* qkv, float* out, int B, int N, int H, int d, float scale,
                                    iggt_stream_t stream) {
  if (B <= 0 || N <= 0 || N > 256 || H <= 0 || d <= 0) return -1;
  const size_t smem = (2 * static_cast<size_t>(N) * d + 4 * N) * sizeof(float);
  if (smem > 200 * 1024) return -1;
  const cudaError_t e = opt_in_smem<small_attention_kernel>(200 * 1024);
  if (e != cudaSuccess) return (int)e;
  small_attention_kernel<<<B * H, 128, smem, (cudaStream_t)stream>>>(qkv, out, N, H, d, scale);
  return (int)cudaGetLastError();
}

extern "C" int iggt_token_attention(const float* qkv, float* out, int B, int N, int H, int d, float scale,
                                    iggt_stream_t stream) {
  if (B <= 0 || N <= 0 || H <= 0 || d <= 0 || d > TA_DMAX || (d % 32)) return -1;
  const int64_t qblocks = (static_cast<int64_t>(N) + TA_QB - 1) / TA_QB;
  if (qblocks > 65535 || static_cast<int64_t>(B) * H > 0x7fffffff) return -1;
  // the largest element index, (B*N) * (3*H*d), must fit int64: check in steps that cannot overflow themselves
  const int64_t rows = static_cast<int64_t>(B) * N, width = 3 * static_cast<int64_t>(H) * d;
  if (rows > INT64_MAX / width) return -1;
  if (reinterpret_cast<uintptr_t>(qkv) % 16) return -1;           // float4 loads of the q, k and v rows
  void (*kern)(const float*, float*, int, int, float);
  switch (d / 32) {
    case 1: kern = token_attention_kernel<1>; break;
    case 2: kern = token_attention_kernel<2>; break;
    case 3: kern = token_attention_kernel<3>; break;
    default: kern = token_attention_kernel<4>; break;
  }
  const cudaError_t e = opt_in_smem<token_attention_kernel<1>, token_attention_kernel<2>, token_attention_kernel<3>,
                                    token_attention_kernel<4>>(TA_SMEM);
  if (e != cudaSuccess) return (int)e;
  const dim3 grid(static_cast<unsigned>(B * H), static_cast<unsigned>(qblocks));
  kern<<<grid, 128, TA_SMEM, (cudaStream_t)stream>>>(qkv, out, N, H, scale);
  return (int)cudaGetLastError();
}
