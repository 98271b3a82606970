// HBM-bound kernels of the trunk: LayerNorm (fp32 in, 16-bit or fp32 out, optional row remap),
// patch im2col with ImageNet normalisation, DINOv2 / aggregator token assembly.
// All are one-pass, vectorised (16 B per lane), warp-shuffle reductions only.
#include "ptx.cuh"
#include "launch.cuh"
#include "../../include/iggt_b200.h"

namespace iggt {

// One warp per row. Row r_out = g*rows_out + i  <-  r_in = g*rows_in + in_off + i  (i < rows_out).
// VEC = C / 128 float4 per lane.
template <int VEC, bool OUT32, bool BF16>
__global__ void __launch_bounds__(256)
layernorm_kernel(const float* __restrict__ x, int64_t ldx, void* __restrict__ y, int64_t ldy,
                 const float* __restrict__ w, const float* __restrict__ b, float eps, int64_t n_rows_out,
                 int rows_out, int rows_in, int in_off, int out_rows_per_group, int out_off) {
  griddep_wait();
  griddep_launch();
  const int64_t r = static_cast<int64_t>(blockIdx.x) * 8 + (threadIdx.x >> 5);
  if (r >= n_rows_out) return;
  const int lane = threadIdx.x & 31;
  const int64_t g = r / rows_out, i = r % rows_out;
  const float* xr = x + (g * rows_in + in_off + i) * ldx;
  const int64_t ro = g * out_rows_per_group + out_off + i;
  float4 v[VEC];
  float s = 0.f;
#pragma unroll
  for (int k = 0; k < VEC; ++k) {
    v[k] = __ldg(reinterpret_cast<const float4*>(xr) + lane + 32 * k);
    s += v[k].x + v[k].y + v[k].z + v[k].w;
  }
  constexpr float invC = 1.0f / (VEC * 128);
  const float mean = warp_sum(s) * invC;
  float q = 0.f;
#pragma unroll
  for (int k = 0; k < VEC; ++k) {
    const float a = v[k].x - mean, bq = v[k].y - mean, c = v[k].z - mean, d = v[k].w - mean;
    q += a * a + bq * bq + c * c + d * d;
  }
  const float rstd = rsqrtf(warp_sum(q) * invC + eps);
#pragma unroll
  for (int k = 0; k < VEC; ++k) {
    const int col = (lane + 32 * k) * 4;
    float4 o;
    o.x = (v[k].x - mean) * rstd; o.y = (v[k].y - mean) * rstd;
    o.z = (v[k].z - mean) * rstd; o.w = (v[k].w - mean) * rstd;
    if (w) {
      const float4 ww = __ldg(reinterpret_cast<const float4*>(w + col));
      o.x *= ww.x; o.y *= ww.y; o.z *= ww.z; o.w *= ww.w;
    }
    if (b) {
      const float4 bb = __ldg(reinterpret_cast<const float4*>(b + col));
      o.x += bb.x; o.y += bb.y; o.z += bb.z; o.w += bb.w;
    }
    if constexpr (OUT32) {
      *reinterpret_cast<float4*>(reinterpret_cast<float*>(y) + ro * ldy + col) = o;
    } else {
      uint2 u;
      u.x = pack16x2<BF16>(o.x, o.y);
      u.y = pack16x2<BF16>(o.z, o.w);
      *reinterpret_cast<uint2*>(reinterpret_cast<uint16_t*>(y) + ro * ldy + col) = u;
    }
  }
}

// images [NI,3,H,W] fp32 in [0,1]  ->  A[NI*gh*gw, KP] 16-bit, k = c*196 + ky*14 + kx, zero padded
// to KP; fuses (x - mean) / std  (iggt/models/aggregator.py:206, iggt/layers/patch_embed.py:75-77).
template <bool BF16>
__global__ void __launch_bounds__(256)
patchify_kernel(const float* __restrict__ img, uint16_t* __restrict__ A, int NI, int H, int W, int gh,
                int gw, int KP) {
  const int64_t patch = blockIdx.x;  // one CTA per patch
  const int n = patch / (gh * gw);
  const int pr = (patch % (gh * gw)) / gw, pc = patch % gw;
  const float mean[3] = {0.485f, 0.456f, 0.406f};
  const float stdv[3] = {0.229f, 0.224f, 0.225f};
  for (int k = threadIdx.x; k < KP; k += blockDim.x) {
    float val = 0.f;
    if (k < 588) {
      const int c = k / 196, ky = (k % 196) / 14, kx = k % 14;
      const float px = __ldg(img + ((static_cast<int64_t>(n) * 3 + c) * H + pr * 14 + ky) * W + pc * 14 + kx);
      val = (px - mean[c]) / stdv[c];
    }
    A[patch * KP + k] = st16<BF16>(val);
  }
}

// DINOv2 token assembly (iggt/layers/vision_transformer.py:217-236):
//   x[n,0] = cls + pos[0];  x[n,1..R] = reg;  x[n,1+R+p] = float(pe16[n,p]) + pos[1+p]
template <bool BF16>
__global__ void __launch_bounds__(256)
dino_assemble_kernel(const uint16_t* __restrict__ pe, const float* __restrict__ cls,
                     const float* __restrict__ reg, const float* __restrict__ pos, float* __restrict__ x,
                     int P, int R, int C) {
  const int64_t row = blockIdx.x;  // n*(1+R+P) + t
  const int T = 1 + R + P;
  const int n = row / T, t = row % T;
  for (int c = threadIdx.x * 4; c < C; c += blockDim.x * 4) {
    float4 o;
    if (t == 0) {
      const float4 a = __ldg(reinterpret_cast<const float4*>(cls + c));
      const float4 b = __ldg(reinterpret_cast<const float4*>(pos + c));
      o = make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w);
    } else if (t <= R) {
      o = __ldg(reinterpret_cast<const float4*>(reg + static_cast<int64_t>(t - 1) * C + c));
    } else {
      const int pidx = t - 1 - R;
      const uint2 u = __ldg(reinterpret_cast<const uint2*>(pe + (static_cast<int64_t>(n) * P + pidx) * C + c));
      const float4 b = __ldg(reinterpret_cast<const float4*>(pos + static_cast<int64_t>(1 + pidx) * C + c));
      const float2 f01 = cvt16x2<BF16>(u.x), f23 = cvt16x2<BF16>(u.y);
      o = make_float4(f01.x + b.x, f01.y + b.y, f23.x + b.z, f23.y + b.w);
    }
    *reinterpret_cast<float4*>(x + row * C + c) = o;
  }
}

// Aggregator special tokens (iggt/models/aggregator.py:230-234,338-361): rows [n*T, n*T+ns) of x get
// the camera token and the 4 register tokens; variant 0 for the first view of a scene, 1 otherwise
// (local view n is view  view_offset + n % S_loc  of its scene, so a view-sharded rank indexes correctly).
__global__ void __launch_bounds__(256)
special_tokens_kernel(const float* __restrict__ cam, const float* __restrict__ reg, float* __restrict__ x,
                      int T, int R, int C, int S_loc, int view_offset) {
  const int n = blockIdx.x / (1 + R), t = blockIdx.x % (1 + R);
  const int s_global = view_offset + (n % S_loc);  // view index inside its scene
  const int variant = (s_global == 0) ? 0 : 1;
  const float* src = (t == 0) ? cam + static_cast<int64_t>(variant) * C
                              : reg + (static_cast<int64_t>(variant) * R + (t - 1)) * C;
  for (int c = threadIdx.x * 4; c < C; c += blockDim.x * 4)
    *reinterpret_cast<float4*>(x + (static_cast<int64_t>(n) * T + t) * C + c) =
        __ldg(reinterpret_cast<const float4*>(src + c));
}

}  // namespace iggt

using namespace iggt;

extern "C" int iggt_layernorm(const float* x, int64_t ldx, void* y, int64_t ldy, int C, const float* w,
                              const float* b, float eps, int64_t groups, int rows_out, int rows_in,
                              int in_off, int out_rows_per_group, int out_off, int out_kind,
                              iggt_stream_t stream) {
  if (out_kind < 0 || out_kind > 2) return -3;
  if (C != 1024 && C != 2048) return -1;
  if ((ldx % 4) || (ldy % 4)) return -2;
  if (groups <= 0 || rows_out <= 0) return 0;
  const int64_t n = groups * rows_out;
  const unsigned grid = static_cast<unsigned>((n + 7) / 8);
  cudaStream_t s = (cudaStream_t)stream;
#define LN_LAUNCH(VEC, O32, BF)                                                                        \
  launch_pdl(layernorm_kernel<VEC, O32, BF>, dim3(grid), dim3(256), 0, s, x, ldx, y, ldy, w, b, eps, n, rows_out, rows_in, \
             in_off, out_rows_per_group, out_off)
  if (C == 1024) {
    if (out_kind == 2) LN_LAUNCH(8, true, false);
    else if (out_kind == 1) LN_LAUNCH(8, false, true);
    else LN_LAUNCH(8, false, false);
  } else {
    if (out_kind == 2) LN_LAUNCH(16, true, false);
    else if (out_kind == 1) LN_LAUNCH(16, false, true);
    else LN_LAUNCH(16, false, false);
  }
#undef LN_LAUNCH
  return (int)cudaGetLastError();
}

extern "C" int iggt_patchify(const float* images, void* A, int NI, int H, int W, int KP, int dtype,
                             iggt_stream_t stream) {
  return dispatch_dtype(dtype, [&](auto bf16) {
    if (NI <= 0 || (H % 14) || (W % 14) || KP < 588 || (KP % 8)) return -1;
    const int gh = H / 14, gw = W / 14;
    const unsigned grid = static_cast<unsigned>(NI) * gh * gw;
    patchify_kernel<bf16><<<grid, 256, 0, (cudaStream_t)stream>>>(images, (uint16_t*)A, NI, H, W, gh, gw, KP);
    return (int)cudaGetLastError();
  });
}

extern "C" int iggt_dino_assemble(const void* pe16, const float* cls, const float* reg, const float* pos,
                                  float* x, int NI, int P, int R, int C, int dtype, iggt_stream_t stream) {
  return dispatch_dtype(dtype, [&](auto bf16) {
    if (NI <= 0 || P <= 0 || (C % 4)) return -1;
    const unsigned grid = static_cast<unsigned>(NI) * (1 + R + P);
    dino_assemble_kernel<bf16><<<grid, 256, 0, (cudaStream_t)stream>>>((const uint16_t*)pe16, cls, reg, pos, x, P, R, C);
    return (int)cudaGetLastError();
  });
}

extern "C" int iggt_special_tokens(const float* cam, const float* reg, float* x, int NI, int T, int R,
                                   int C, int S_loc, int view_offset, iggt_stream_t stream) {
  if (NI <= 0 || S_loc <= 0 || (C % 4)) return -1;
  special_tokens_kernel<<<NI * (1 + R), 256, 0, (cudaStream_t)stream>>>(cam, reg, x, T, R, C, S_loc,
                                                                        view_offset);
  return (int)cudaGetLastError();
}
