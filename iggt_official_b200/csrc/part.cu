// Kernels of the part (instance-feature) path that are not GEMM-shaped enough for the wgmma main loop:
// small-C LayerNorm on 16-bit NHWC rows, the k4/s2/p1 ConvTranspose gather, the two 8x8-window attentions
// (OCAB with 12x12 overlapping keys + relative-position bias and the reference's scrambled query windows;
// HAB plain window self-attention; the tensor-core kernels are in winattn.cuh), and the CAB channel-attention
// (squeeze-excite) pieces.
// Reference: iggt/heads/adaptor.py:140-226, iggt/heads/part_head.py:148-243, iggt/heads/window_sa.py.
#include "ptx.cuh"
#include "launch.cuh"
#include "winattn.cuh"
#include "../../include/iggt_b200.h"

namespace iggt {

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
  const float mean = warp_sum(s) / C;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < PER; ++i) { const float d = v[i] - mean; q += d * d; }
  const float rstd = rsqrtf(warp_sum(q) / C + eps);
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
    *reinterpret_cast<uint4*>(out + ((static_cast<int64_t>(n) * H + oy) * W + ox) * C + c8 * 8) = pack8<BF16>(acc);
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
    *reinterpret_cast<uint4*>(y + off) = pack8<BF16>(o);
  }
}

}  // namespace iggt

using namespace iggt;

extern "C" int iggt_layernorm16(const void* x, void* y, int64_t rows, int C, const float* w, const float* b,
                                float eps, int dtype, iggt_stream_t stream) {
  return dispatch_dtype(dtype, [&](auto bf16) {
    if (rows <= 0) return 0;
    if (!w || !b) return -1;
    const unsigned grid = static_cast<unsigned>((rows + 7) / 8);
    cudaStream_t s = (cudaStream_t)stream;
#define L16(CC) layernorm16_kernel<bf16, CC><<<grid, 256, 0, s>>>((const uint16_t*)x, (uint16_t*)y, w, b, eps, rows)
    if (C == 256) L16(256);
    else if (C == 128) L16(128);
    else if (C == 64) L16(64);
    else return -1;
#undef L16
    return (int)cudaGetLastError();
  });
}

extern "C" int iggt_col2im_k4s2p1(const void* Y, const float* bias, void* out, int NB, int h, int w, int C,
                                  int dtype, iggt_stream_t stream) {
  return dispatch_dtype(dtype, [&](auto bf16) {
    if (NB <= 0 || (C % 8) || !bias) return -1;
    const int64_t total = static_cast<int64_t>(NB) * 4 * h * w * (C / 8);
    col2im_k4s2p1_kernel<bf16><<<grid_stride_blocks(total), 256, 0, (cudaStream_t)stream>>>(
        (const uint16_t*)Y, bias, (uint16_t*)out, NB, h, w, C);
    return (int)cudaGetLastError();
  });
}

extern "C" int iggt_ocab_attention(const void* q, const void* k, const void* v, const float* table, const int* rpi,
                                   void* out, int NB, int h, int w, int dtype, iggt_stream_t stream) {
  return dispatch_dtype(dtype, [&](auto bf16) {
    if (NB <= 0 || (h % 8) || (w % 8)) return -1;
    const cudaError_t e = opt_in_smem<ocab_attention_tc_kernel<bf16>>(OA_SMEM);
    if (e != cudaSuccess) return (int)e;
    const unsigned grid = static_cast<unsigned>(NB) * (h / 8) * (w / 8) * 4;
    ocab_attention_tc_kernel<bf16><<<grid, 128, OA_SMEM, (cudaStream_t)stream>>>(
        (const uint16_t*)q, (const uint16_t*)k, (const uint16_t*)v, table, rpi, (uint16_t*)out, h, w);
    return (int)cudaGetLastError();
  });
}

extern "C" int iggt_window_attention(const void* qkv, void* out, int NB, int h, int w, int dtype,
                                     iggt_stream_t stream) {
  return dispatch_dtype(dtype, [&](auto bf16) {
    if (NB <= 0 || (h % 8) || (w % 8)) return -1;
    const unsigned grid = static_cast<unsigned>(NB) * (h / 8) * (w / 8) * 4;
    window_attention_tc_kernel<bf16><<<grid, 128, 0, (cudaStream_t)stream>>>((const uint16_t*)qkv, (uint16_t*)out, h, w);
    return (int)cudaGetLastError();
  });
}

extern "C" int iggt_channel_mean(const void* x, float* mean, int NB, int64_t hw, int C, int dtype,
                                 iggt_stream_t stream) {
  return dispatch_dtype(dtype, [&](auto bf16) {
    if (NB <= 0 || C <= 0 || C > 256 || (256 % C)) return -1;
    cudaError_t e = cudaMemsetAsync(mean, 0, sizeof(float) * NB * C, (cudaStream_t)stream);
    if (e != cudaSuccess) return (int)e;
    dim3 grid(static_cast<unsigned>(hw / 64 > 0 ? (hw / 64 < 296 ? hw / 64 : 296) : 1), NB);
    channel_mean_kernel<bf16><<<grid, 256, 0, (cudaStream_t)stream>>>((const uint16_t*)x, mean, hw, C, 1.0f / hw);
    return (int)cudaGetLastError();
  });
}

extern "C" int iggt_se_scale_add(const void* y0, const void* cx, const float* mean, const float* w1, const float* b1,
                                 const float* w2, const float* b2, void* y, int NB, int64_t hw, int C, int R,
                                 float alpha, int dtype, iggt_stream_t stream) {
  return dispatch_dtype(dtype, [&](auto bf16) {
    if (NB <= 0 || C > 256 || (C % 8) || R > 16) return -1;
    dim3 grid(grid_stride_blocks(hw * (C / 8)) / 2 + 1, NB);
    se_scale_add_kernel<bf16><<<grid, 256, 0, (cudaStream_t)stream>>>(
        (const uint16_t*)y0, (const uint16_t*)cx, mean, w1, b1, w2, b2, (uint16_t*)y, hw, C, R, alpha);
    return (int)cudaGetLastError();
  });
}
