// Point-cloud export on the device (demo.py:618-657 export_glb_visualizations -> visual_util.py:38-238
// predictions_to_glb, which masks, compacts and takes percentiles in numpy on the host).
//
// One call of the public function (iggt_official_b200/visual_util.py) runs:
//   1. iggt_select over the confidences -> the threshold, left on the device (skipped for conf_thres == 0);
//   2. iggt_pointcloud_select: one pass over the points that reads the threshold through a device pointer, evaluates
//      the confidence and background masks, converts the colour source to RGBA bytes and writes the mask, the colours,
//      the three coordinate planes [3, n] and the kept count of every tile of 1024 points;
//   3. iggt_select over the three planes with the mask shared by the rows (ldm = 0) -> the 5 % / 95 % percentiles;
//   4. iggt_pointcloud_compact: an exclusive scan of the tile counts (one CTA), then one CTA per tile writes the kept
//      points in pixel order into the GLB's point section (xyz fp32 [m, 3], then RGBA [m, 4]) and the per-axis
//      min / max.
// Every output position is a function of the mask alone and min / max are exact, so repeated calls give identical
// bytes.  Indices are 32-bit: n < 2^32, as iggt_select requires.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "../../include/iggt_b200.h"

namespace iggt {

constexpr int PC_THREADS = 256;
constexpr int PC_PER = 4;                         // points per thread per tile
constexpr int PC_TILE = PC_THREADS * PC_PER;      // points per tile (= per CTA)
constexpr int PC_WARPS = PC_THREADS / 32;
constexpr int PC_SCAN_THREADS = 1024;

struct PcColor {                                  // element (point i, channel c) at (i / hw) * sf + c * sc + (i % hw) * sp
  const void* p;
  int u8;
  uint32_t hw;
  int64_t sf, sc, sp;
};

// (c * 255).astype(uint8): fp32 sources round the product in fp32 and truncate it (cvt.rzi, then the low byte, as
// the x86 cast does for values in int32 range); uint8 sources wrap mod 256, so c becomes (256 - c) mod 256.
__device__ __forceinline__ uint32_t pc_channel(const PcColor& c, int64_t off) {
  if (c.u8) return (256u - __ldg(static_cast<const uint8_t*>(c.p) + off)) & 0xffu;
  const float v = __fmul_rn(__ldg(static_cast<const float*>(c.p) + off), 255.f);
  return static_cast<uint32_t>(__float2int_rz(v)) & 0xffu;
}

__device__ __forceinline__ uint32_t pc_rgba(const PcColor& c, uint32_t i) {
  const uint32_t s = i / c.hw, pix = i - s * c.hw;
  const int64_t base = static_cast<int64_t>(s) * c.sf + static_cast<int64_t>(pix) * c.sp;
  return pc_channel(c, base) | pc_channel(c, base + c.sc) << 8 | pc_channel(c, base + 2 * c.sc) << 16 | 0xff000000u;
}

__global__ void __launch_bounds__(PC_THREADS)
pc_select_kernel(const float* __restrict__ pts, const float* __restrict__ conf, uint32_t n, const float* __restrict__ thr,
                 PcColor col, int bg, uint8_t* __restrict__ mask, float* __restrict__ planes, int64_t ldp,
                 uint32_t* __restrict__ rgba, uint32_t* __restrict__ tile_count) {
  const float th = thr ? __ldg(thr) : 0.f;
  const float eps = static_cast<float>(1e-5);   // numpy 2 compares float32 data with the Python float 1e-5 in fp32
  const uint32_t t0 = blockIdx.x * PC_TILE;
  int kept = 0;
#pragma unroll
  for (int k = 0; k < PC_PER; ++k) {
    const uint32_t i = t0 + k * PC_THREADS + threadIdx.x;
    bool keep = false;
    if (i < n) {
      const float c = __ldg(conf + i);
      keep = c >= th && c > eps;                 // a NaN confidence or threshold keeps nothing
      const uint32_t rgb = pc_rgba(col, i);
      const uint32_t r = rgb & 0xffu, g = (rgb >> 8) & 0xffu, b = (rgb >> 16) & 0xffu;
      if (bg & IGGT_PC_MASK_BLACK) keep = keep && r + g + b >= 16u;
      if (bg & IGGT_PC_MASK_WHITE) keep = keep && !(r > 240u && g > 240u && b > 240u);
      mask[i] = keep ? 1 : 0;
      rgba[i] = rgb;
#pragma unroll
      for (int j = 0; j < 3; ++j) planes[j * ldp + i] = __ldg(pts + 3 * static_cast<int64_t>(i) + j);
    }
    kept += __syncthreads_count(keep);
  }
  if (threadIdx.x == 0) tile_count[blockIdx.x] = static_cast<uint32_t>(kept);
}

// One CTA: exclusive prefix of the tile counts, the total, and the min / max slots set to +inf / -inf.
__global__ void __launch_bounds__(PC_SCAN_THREADS)
pc_scan_kernel(const uint32_t* __restrict__ tile_count, uint32_t ntiles, uint32_t* __restrict__ tile_offset,
               uint32_t* __restrict__ count, float* __restrict__ minmax) {
  __shared__ uint32_t wsum[32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint32_t carry = 0;
  for (uint32_t b = 0; b < ntiles; b += PC_SCAN_THREADS) {
    const uint32_t i = b + threadIdx.x;
    const uint32_t v = i < ntiles ? tile_count[i] : 0u;
    uint32_t incl = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t u = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += u;
    }
    if (lane == 31) wsum[warp] = incl;
    __syncthreads();
    if (warp == 0) {
      uint32_t s = wsum[lane];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const uint32_t u = __shfl_up_sync(0xffffffffu, s, o);
        if (lane >= o) s += u;
      }
      wsum[lane] = s;
    }
    __syncthreads();
    if (i < ntiles) tile_offset[i] = carry + (warp ? wsum[warp - 1] : 0u) + incl - v;
    carry += wsum[31];
    __syncthreads();                              // wsum is rewritten by the next chunk
  }
  if (threadIdx.x == 0) *count = carry;
  if (threadIdx.x < 6) minmax[threadIdx.x] = threadIdx.x < 3 ? INFINITY : -INFINITY;
}

// Order-preserving key of a non-NaN float (-0 below +0), and back.
__device__ __forceinline__ uint32_t pc_key(float f) {
  const uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float pc_unkey(uint32_t k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

// Float min / max by integer atomics in the same order (-0 below +0): exact, so the result does not depend on the order
// the CTAs arrive in.  Non-negative floats order as signed ints; negative floats order in reverse as unsigned ints and
// above every non-negative float.
__device__ __forceinline__ void pc_atomic_min(float* a, float v) {
  if (!signbit(v)) atomicMin(reinterpret_cast<int*>(a), __float_as_int(v));
  else atomicMax(reinterpret_cast<unsigned*>(a), __float_as_uint(v));
}
__device__ __forceinline__ void pc_atomic_max(float* a, float v) {
  if (!signbit(v)) atomicMax(reinterpret_cast<int*>(a), __float_as_int(v));
  else atomicMin(reinterpret_cast<unsigned*>(a), __float_as_uint(v));
}

__global__ void __launch_bounds__(PC_THREADS)
pc_compact_kernel(const float* __restrict__ pts, const uint8_t* __restrict__ mask, const uint32_t* __restrict__ rgba,
                  uint32_t n, const uint32_t* __restrict__ tile_offset, const uint32_t* __restrict__ count,
                  float* __restrict__ out, float* __restrict__ minmax) {
  __shared__ uint32_t wcount[PC_PER][PC_WARPS];
  __shared__ uint32_t red[2][3][PC_WARPS];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t t0 = blockIdx.x * PC_TILE;
  bool keep[PC_PER];
  uint32_t pre[PC_PER];
#pragma unroll
  for (int k = 0; k < PC_PER; ++k) {
    const uint32_t i = t0 + k * PC_THREADS + threadIdx.x;
    keep[k] = i < n && mask[i] != 0;
    const uint32_t bal = __ballot_sync(0xffffffffu, keep[k]);
    pre[k] = __popc(bal & ((1u << lane) - 1u));
    if (lane == 0) wcount[k][warp] = __popc(bal);
  }
  __syncthreads();
  const uint32_t total = *count;
  uint32_t* colors = reinterpret_cast<uint32_t*>(out + 3 * static_cast<int64_t>(total));
  uint32_t lo[3] = {0xffffffffu, 0xffffffffu, 0xffffffffu}, hi[3] = {0u, 0u, 0u};   // none yet (no NaN has these keys)
  uint32_t run = tile_offset[blockIdx.x];
#pragma unroll
  for (int k = 0; k < PC_PER; ++k) {
    uint32_t before = 0, all = 0;
#pragma unroll
    for (int w = 0; w < PC_WARPS; ++w) {
      before += w < warp ? wcount[k][w] : 0u;
      all += wcount[k][w];
    }
    if (keep[k]) {
      const uint32_t i = t0 + k * PC_THREADS + threadIdx.x;
      const int64_t o = run + before + pre[k];
#pragma unroll
      for (int j = 0; j < 3; ++j) {
        const float v = __ldg(pts + 3 * static_cast<int64_t>(i) + j);
        out[3 * o + j] = v;
        if (v == v) {                             // NaN coordinates stay out of the accessor bounds
          lo[j] = min(lo[j], pc_key(v));
          hi[j] = max(hi[j], pc_key(v));
        }
      }
      colors[o] = __ldg(rgba + i);
    }
    run += all;
  }
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    lo[j] = __reduce_min_sync(0xffffffffu, lo[j]);
    hi[j] = __reduce_max_sync(0xffffffffu, hi[j]);
    if (lane == 0) { red[0][j][warp] = lo[j]; red[1][j][warp] = hi[j]; }
  }
  __syncthreads();
  if (threadIdx.x < 6) {
    const int which = threadIdx.x / 3, j = threadIdx.x % 3;
    uint32_t k = red[which][j][0];
#pragma unroll
    for (int w = 1; w < PC_WARPS; ++w) k = which ? max(k, red[1][j][w]) : min(k, red[0][j][w]);
    if (which == 0 && k != 0xffffffffu) pc_atomic_min(minmax + j, pc_unkey(k));
    if (which == 1 && k != 0u) pc_atomic_max(minmax + 3 + j, pc_unkey(k));
  }
}

inline int64_t pc_tiles(int64_t n) { return (n + PC_TILE - 1) / PC_TILE; }

}  // namespace iggt

using namespace iggt;

extern "C" int iggt_pointcloud_workspace(int64_t n, int64_t* bytes) {
  if (!bytes || n <= 0 || n >= (1LL << 32)) return -1;
  *bytes = 2 * pc_tiles(n) * static_cast<int64_t>(sizeof(uint32_t));
  return 0;
}

extern "C" int iggt_pointcloud_select(const float* points, const float* conf, int64_t n, const float* thr,
                                      const void* color, int color_kind, int64_t color_hw, int64_t color_sf,
                                      int64_t color_sc, int64_t color_sp, int bg_flags, uint8_t* mask, float* planes,
                                      int64_t ldp, uint32_t* rgba, void* workspace, iggt_stream_t stream) {
  if (!points || !conf || !color || !mask || !planes || !rgba || !workspace || n <= 0 || n >= (1LL << 32) || ldp < n ||
      (color_kind != IGGT_PC_COLOR_F32 && color_kind != IGGT_PC_COLOR_U8) || color_hw <= 0 || color_hw > n ||
      (bg_flags & ~(IGGT_PC_MASK_BLACK | IGGT_PC_MASK_WHITE)))
    return -1;
  const PcColor col{color, color_kind == IGGT_PC_COLOR_U8, static_cast<uint32_t>(color_hw), color_sf, color_sc, color_sp};
  const unsigned grid = static_cast<unsigned>(pc_tiles(n));
  pc_select_kernel<<<grid, PC_THREADS, 0, (cudaStream_t)stream>>>(points, conf, static_cast<uint32_t>(n), thr, col,
                                                                   bg_flags, mask, planes, ldp, rgba,
                                                                   static_cast<uint32_t*>(workspace));
  return (int)cudaGetLastError();
}

extern "C" int iggt_pointcloud_compact(const float* points, const uint8_t* mask, const uint32_t* rgba, int64_t n,
                                       void* workspace, void* out, uint32_t* count, float* minmax,
                                       iggt_stream_t stream) {
  if (!points || !mask || !rgba || !workspace || !out || !count || !minmax || n <= 0 || n >= (1LL << 32)) return -1;
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t ntiles = pc_tiles(n);
  uint32_t* tile_count = static_cast<uint32_t*>(workspace);
  uint32_t* tile_offset = tile_count + ntiles;
  pc_scan_kernel<<<1, PC_SCAN_THREADS, 0, st>>>(tile_count, static_cast<uint32_t>(ntiles), tile_offset, count, minmax);
  pc_compact_kernel<<<static_cast<unsigned>(ntiles), PC_THREADS, 0, st>>>(points, mask, rgba, static_cast<uint32_t>(n),
                                                                          tile_offset, count,
                                                                          static_cast<float*>(out), minmax);
  return (int)cudaGetLastError();
}
