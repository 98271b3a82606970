// Exact k-nearest-neighbour feature averaging over a multi-view point map (SURVEY.md 8f row 2).
//
// The reference smooths the per-pixel instance features over the k = 20 nearest 3-D points of ALL views before
// clustering (demo.py:376-378 -> iggt/utils/misc.py:24-78: torch_geometric knn_graph(loop=False) + torch_scatter
// scatter_mean, on the CPU by default).  GPU design: no tree, no hash grid - points are ordered along a 63-bit
// Morton curve (the sort itself is a library radix sort on the host side of the C ABI), cut into tiles of 256
// consecutive points with an axis-aligned bounding box each, and every tile of queries runs a block-pruned brute-force
// search: 256 threads = 256 queries, candidate tiles staged in shared memory and broadcast to all threads, a per-thread
// top-k in registers, tiles skipped when their box is farther than the current k-th distance (first for the whole
// query tile, then per warp).  The search is exact for ANY ordering; the Morton order only makes the boxes tight, and
// because tiles hold a fixed number of points they adapt to the 1/depth^2 density of un-projected depth maps and to
// far outliers, where a uniform grid degenerates.  The mean over the neighbours' feature rows is fused into the tail.
#include <cuda_runtime.h>
#include <math_constants.h>
#include <stdint.h>
#include "../../include/iggt_b200.h"

namespace iggt {

constexpr int KNN_TILE = 256;
constexpr float KNN_SLACK = 1.000002f;      // boxes are pruned only when farther than worst * SLACK (fp32 rounding)

__device__ __forceinline__ uint64_t spread21(uint32_t v) {
  uint64_t x = v & 0x1fffffu;
  x = (x | x << 32) & 0x1f00000000ffffULL;
  x = (x | x << 16) & 0x1f0000ff0000ffULL;
  x = (x | x << 8) & 0x100f00f00f00f00fULL;
  x = (x | x << 4) & 0x10c30c30c30c30c3ULL;
  x = (x | x << 2) & 0x1249249249249249ULL;
  return x;
}

// 63-bit Morton code of every point on a cubic lattice spanning the bounding box [lo, hi] (device pointers).
__global__ void __launch_bounds__(256)
knn_morton_kernel(const float* __restrict__ pts, int64_t n, const float* __restrict__ lo, const float* __restrict__ hi,
                  int64_t* __restrict__ codes) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float l0 = lo[0], l1 = lo[1], l2 = lo[2];
  const float ext = fmaxf(fmaxf(hi[0] - l0, hi[1] - l1), hi[2] - l2);
  const float s = ext > 0.f ? 2097151.0f / ext : 0.f;
  const uint32_t cx = static_cast<uint32_t>(fminf(fmaxf((pts[i * 3 + 0] - l0) * s, 0.f), 2097151.f));
  const uint32_t cy = static_cast<uint32_t>(fminf(fmaxf((pts[i * 3 + 1] - l1) * s, 0.f), 2097151.f));
  const uint32_t cz = static_cast<uint32_t>(fminf(fmaxf((pts[i * 3 + 2] - l2) * s, 0.f), 2097151.f));
  codes[i] = static_cast<int64_t>(spread21(cx) | (spread21(cy) << 1) | (spread21(cz) << 2));
}

// Gather the points into curve order as (x, y, z, original index) and box every tile of 256.
__global__ void __launch_bounds__(KNN_TILE)
knn_reorder_kernel(const float* __restrict__ pts, const int64_t* __restrict__ order, int64_t n,
                   float4* __restrict__ sorted, float* __restrict__ aabb) {
  __shared__ float red[6][KNN_TILE / 32];
  const int t = threadIdx.x;
  const int64_t pos = static_cast<int64_t>(blockIdx.x) * KNN_TILE + t;
  float mn[3] = {CUDART_INF_F, CUDART_INF_F, CUDART_INF_F}, mx[3] = {-CUDART_INF_F, -CUDART_INF_F, -CUDART_INF_F};
  if (pos < n) {
    const int64_t id = order[pos];
    const float x = pts[id * 3], y = pts[id * 3 + 1], z = pts[id * 3 + 2];
    sorted[pos] = make_float4(x, y, z, __int_as_float(static_cast<int>(id)));
    mn[0] = mx[0] = x; mn[1] = mx[1] = y; mn[2] = mx[2] = z;
  }
#pragma unroll
  for (int a = 0; a < 3; ++a) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      mn[a] = fminf(mn[a], __shfl_xor_sync(0xffffffffu, mn[a], o));
      mx[a] = fmaxf(mx[a], __shfl_xor_sync(0xffffffffu, mx[a], o));
    }
    if ((t & 31) == 0) { red[a][t >> 5] = mn[a]; red[3 + a][t >> 5] = mx[a]; }
  }
  __syncthreads();
  if (t < 6) {
    float v = red[t][0];
    for (int w = 1; w < KNN_TILE / 32; ++w) v = t < 3 ? fminf(v, red[t][w]) : fmaxf(v, red[t][w]);
    aabb[static_cast<int64_t>(blockIdx.x) * 6 + t] = v;
  }
}

__device__ __forceinline__ float point_box_d2(const float4& q, const float* __restrict__ b) {
  const float dx = fmaxf(fmaxf(b[0] - q.x, q.x - b[3]), 0.f);
  const float dy = fmaxf(fmaxf(b[1] - q.y, q.y - b[4]), 0.f);
  const float dz = fmaxf(fmaxf(b[2] - q.z, q.z - b[5]), 0.f);
  return fmaf(dz, dz, fmaf(dy, dy, dx * dx));
}
__device__ __forceinline__ float box_box_d2(const float* __restrict__ a, const float* __restrict__ b) {
  const float dx = fmaxf(fmaxf(b[0] - a[3], a[0] - b[3]), 0.f);
  const float dy = fmaxf(fmaxf(b[1] - a[4], a[1] - b[4]), 0.f);
  const float dz = fmaxf(fmaxf(b[2] - a[5], a[2] - b[5]), 0.f);
  return fmaf(dz, dz, fmaf(dy, dy, dx * dx));
}

// One CTA = KNN_QT consecutive queries of the curve order (a quarter of a tile: small CTAs keep the bounding box of
// the queries tight and confine the wait-for-the-slowest-warp at the tile barriers to two warps; ~9 CTAs per SM hide
// each other's latencies).  KMAX >= k list slots live in registers: slots [0, k) start at +inf (worst first, replaced
// first), slots [k, KMAX) at -inf (never the worst, never replaced).
// Candidates that beat the current k-th distance are not inserted on the spot - a lane that inserts would drag the
// other 31 through ~100 predicated instructions - but parked in a per-thread shared-memory queue (KNN_Q deep) that the
// whole warp drains together when any lane's queue could overflow and at the end of every tile.
constexpr int KNN_QT = 64;     // queries per CTA
constexpr int KNN_Q = 16;      // queue depth per thread
constexpr int KNN_G = 8;       // candidates between two "is any queue nearly full" votes
constexpr int KNN_PT = KNN_TILE / KNN_QT;   // candidate points each thread stages per tile

template <int KMAX>
__global__ void __launch_bounds__(KNN_QT)
knn_mean_kernel(const float4* __restrict__ sorted, const float* __restrict__ aabb, int64_t n, int nblocks, int k,
                const float* __restrict__ feats, int F, float* __restrict__ out, int32_t* __restrict__ out_idx,
                float* __restrict__ out_d2, unsigned long long* __restrict__ stats) {
  __shared__ float4 tile[KNN_TILE];
  __shared__ float tile_box[6];
  __shared__ float q_d[KNN_Q][KNN_QT];
  __shared__ int q_i[KNN_Q][KNN_QT];
  __shared__ int list[KNN_TILE];
  __shared__ int warp_cnt[KNN_QT / 32];
  __shared__ float red[6][KNN_QT / 32];
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const int64_t pos = static_cast<int64_t>(blockIdx.x) * KNN_QT + t;
  const int b = static_cast<int>(pos / KNN_TILE);          // the candidate tile this CTA's queries live in
  const bool valid = pos < n;
  const float4 q = valid ? sorted[pos] : make_float4(0.f, 0.f, 0.f, 0.f);

  // bounding box of this CTA's queries
  float my_box[6];
  {
    float v[6] = {valid ? q.x : CUDART_INF_F, valid ? q.y : CUDART_INF_F, valid ? q.z : CUDART_INF_F,
                  valid ? -q.x : CUDART_INF_F, valid ? -q.y : CUDART_INF_F, valid ? -q.z : CUDART_INF_F};
#pragma unroll
    for (int a = 0; a < 6; ++a) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) v[a] = fminf(v[a], __shfl_xor_sync(0xffffffffu, v[a], o));
      if (lane == 0) red[a][warp] = v[a];
    }
    __syncthreads();
#pragma unroll
    for (int a = 0; a < 6; ++a) {
      float m = red[a][0];
#pragma unroll
      for (int w = 1; w < KNN_QT / 32; ++w) m = fminf(m, red[a][w]);
      my_box[a] = a < 3 ? m : -m;
    }
    __syncthreads();
  }

  float dist[KMAX];
  int idx[KMAX];
#pragma unroll
  for (int i = 0; i < KMAX; ++i) { dist[i] = (valid && i < k) ? CUDART_INF_F : -CUDART_INF_F; idx[i] = -1; }
  float worst = valid ? CUDART_INF_F : -CUDART_INF_F;   // an idle thread (past the end) never wants anything
  int slot = 0;
  int queued = 0;
  unsigned long long st_loaded = 0, st_computed = 0, st_drains = 0;

  // merge this thread's parked candidates into its top-k (warp-converged: every lane calls it together)
  auto drain = [&]() {
    const int deepest = __reduce_max_sync(0xffffffffu, queued);
    for (int e = 0; e < deepest; ++e) {
      const float d = e < queued ? q_d[e][t] : CUDART_INF_F;
      if (d < worst) {                                   // re-check: the bound may have moved since it was parked
        const int id = q_i[e][t];
#pragma unroll
        for (int i = 0; i < KMAX; ++i)
          if (i == slot) { dist[i] = d; idx[i] = id; }
        worst = -CUDART_INF_F;
#pragma unroll
        for (int i = 0; i < KMAX; ++i)
          if (dist[i] > worst) { worst = dist[i]; slot = i; }
      }
    }
    queued = 0;
    ++st_drains;
  };

  auto process_tile = [&](int c) {
    __syncthreads();                                     // everyone is done with the previous tile
#pragma unroll
    for (int r = 0; r < KNN_PT; ++r) {
      const int64_t cp = static_cast<int64_t>(c) * KNN_TILE + r * KNN_QT + t;
      tile[r * KNN_QT + t] =
          cp < n ? sorted[cp] : make_float4(CUDART_INF_F, CUDART_INF_F, CUDART_INF_F, __int_as_float(-1));
    }
    if (t < 6) tile_box[t] = aabb[static_cast<int64_t>(c) * 6 + t];
    __syncthreads();
    ++st_loaded;
    const bool want = point_box_d2(q, tile_box) <= worst * KNN_SLACK;
    if (!__any_sync(0xffffffffu, want)) return;          // the whole warp skips a tile nobody can improve from
    ++st_computed;
    const int self = (c == b) ? static_cast<int>(pos - static_cast<int64_t>(b) * KNN_TILE) : -1;
#pragma unroll 1
    for (int j0 = 0; j0 < KNN_TILE; j0 += KNN_G) {
      float d[KNN_G];
      int id[KNN_G];
#pragma unroll
      for (int j = 0; j < KNN_G; ++j) {                  // straight-line: the KNN_G broadcast loads go out together
        const float4 cpt = tile[j0 + j];
        const float dx = cpt.x - q.x, dy = cpt.y - q.y, dz = cpt.z - q.z;
        d[j] = (j0 + j != self) ? fmaf(dz, dz, fmaf(dy, dy, dx * dx)) : CUDART_INF_F;   // loop=False: not its own neighbour
        id[j] = __float_as_int(cpt.w);
      }
      float dmin = d[0];
#pragma unroll
      for (int j = 1; j < KNN_G; ++j) dmin = fminf(dmin, d[j]);
      if (__any_sync(0xffffffffu, dmin < worst)) {
#pragma unroll
        for (int j = 0; j < KNN_G; ++j) {
          if (d[j] < worst) {
            q_d[queued][t] = d[j];
            q_i[queued][t] = id[j];
            ++queued;
          }
        }
        // the next group can park up to KNN_G more per lane: drain while every queue still has that much room
        if (__any_sync(0xffffffffu, queued > KNN_Q - KNN_G)) drain();
      }
    }
    if (__any_sync(0xffffffffu, queued > 0)) drain();    // fresh bounds for the next tile's box tests
  };

  // ---- phase 1: the curve neighbourhood gives every query a first k-th distance
  for (int o = 0; o < 5; ++o) {
    const int c = b + ((o & 1) ? (o + 1) / 2 : -(o / 2));   // b, b+1, b-1, b+2, b-2
    if (c >= 0 && c < nblocks) process_tile(c);
  }
  // ---- phase 2: every other tile whose box is within the largest k-th distance of this CTA's queries
  for (int c0 = 0; c0 < nblocks; c0 += KNN_TILE) {
    float r2 = worst;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) r2 = fmaxf(r2, __shfl_xor_sync(0xffffffffu, r2, o));
    __syncthreads();                                     // list / red / warp_cnt of the previous chunk are consumed
    if (lane == 0) red[0][warp] = r2;
    __syncthreads();
    r2 = red[0][0];
#pragma unroll
    for (int w = 1; w < KNN_QT / 32; ++w) r2 = fmaxf(r2, red[0][w]);
    const float r2s = r2 * KNN_SLACK;
    int total = 0;
#pragma unroll 1
    for (int r = 0; r < KNN_PT; ++r) {                   // KNN_QT threads test a chunk of KNN_TILE boxes in KNN_PT rounds
      const int c = c0 + r * KNN_QT + t;
      const bool keep = c < nblocks && (c < b - 2 || c > b + 2) &&
                        box_box_d2(my_box, aabb + static_cast<int64_t>(c) * 6) <= r2s;
      const uint32_t m = __ballot_sync(0xffffffffu, keep);
      if (lane == 0) warp_cnt[warp] = __popc(m);
      __syncthreads();
      int base = total;
#pragma unroll
      for (int w = 0; w < KNN_QT / 32; ++w) {
        if (w < warp) base += warp_cnt[w];
        total += warp_cnt[w];
      }
      if (keep) list[base + __popc(m & ((1u << lane) - 1u))] = c;
      __syncthreads();
    }
    for (int i = 0; i < total; ++i) process_tile(list[i]);
  }

  if (stats && lane == 0) {
    if (warp == 0) atomicAdd(stats + 0, st_loaded);
    atomicAdd(stats + 1, st_computed);
    atomicAdd(stats + 2, st_drains);
  }
  // ---- tail: mean of the neighbours' feature rows (scatter_mean: sum / max(count, 1)), written at the ORIGINAL index
  if (!valid) return;
  const int64_t qid = __float_as_int(q.w);
  int cnt = 0;
#pragma unroll
  for (int i = 0; i < KMAX; ++i) cnt += (i < k && idx[i] >= 0) ? 1 : 0;
  const float denom = static_cast<float>(cnt > 0 ? cnt : 1);
  if (feats && out) {
    if ((F & 3) == 0) {
      for (int f0 = 0; f0 < F; f0 += 4) {
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int i = 0; i < KMAX; ++i) {
          if (i < k && idx[i] >= 0) {
            const float4 v = __ldg(reinterpret_cast<const float4*>(feats + static_cast<int64_t>(idx[i]) * F + f0));
            acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
          }
        }
        *reinterpret_cast<float4*>(out + qid * F + f0) =
            make_float4(acc.x / denom, acc.y / denom, acc.z / denom, acc.w / denom);
      }
    } else {
      for (int f = 0; f < F; ++f) {
        float acc = 0.f;
#pragma unroll
        for (int i = 0; i < KMAX; ++i)
          if (i < k && idx[i] >= 0) acc += __ldg(feats + static_cast<int64_t>(idx[i]) * F + f);
        out[qid * F + f] = acc / denom;
      }
    }
  }
  if (out_idx) {
#pragma unroll
    for (int i = 0; i < KMAX; ++i)
      if (i < k) {
        out_idx[qid * k + i] = idx[i];
        if (out_d2) out_d2[qid * k + i] = dist[i];
      }
  }
}

}  // namespace iggt

using namespace iggt;

extern "C" int iggt_knn_morton(const float* points, int64_t n, const float* lo, const float* hi, int64_t* codes,
                               iggt_stream_t stream) {
  if (!points || !lo || !hi || !codes || n <= 0) return -1;
  knn_morton_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(points, n, lo, hi, codes);
  return (int)cudaGetLastError();
}

extern "C" int iggt_knn_reorder(const float* points, const int64_t* order, int64_t n, float* sorted4, float* aabb,
                                iggt_stream_t stream) {
  if (!points || !order || !sorted4 || !aabb || n <= 0 || n >= (1LL << 31)) return -1;
  const unsigned nblocks = static_cast<unsigned>((n + KNN_TILE - 1) / KNN_TILE);
  knn_reorder_kernel<<<nblocks, KNN_TILE, 0, (cudaStream_t)stream>>>(points, order, n,
                                                                    reinterpret_cast<float4*>(sorted4), aabb);
  return (int)cudaGetLastError();
}

extern "C" int iggt_knn_mean_features(const float* sorted4, const float* aabb, int64_t n, int k, const float* feats,
                                      int F, float* out, int32_t* out_idx, float* out_d2, uint64_t* stats,
                                      iggt_stream_t stream) {
  if (!sorted4 || !aabb || n <= 0 || n >= (1LL << 31) || k <= 0 || k > 32) return -1;
  if ((feats == nullptr) != (out == nullptr) || (feats && F <= 0)) return -1;
  if (!out && !out_idx) return -1;
  const int nblocks = static_cast<int>((n + KNN_TILE - 1) / KNN_TILE);
  const unsigned grid = static_cast<unsigned>((n + KNN_QT - 1) / KNN_QT);
  const float4* s4 = reinterpret_cast<const float4*>(sorted4);
  cudaStream_t st = (cudaStream_t)stream;
  if (k <= 8) knn_mean_kernel<8><<<grid, KNN_QT, 0, st>>>(s4, aabb, n, nblocks, k, feats, F, out, out_idx, out_d2,
                                                       reinterpret_cast<unsigned long long*>(stats));
  else if (k <= 16) knn_mean_kernel<16><<<grid, KNN_QT, 0, st>>>(s4, aabb, n, nblocks, k, feats, F, out, out_idx, out_d2,
                                                       reinterpret_cast<unsigned long long*>(stats));
  else if (k <= 24) knn_mean_kernel<24><<<grid, KNN_QT, 0, st>>>(s4, aabb, n, nblocks, k, feats, F, out, out_idx, out_d2,
                                                       reinterpret_cast<unsigned long long*>(stats));
  else knn_mean_kernel<32><<<grid, KNN_QT, 0, st>>>(s4, aabb, n, nblocks, k, feats, F, out, out_idx, out_d2,
                                                       reinterpret_cast<unsigned long long*>(stats));
  return (int)cudaGetLastError();
}
