// HDBSCAN of the per-pixel instance features on the device (demo.py:389-397 -> iggt/utils/misc.py:81-170, which
// calls cuML / the scikit-learn-contrib `hdbscan` package on the host).
//
// Device part, all in fp32 over 8-d points (smaller C is zero-padded):
//   1. core distances: the exact distance to the k-th nearest OTHER point (k = min_samples, contrib semantics);
//   2. the minimum spanning tree of the mutual-reachability graph mrd(i,j) = max(core_i, core_j, d_ij), by Boruvka;
//   3. the noise fill: every noise point takes the label of its exact nearest labelled point, fused with colouring.
// Every search reuses the idea of knn.cu (whose kernels are not shared or changed): points are sorted along a Morton
// key, cut into tiles of 256 consecutive points with an 8-d bounding box each, and a tile is skipped when its box
// bound cannot beat the current best.  Here one warp holds 32 consecutive queries and reads candidate points straight
// from global memory (every lane reads the same point: one broadcast transaction); a warp first tests 32 tile boxes at
// once against the box of its own queries, then each surviving tile against each query.  Distances to boxes and to
// points are evaluated with the same operation order, so rounding keeps the box bound below every point distance in
// the box and the searches are exact for any point order.  All distances are kept squared.
//
// Host part (no GPU): iggt_hdbscan_labels turns the sorted MST into labels exactly as scikit-learn 1.9's
// tree_to_labels does (single-linkage tree, condensed tree, stabilities, excess-of-mass selection with the
// cluster_selection_epsilon rule, labelling), restated below.
#include <cuda_runtime.h>
#include <math_constants.h>
#include <stdint.h>

#include <algorithm>
#include <cmath>
#include <vector>

#include "launch.cuh"
#include "../../include/iggt_b200.h"

namespace iggt {

constexpr int CL_TILE = 256;     // points per tile (and per bounding box)
constexpr int CL_CTA = 64;       // threads per CTA of the search kernels: two independent warps
constexpr int CL_KMAX = 512;     // largest k of the core-distance search (its max-heap lives in shared memory)

__device__ __forceinline__ uint64_t spread8(uint32_t v) {   // 7 bits -> every 8th bit
  uint64_t x = 0;
#pragma unroll
  for (int b = 0; b < 7; ++b) x |= static_cast<uint64_t>((v >> b) & 1u) << (8 * b);
  return x;
}

// 56-bit Morton key of every 8-d point on a 128^8 lattice spanning each axis' extent [lo, hi].
__global__ void __launch_bounds__(256)
cl_morton_kernel(const float* __restrict__ x, int64_t n, const float* __restrict__ lo, const float* __restrict__ hi,
                 int64_t* __restrict__ codes) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint64_t code = 0;
#pragma unroll
  for (int a = 0; a < 8; ++a) {
    const float ext = hi[a] - lo[a];
    const float s = ext > 0.f ? 127.0f / ext : 0.f;
    const uint32_t c = static_cast<uint32_t>(fminf(fmaxf((x[i * 8 + a] - lo[a]) * s, 0.f), 127.f));
    code |= spread8(c) << a;
  }
  codes[i] = static_cast<int64_t>(code);
}

// Gather the points into key order with their original index, and box every tile (min 8, max 8).
__global__ void __launch_bounds__(CL_TILE)
cl_reorder_kernel(const float* __restrict__ x, const int64_t* __restrict__ order, int64_t n, float4* __restrict__ sorted,
                  int32_t* __restrict__ orig, float* __restrict__ box) {
  __shared__ float red[16][CL_TILE / 32];
  const int t = threadIdx.x;
  const int64_t pos = static_cast<int64_t>(blockIdx.x) * CL_TILE + t;
  float v[16];
#pragma unroll
  for (int a = 0; a < 8; ++a) { v[a] = CUDART_INF_F; v[8 + a] = -CUDART_INF_F; }
  if (pos < n) {
    const int64_t id = order[pos];
    const float4 p0 = *reinterpret_cast<const float4*>(x + id * 8);
    const float4 p1 = *reinterpret_cast<const float4*>(x + id * 8 + 4);
    sorted[pos * 2] = p0;
    sorted[pos * 2 + 1] = p1;
    orig[pos] = static_cast<int32_t>(id);
    const float p[8] = {p0.x, p0.y, p0.z, p0.w, p1.x, p1.y, p1.z, p1.w};
#pragma unroll
    for (int a = 0; a < 8; ++a) { v[a] = p[a]; v[8 + a] = p[a]; }
  }
#pragma unroll
  for (int a = 0; a < 16; ++a) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float w = __shfl_xor_sync(0xffffffffu, v[a], o);
      v[a] = a < 8 ? fminf(v[a], w) : fmaxf(v[a], w);
    }
    if ((t & 31) == 0) red[a][t >> 5] = v[a];
  }
  __syncthreads();
  if (t < 16) {
    float r = red[t][0];
    for (int w = 1; w < CL_TILE / 32; ++w) r = t < 8 ? fminf(r, red[t][w]) : fmaxf(r, red[t][w]);
    box[static_cast<int64_t>(blockIdx.x) * 16 + t] = r;
  }
}

// Squared distances, all evaluated in the same order (monotone rounding: box bound <= any point distance in the box).
__device__ __forceinline__ float d2_acc(float acc, float d) { return fmaf(d, d, acc); }
__device__ __forceinline__ float point_d2(const float (&q)[8], const float4& a, const float4& b) {
  float acc = (a.x - q[0]) * (a.x - q[0]);
  acc = d2_acc(acc, a.y - q[1]); acc = d2_acc(acc, a.z - q[2]); acc = d2_acc(acc, a.w - q[3]);
  acc = d2_acc(acc, b.x - q[4]); acc = d2_acc(acc, b.y - q[5]); acc = d2_acc(acc, b.z - q[6]);
  return d2_acc(acc, b.w - q[7]);
}
// Gap of a point to [lo, hi] on one axis: |p - q| >= gap for every p in the box, and the rounding of the
// subtraction is monotone, so gap^2 <= fl(p - q)^2.
__device__ __forceinline__ float gap(float q, float lo, float hi) { return fmaxf(fmaxf(lo - q, q - hi), 0.f); }
__device__ __forceinline__ float point_box_d2(const float (&q)[8], const float* __restrict__ b) {
  float g = gap(q[0], b[0], b[8]);
  float acc = g * g;
#pragma unroll
  for (int a = 1; a < 8; ++a) { g = gap(q[a], b[a], b[8 + a]); acc = d2_acc(acc, g); }
  return acc;
}
__device__ __forceinline__ float box_box_d2(const float (&w)[16], const float* __restrict__ b) {
  float g = fmaxf(fmaxf(b[0] - w[8], w[0] - b[8]), 0.f);
  float acc = g * g;
#pragma unroll
  for (int a = 1; a < 8; ++a) { g = fmaxf(fmaxf(b[a] - w[8 + a], w[a] - b[8 + a]), 0.f); acc = d2_acc(acc, g); }
  return acc;
}

// The block-pruned search of one warp over all tiles.  The policy P holds each lane's state and provides
//   bound()            the lane's pruning bound (-inf: the lane wants nothing),
//   floor()            a lower bound of every candidate's cost for this lane, independent of the tile,
//   tile_floor(c)      a lower bound of every candidate's cost in tile c, independent of the query,
//   skip(c)            the lane needs nothing from tile c;  warp_skip(c): no lane of the warp needs anything from it,
//   want(lb, bound)    whether a cost lower bound lb can still beat the bound (strict or not, per policy),
//   visit(j, d2)       one candidate (sorted position j, squared distance d2),
//   after_tile()       called by every lane after each searched tile.
// Cost lower bound of tile c for a lane: max(point-box distance, floor(), tile_floor(c)).
template <class P>
__device__ void warp_search(P& p, const float4* __restrict__ sorted, const float* __restrict__ box, int64_t n, int nb,
                            const float (&q)[8], bool active, int64_t pos0) {
  const int lane = threadIdx.x & 31;
  float wb[16];                                         // the box of the warp's active queries
#pragma unroll
  for (int a = 0; a < 8; ++a) {
    float mn = active ? q[a] : CUDART_INF_F, mx = active ? q[a] : -CUDART_INF_F;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    }
    wb[a] = mn; wb[8 + a] = mx;
  }
  if (!__any_sync(0xffffffffu, active)) return;
  const int b = static_cast<int>(pos0 / CL_TILE);

  auto search_tile = [&](int c) {
    const float lb = fmaxf(fmaxf(point_box_d2(q, box + static_cast<int64_t>(c) * 16), p.floor()), p.tile_floor(c));
    const bool want = !p.skip(c) && p.want(lb, p.bound());
    if (!__any_sync(0xffffffffu, want)) return;
    const int64_t j0 = static_cast<int64_t>(c) * CL_TILE;
    const int cnt = static_cast<int>(min(static_cast<int64_t>(CL_TILE), n - j0));
#pragma unroll 4
    for (int jj = 0; jj < cnt; ++jj) {
      const int64_t j = j0 + jj;
      const float4 a = __ldg(sorted + j * 2), bq = __ldg(sorted + j * 2 + 1);
      p.visit(static_cast<int>(j), point_d2(q, a, bq));
    }
    p.after_tile();
  };

  // the curve neighbourhood first: it gives every lane a tight bound early
  for (int o = 0; o < 5; ++o) {
    const int c = b + ((o & 1) ? (o + 1) / 2 : -(o / 2));   // b, b+1, b-1, b+2, b-2
    if (c >= 0 && c < nb) search_tile(c);
  }
  for (int c0 = 0; c0 < nb; c0 += 32) {
    float wbound = p.bound(), wfloor = active ? p.floor() : CUDART_INF_F;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      wbound = fmaxf(wbound, __shfl_xor_sync(0xffffffffu, wbound, o));
      wfloor = fminf(wfloor, __shfl_xor_sync(0xffffffffu, wfloor, o));
    }
    const int c = c0 + lane;
    bool keep = c < nb && (c < b - 2 || c > b + 2) && !p.warp_skip(c);
    if (keep) keep = p.want(fmaxf(fmaxf(box_box_d2(wb, box + static_cast<int64_t>(c) * 16), wfloor), p.tile_floor(c)),
                            wbound);
    uint32_t m = __ballot_sync(0xffffffffu, keep);
    while (m) {
      const int cc = c0 + __ffs(m) - 1;
      m &= m - 1;
      search_tile(cc);
    }
  }
}

// ---- 1. core distances: the k-th smallest squared distance to another point, one max-heap of k per lane
struct CorePolicy {
  float* heap;         // shared memory, slot s of this lane at heap[s * CL_CTA]
  int k;
  int self;
  bool active;
  float worst;         // heap[0]
  __device__ float bound() const { return active ? worst : -CUDART_INF_F; }
  __device__ float floor() const { return 0.f; }
  __device__ float tile_floor(int) const { return 0.f; }
  __device__ bool skip(int) const { return false; }
  __device__ bool warp_skip(int) const { return false; }
  __device__ bool want(float lb, float bound) const { return lb < bound; }
  __device__ void after_tile() {}
  __device__ void visit(int j, float d2) {
    if (!(d2 < worst) || j == self) return;
    int s = 0;                                          // replace the root and sift down
    while (true) {
      const int l = 2 * s + 1, r = l + 1;
      if (l >= k) break;
      int c = l;
      float cv = heap[l * CL_CTA];
      if (r < k) {
        const float rv = heap[r * CL_CTA];
        if (rv > cv) { c = r; cv = rv; }
      }
      if (!(cv > d2)) break;
      heap[s * CL_CTA] = cv;
      s = c;
    }
    heap[s * CL_CTA] = d2;
    worst = heap[0];
  }
};

__global__ void __launch_bounds__(CL_CTA)
cl_core_kernel(const float4* __restrict__ sorted, const float* __restrict__ box, int64_t n, int nb, int k,
               float* __restrict__ core2) {
  extern __shared__ float heap_smem[];
  const int t = threadIdx.x;
  const int64_t pos = static_cast<int64_t>(blockIdx.x) * CL_CTA + t;
  const bool active = pos < n;
  float q[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  if (active) {
    const float4 a = sorted[pos * 2], b = sorted[pos * 2 + 1];
    q[0] = a.x; q[1] = a.y; q[2] = a.z; q[3] = a.w; q[4] = b.x; q[5] = b.y; q[6] = b.z; q[7] = b.w;
  }
  CorePolicy p;
  p.heap = heap_smem + t;
  p.k = k;
  p.self = static_cast<int>(pos);
  p.active = active;
  p.worst = CUDART_INF_F;
  for (int s = 0; s < k; ++s) p.heap[s * CL_CTA] = CUDART_INF_F;
  warp_search(p, sorted, box, n, nb, q, active, pos - (t & 31));
  if (active) core2[pos] = p.worst;
}

// ---- 2. Boruvka on the mutual-reachability graph.  Components are named by a root (sorted position).  Each round,
// every point finds its cheapest edge to another component under the total order (weight, smaller original index,
// larger original index); each component keeps its minimum through a 64-bit atomicMin on (weight bits, smaller index)
// and then a 32-bit atomicMin on the larger index among the points that hold that key.
__device__ __forceinline__ unsigned long long key1_of(float w2, int lo) {
  return (static_cast<unsigned long long>(__float_as_uint(w2)) << 32) | static_cast<uint32_t>(lo);
}

struct BoruvkaPolicy {
  const int32_t* comp; const float* core2; const int32_t* orig; const int32_t* tcomp; const float* tcore;
  unsigned long long* key1;
  int ci, oi, wcomp;   // wcomp: the warp's common component, or -2
  float c2, bw2, cw2;
  int bj, bo;
  bool active;
  unsigned long long published;
  __device__ float bound() const { return active ? fminf(bw2, cw2) : -CUDART_INF_F; }
  __device__ float floor() const { return c2; }
  __device__ float tile_floor(int c) const { return tcore[c]; }
  __device__ bool skip(int c) const { return tcomp[c] == ci; }
  __device__ bool warp_skip(int c) const { return tcomp[c] == wcomp; }
  __device__ bool want(float lb, float bound) const { return lb <= bound; }   // ties can still win on the index
  __device__ void visit(int j, float d2) {
    if (!active) return;
    const float w2 = fmaxf(fmaxf(c2, __ldg(core2 + j)), d2);
    if (w2 > bw2 || __ldg(comp + j) == ci) return;
    const int oj = __ldg(orig + j);
    if (w2 == bw2) {
      const int lo = min(oi, oj), hi = max(oi, oj), blo = min(oi, bo), bhi = max(oi, bo);
      if (lo > blo || (lo == blo && hi >= bhi)) return;
    }
    bw2 = w2; bj = j; bo = oj;
  }
  __device__ void after_tile() {
    if (!active) return;
    if (bj >= 0) {
      const unsigned long long k1 = key1_of(bw2, min(oi, bo));
      if (k1 < published) { atomicMin(key1 + ci, k1); published = k1; }
    }
    cw2 = __uint_as_float(static_cast<uint32_t>(*reinterpret_cast<volatile unsigned long long*>(key1 + ci) >> 32));
  }
};

__global__ void __launch_bounds__(CL_CTA)
cl_boruvka_search_kernel(const float4* __restrict__ sorted, const float* __restrict__ box, int64_t n, int nb,
                         const int32_t* __restrict__ comp, const float* __restrict__ core2, const int32_t* __restrict__ orig,
                         const int32_t* __restrict__ tcomp, const float* __restrict__ tcore, unsigned long long* key1,
                         float* __restrict__ qw2, int32_t* __restrict__ qj) {
  const int t = threadIdx.x;
  const int64_t pos = static_cast<int64_t>(blockIdx.x) * CL_CTA + t;
  const bool valid = pos < n;
  float q[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  BoruvkaPolicy p;
  p.comp = comp; p.core2 = core2; p.orig = orig; p.tcomp = tcomp; p.tcore = tcore; p.key1 = key1;
  p.ci = valid ? comp[pos] : -1;
  p.oi = valid ? orig[pos] : 0;
  p.c2 = valid ? core2[pos] : 0.f;
  p.bw2 = CUDART_INF_F; p.bj = -1; p.bo = 0;
  p.published = ~0ull;
  p.cw2 = valid ? __uint_as_float(static_cast<uint32_t>(key1[p.ci] >> 32)) : CUDART_INF_F;
  p.active = valid && !(p.c2 > p.cw2);                  // every edge of this point costs at least its core distance
  if (valid) {
    const float4 a = sorted[pos * 2], b = sorted[pos * 2 + 1];
    q[0] = a.x; q[1] = a.y; q[2] = a.z; q[3] = a.w; q[4] = b.x; q[5] = b.y; q[6] = b.z; q[7] = b.w;
  }
  const int first = __shfl_sync(0xffffffffu, p.ci, 0);
  p.wcomp = __all_sync(0xffffffffu, !valid || p.ci == first) ? first : -2;
  warp_search(p, sorted, box, n, nb, q, p.active, pos - (t & 31));
  if (!valid) return;
  qj[pos] = p.bj;
  qw2[pos] = p.bw2;
  if (p.bj >= 0) {
    const unsigned long long k1 = key1_of(p.bw2, min(p.oi, p.bo));
    if (k1 < p.published) atomicMin(key1 + p.ci, k1);
  }
}

// per tile: the component all its points share (-1 if mixed) and the smallest core distance
__global__ void __launch_bounds__(CL_TILE)
cl_tile_info_kernel(const int32_t* __restrict__ comp, const float* __restrict__ core2, int64_t n,
                    int32_t* __restrict__ tcomp, float* __restrict__ tcore) {
  __shared__ float red[CL_TILE / 32];
  const int64_t j0 = static_cast<int64_t>(blockIdx.x) * CL_TILE;
  const int64_t j = j0 + threadIdx.x;
  const int c0 = comp[j0];
  const bool same = __syncthreads_and(j >= n || comp[j] == c0);
  float m = j < n ? core2[j] : CUDART_INF_F;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fminf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < CL_TILE / 32; ++w) m = fminf(m, red[w]);
    tcore[blockIdx.x] = fminf(m, red[0]);
    tcomp[blockIdx.x] = same ? c0 : -1;
  }
}

__global__ void cl_mst_init_kernel(int64_t n, int32_t* comp, int32_t* parent, unsigned long long* key1, uint32_t* key2,
                                   int32_t* pick_i) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  comp[i] = static_cast<int32_t>(i); parent[i] = static_cast<int32_t>(i);
  key1[i] = ~0ull; key2[i] = ~0u; pick_i[i] = -1;
}

// the points that hold their component's (weight, smaller index) compete on the larger index
__global__ void cl_boruvka_pick_kernel(int64_t n, const int32_t* __restrict__ comp, const int32_t* __restrict__ orig,
                                       const float* __restrict__ qw2, const int32_t* __restrict__ qj,
                                       const unsigned long long* __restrict__ key1, uint32_t* key2) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n || qj[i] < 0) return;
  const int oi = orig[i], oj = orig[qj[i]], c = comp[i];
  if (key1_of(qw2[i], min(oi, oj)) == key1[c]) atomicMin(key2 + c, static_cast<uint32_t>(max(oi, oj)));
}

__global__ void cl_boruvka_select_kernel(int64_t n, const int32_t* __restrict__ comp, const int32_t* __restrict__ orig,
                                         const float* __restrict__ qw2, const int32_t* __restrict__ qj,
                                         const unsigned long long* __restrict__ key1, const uint32_t* __restrict__ key2,
                                         int32_t* pick_i, int32_t* pick_j) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n || qj[i] < 0) return;
  const int oi = orig[i], oj = orig[qj[i]], c = comp[i];
  if (key1_of(qw2[i], min(oi, oj)) == key1[c] && static_cast<uint32_t>(max(oi, oj)) == key2[c]) {
    pick_i[c] = static_cast<int32_t>(i);
    pick_j[c] = qj[i];
  }
}

// Every component hooks onto the component at the other end of its edge, except the smaller root of a pair that
// picked the same edge; each hook adds its edge to the tree.
__global__ void cl_boruvka_hook_kernel(int64_t n, const int32_t* __restrict__ comp, const int32_t* __restrict__ orig,
                                       const int32_t* __restrict__ pick_i, const int32_t* __restrict__ pick_j,
                                       const unsigned long long* __restrict__ key1, int32_t* parent, uint32_t* counter,
                                       int32_t* ea, int32_t* eb, float* ew2) {
  const int64_t r = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (r >= n || comp[r] != r || pick_i[r] < 0) return;
  const int s = comp[pick_j[r]];
  if (pick_i[s] >= 0 && comp[pick_j[s]] == r && r < s) return;
  parent[r] = s;
  const uint32_t e = atomicAdd(counter, 1u);
  if (e >= n - 1) return;                               // a tree has n - 1 edges (the launcher reports the overflow)
  ea[e] = orig[pick_i[r]];
  eb[e] = orig[pick_j[r]];
  ew2[e] = __uint_as_float(static_cast<uint32_t>(key1[r] >> 32));
}

__global__ void cl_jump_kernel(int64_t n, const int32_t* __restrict__ comp, int32_t* parent, uint32_t* changed) {
  const int64_t r = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (r >= n || comp[r] != r) return;
  const int p = parent[r], pp = parent[p];
  if (p != pp) { parent[r] = pp; *changed = 1u; }
}

__global__ void cl_relabel_kernel(int64_t n, int32_t* comp, const int32_t* __restrict__ parent,
                                  unsigned long long* key1, uint32_t* key2, int32_t* pick_i) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  comp[i] = parent[comp[i]];
  key1[i] = ~0ull; key2[i] = ~0u; pick_i[i] = -1;
}

// ---- 3. noise fill: nearest labelled point (ties: lowest original index); label and colour at the original index
struct FillPolicy {
  const int32_t* label; const int32_t* orig; const int32_t* tcount;
  bool active;
  float bd2;
  int bo, bl;
  __device__ float bound() const { return active ? bd2 : -CUDART_INF_F; }
  __device__ float floor() const { return 0.f; }
  __device__ float tile_floor(int) const { return 0.f; }
  __device__ bool skip(int c) const { return tcount[c] == 0; }
  __device__ bool warp_skip(int c) const { return tcount[c] == 0; }
  __device__ bool want(float lb, float bound) const { return lb <= bound; }
  __device__ void after_tile() {}
  __device__ void visit(int j, float d2) {
    if (!active || d2 > bd2) return;
    const int l = __ldg(label + j);
    if (l < 0) return;
    const int oj = __ldg(orig + j);
    if (d2 == bd2 && oj >= bo) return;
    bd2 = d2; bo = oj; bl = l;
  }
};

__global__ void __launch_bounds__(CL_TILE)
cl_tile_count_kernel(const int32_t* __restrict__ label, int64_t n, int32_t* __restrict__ tcount) {
  const int64_t j = static_cast<int64_t>(blockIdx.x) * CL_TILE + threadIdx.x;
  const int c = __syncthreads_count(j < n && label[j] >= 0);
  if (threadIdx.x == 0) tcount[blockIdx.x] = c;
}

__global__ void __launch_bounds__(CL_CTA)
cl_fill_kernel(const float4* __restrict__ sorted, const float* __restrict__ box, int64_t n, int nb,
               const int32_t* __restrict__ orig, const int32_t* __restrict__ label, const int32_t* __restrict__ tcount,
               const uint8_t* __restrict__ palette, int64_t* __restrict__ out_label, uint8_t* __restrict__ out_rgb) {
  const int t = threadIdx.x;
  const int64_t pos = static_cast<int64_t>(blockIdx.x) * CL_CTA + t;
  const bool valid = pos < n;
  const int own = valid ? label[pos] : 0;
  float q[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  if (valid) {
    const float4 a = sorted[pos * 2], b = sorted[pos * 2 + 1];
    q[0] = a.x; q[1] = a.y; q[2] = a.z; q[3] = a.w; q[4] = b.x; q[5] = b.y; q[6] = b.z; q[7] = b.w;
  }
  FillPolicy p;
  p.label = label; p.orig = orig; p.tcount = tcount;
  p.active = valid && own < 0;
  p.bd2 = CUDART_INF_F; p.bo = 0x7fffffff; p.bl = -1;
  warp_search(p, sorted, box, n, nb, q, p.active, pos - (t & 31));
  if (!valid) return;
  const int l = own >= 0 ? own : p.bl;
  const int64_t o = orig[pos];
  out_label[o] = l;
  if (out_rgb && l >= 0) {
    out_rgb[o * 3] = palette[l * 3]; out_rgb[o * 3 + 1] = palette[l * 3 + 1]; out_rgb[o * 3 + 2] = palette[l * 3 + 2];
  }
}

// ---- host: single-linkage tree -> condensed tree -> EOM (+ epsilon) selection -> labels (scikit-learn 1.9 semantics)
struct Hierarchy {
  std::vector<int64_t> left, right, size;
  std::vector<double> value;
};

struct Condensed {           // rows of the condensed tree, in the order they are produced
  std::vector<int64_t> parent, child, size;
  std::vector<double> lambda;
};

static void bfs_hierarchy(const Hierarchy& h, int64_t n, int64_t root, std::vector<int64_t>& out) {
  out.clear();
  out.push_back(root);
  for (size_t head = 0; head < out.size(); ++head) {
    const int64_t x = out[head];
    if (x >= n) { out.push_back(h.left[x - n]); out.push_back(h.right[x - n]); }
  }
}

static int64_t node_size(const Hierarchy& h, int64_t n, int64_t x) { return x >= n ? h.size[x - n] : 1; }

}  // namespace iggt

using namespace iggt;

extern "C" int iggt_cluster_morton(const float* feats8, int64_t n, const float* lo, const float* hi, int64_t* codes,
                                   iggt_stream_t stream) {
  if (!feats8 || !lo || !hi || !codes || n <= 0) return -1;
  cl_morton_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(feats8, n, lo, hi, codes);
  return (int)cudaGetLastError();
}

extern "C" int iggt_cluster_reorder(const float* feats8, const int64_t* order, int64_t n, float* sorted8, int32_t* orig,
                                    float* box, iggt_stream_t stream) {
  if (!feats8 || !order || !sorted8 || !orig || !box || n <= 0 || n >= (1LL << 31)) return -1;
  const unsigned nb = static_cast<unsigned>((n + CL_TILE - 1) / CL_TILE);
  cl_reorder_kernel<<<nb, CL_TILE, 0, (cudaStream_t)stream>>>(feats8, order, n, reinterpret_cast<float4*>(sorted8), orig,
                                                              box);
  return (int)cudaGetLastError();
}

extern "C" int iggt_cluster_core(const float* sorted8, const float* box, int64_t n, int k, float* core2,
                                 iggt_stream_t stream) {
  if (!sorted8 || !box || !core2 || n <= 0 || n >= (1LL << 31) || k < 1 || k > CL_KMAX || k >= n) return -1;
  const size_t smem = static_cast<size_t>(k) * CL_CTA * sizeof(float);
  const cudaError_t e = opt_in_smem<cl_core_kernel>(CL_KMAX * CL_CTA * sizeof(float));
  if (e != cudaSuccess) return (int)e;
  const int nb = static_cast<int>((n + CL_TILE - 1) / CL_TILE);
  cl_core_kernel<<<static_cast<unsigned>((n + CL_CTA - 1) / CL_CTA), CL_CTA, smem, (cudaStream_t)stream>>>(
      reinterpret_cast<const float4*>(sorted8), box, n, nb, k, core2);
  return (int)cudaGetLastError();
}

namespace {
struct MstWorkspace {
  unsigned long long* key1; int32_t* comp; int32_t* parent; uint32_t* key2; float* qw2; int32_t* qj;
  int32_t* pick_i; int32_t* pick_j; int32_t* tcomp; float* tcore; uint32_t* counters;
};
int64_t mst_workspace(int64_t n, char* base, MstWorkspace* w) {
  const int64_t nb = (n + CL_TILE - 1) / CL_TILE;
  int64_t off = 0;
  auto take = [&](int64_t bytes) { char* p = base ? base + off : nullptr; off += (bytes + 255) / 256 * 256; return p; };
  MstWorkspace t;
  t.key1 = reinterpret_cast<unsigned long long*>(take(n * 8));
  t.comp = reinterpret_cast<int32_t*>(take(n * 4));
  t.parent = reinterpret_cast<int32_t*>(take(n * 4));
  t.key2 = reinterpret_cast<uint32_t*>(take(n * 4));
  t.qw2 = reinterpret_cast<float*>(take(n * 4));
  t.qj = reinterpret_cast<int32_t*>(take(n * 4));
  t.pick_i = reinterpret_cast<int32_t*>(take(n * 4));
  t.pick_j = reinterpret_cast<int32_t*>(take(n * 4));
  t.tcomp = reinterpret_cast<int32_t*>(take(nb * 4));
  t.tcore = reinterpret_cast<float*>(take(nb * 4));
  t.counters = reinterpret_cast<uint32_t*>(take(16));
  if (w) *w = t;
  return off;
}
}  // namespace

extern "C" int iggt_cluster_mst_workspace(int64_t n, int64_t* bytes) {
  if (n <= 0 || !bytes) return -1;
  *bytes = mst_workspace(n, nullptr, nullptr);
  return 0;
}

extern "C" int iggt_cluster_mst(const float* sorted8, const float* box, const int32_t* orig, const float* core2,
                                int64_t n, void* workspace, int32_t* edge_a, int32_t* edge_b, float* edge_w2,
                                int32_t* rounds, iggt_stream_t stream) {
  if (!sorted8 || !box || !orig || !core2 || !workspace || !edge_a || !edge_b || !edge_w2 || n < 2 ||
      n >= (1LL << 31))
    return -1;
  cudaStream_t st = (cudaStream_t)stream;
  MstWorkspace w;
  mst_workspace(n, static_cast<char*>(workspace), &w);
  const int nb = static_cast<int>((n + CL_TILE - 1) / CL_TILE);
  const unsigned g256 = static_cast<unsigned>((n + 255) / 256), gs = static_cast<unsigned>((n + CL_CTA - 1) / CL_CTA);
  const float4* s4 = reinterpret_cast<const float4*>(sorted8);
  cl_mst_init_kernel<<<g256, 256, 0, st>>>(n, w.comp, w.parent, w.key1, w.key2, w.pick_i);
  cudaMemsetAsync(w.counters, 0, 16, st);
  uint32_t host[2] = {0, 0};
  int r = 0;
  for (; r < 64 && host[0] < static_cast<uint32_t>(n - 1); ++r) {
    cl_tile_info_kernel<<<nb, CL_TILE, 0, st>>>(w.comp, core2, n, w.tcomp, w.tcore);
    cl_boruvka_search_kernel<<<gs, CL_CTA, 0, st>>>(s4, box, n, nb, w.comp, core2, orig, w.tcomp, w.tcore, w.key1, w.qw2,
                                                    w.qj);
    cl_boruvka_pick_kernel<<<g256, 256, 0, st>>>(n, w.comp, orig, w.qw2, w.qj, w.key1, w.key2);
    cl_boruvka_select_kernel<<<g256, 256, 0, st>>>(n, w.comp, orig, w.qw2, w.qj, w.key1, w.key2, w.pick_i, w.pick_j);
    cl_boruvka_hook_kernel<<<g256, 256, 0, st>>>(n, w.comp, orig, w.pick_i, w.pick_j, w.key1, w.parent, w.counters,
                                                 edge_a, edge_b, edge_w2);
    int jumps = 0;
    do {                                                // pointer jumping until every root points at its final root
      if (++jumps > 64) return -3;                      // the hooks formed a cycle
      cudaMemsetAsync(w.counters + 1, 0, 4, st);
      cl_jump_kernel<<<g256, 256, 0, st>>>(n, w.comp, w.parent, w.counters + 1);
      cudaMemcpyAsync(host, w.counters, 8, cudaMemcpyDeviceToHost, st);
      const cudaError_t e = cudaStreamSynchronize(st);
      if (e != cudaSuccess) return (int)e;
    } while (host[1] != 0);
    cl_relabel_kernel<<<g256, 256, 0, st>>>(n, w.comp, w.parent, w.key1, w.key2, w.pick_i);
  }
  if (rounds) *rounds = r;
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return (int)e;
  return host[0] == static_cast<uint32_t>(n - 1) ? 0 : -2;
}

extern "C" int iggt_cluster_fill(const float* sorted8, const float* box, const int32_t* orig, const int32_t* label,
                                 int64_t n, int32_t* tile_count, const uint8_t* palette, int64_t* out_label,
                                 uint8_t* out_rgb, iggt_stream_t stream) {
  if (!sorted8 || !box || !orig || !label || !tile_count || !out_label || (out_rgb && !palette) || n <= 0 ||
      n >= (1LL << 31))
    return -1;
  cudaStream_t st = (cudaStream_t)stream;
  const int nb = static_cast<int>((n + CL_TILE - 1) / CL_TILE);
  cl_tile_count_kernel<<<nb, CL_TILE, 0, st>>>(label, n, tile_count);
  cl_fill_kernel<<<static_cast<unsigned>((n + CL_CTA - 1) / CL_CTA), CL_CTA, 0, st>>>(
      reinterpret_cast<const float4*>(sorted8), box, n, nb, orig, label, tile_count, palette, out_label, out_rgb);
  return (int)cudaGetLastError();
}

extern "C" int iggt_mst_orient(double* mst, int64_t n, int64_t root) {
  if (!mst || n < 2 || root < 0 || root >= n) return -1;
  const int64_t m = n - 1;
  std::vector<int64_t> start(n + 1, 0), adj(2 * m);
  for (int64_t i = 0; i < m; ++i) {
    const double fa = mst[i * 3], fb = mst[i * 3 + 1];
    if (!(fa >= 0 && fa < n && fb >= 0 && fb < n)) return -1;
    ++start[static_cast<int64_t>(fa) + 1];
    ++start[static_cast<int64_t>(fb) + 1];
  }
  for (int64_t v = 0; v < n; ++v) start[v + 1] += start[v];
  std::vector<int64_t> fill(start.begin(), start.end() - 1);
  for (int64_t i = 0; i < m; ++i) {
    const int64_t a = static_cast<int64_t>(mst[i * 3]), b = static_cast<int64_t>(mst[i * 3 + 1]);
    adj[fill[a]++] = b;
    adj[fill[b]++] = a;
  }
  std::vector<int64_t> depth(n, -1), queue;           // breadth-first from the root: depth in the tree
  queue.reserve(n);
  queue.push_back(root);
  depth[root] = 0;
  for (size_t h = 0; h < queue.size(); ++h) {
    const int64_t v = queue[h];
    for (int64_t e = start[v]; e < start[v + 1]; ++e)
      if (depth[adj[e]] < 0) { depth[adj[e]] = depth[v] + 1; queue.push_back(adj[e]); }
  }
  if (static_cast<int64_t>(queue.size()) != n) return -2;   // not a spanning tree
  for (int64_t i = 0; i < m; ++i) {
    const int64_t a = static_cast<int64_t>(mst[i * 3]), b = static_cast<int64_t>(mst[i * 3 + 1]);
    if (depth[a] > depth[b]) std::swap(mst[i * 3], mst[i * 3 + 1]);
  }
  return 0;
}

extern "C" int iggt_hdbscan_labels(const double* mst, int64_t n, int64_t min_cluster_size, double eps,
                                   int64_t* labels) {
  if (!mst || !labels || n < 2 || min_cluster_size < 2 || !(eps >= 0.0)) return -1;
  const int64_t m = n - 1;
  // 1. single-linkage tree: edge i (in the given order) joins the current trees of its endpoints into node n + i,
  //    the tree of the first endpoint on the left
  Hierarchy h;
  h.left.resize(m); h.right.resize(m); h.size.resize(m); h.value.resize(m);
  {
    std::vector<int64_t> uf(2 * n - 1), sz(2 * n - 1, 1);
    for (int64_t i = 0; i < 2 * n - 1; ++i) uf[i] = i;
    auto find = [&](int64_t x) {
      int64_t r = x;
      while (uf[r] != r) r = uf[r];
      while (uf[x] != r) { const int64_t nx = uf[x]; uf[x] = r; x = nx; }
      return r;
    };
    for (int64_t i = 0; i < m; ++i) {
      const double fa = mst[i * 3], fb = mst[i * 3 + 1];
      if (!(fa >= 0 && fa < n && fb >= 0 && fb < n)) return -1;
      const int64_t a = find(static_cast<int64_t>(fa)), b = find(static_cast<int64_t>(fb));
      if (a == b) return -2;                             // not a spanning tree
      h.left[i] = a; h.right[i] = b; h.value[i] = mst[i * 3 + 2];
      h.size[i] = sz[a] + sz[b];
      uf[a] = uf[b] = n + i;
      sz[n + i] = h.size[i];
    }
  }
  // 2. condensed tree: walk the hierarchy breadth first from the root; a split into two parts of at least
  //    min_cluster_size points makes two new clusters, a smaller part falls out of its cluster point by point
  //    (in breadth-first order of its subtree) at lambda = 1 / distance (inf at distance 0)
  const int64_t root = 2 * n - 2;
  Condensed ct;
  int64_t next_label = n + 1;
  {
    std::vector<int64_t> order, sub;
    bfs_hierarchy(h, n, root, order);
    std::vector<int64_t> relabel(root + 1, 0);
    std::vector<char> ignore(root + 1, 0);
    relabel[root] = n;
    auto emit = [&](int64_t p, int64_t c, double lam, int64_t s) {
      ct.parent.push_back(p); ct.child.push_back(c); ct.lambda.push_back(lam); ct.size.push_back(s);
    };
    auto fall_out = [&](int64_t sub_root, int64_t p, double lam) {
      bfs_hierarchy(h, n, sub_root, sub);
      for (int64_t x : sub) {
        if (x < n) emit(p, x, lam, 1);
        ignore[x] = 1;
      }
    };
    for (int64_t node : order) {
      if (ignore[node] || node < n) continue;
      const int64_t l = h.left[node - n], r = h.right[node - n];
      const double d = h.value[node - n];
      const double lam = d > 0.0 ? 1.0 / d : INFINITY;
      const int64_t lc = node_size(h, n, l), rc = node_size(h, n, r);
      const int64_t p = relabel[node];
      if (lc >= min_cluster_size && rc >= min_cluster_size) {
        relabel[l] = next_label++; emit(p, relabel[l], lam, lc);
        relabel[r] = next_label++; emit(p, relabel[r], lam, rc);
      } else if (lc < min_cluster_size && rc < min_cluster_size) {
        fall_out(l, p, lam);
        fall_out(r, p, lam);
      } else if (lc < min_cluster_size) {
        relabel[r] = p;
        fall_out(l, p, lam);
      } else {
        relabel[l] = p;
        fall_out(r, p, lam);
      }
    }
  }
  // 3. stability of every cluster: sum over its rows of (lambda - lambda at its birth) * size, in row order
  const int64_t nc = next_label - n;                     // clusters n .. next_label - 1; n is the root
  std::vector<double> birth(nc, 0.0), stab(nc, 0.0);
  std::vector<int64_t> cparent(nc, -1);
  std::vector<std::vector<int64_t>> kids(nc);            // cluster children, in row order
  const size_t rows = ct.parent.size();
  for (size_t i = 0; i < rows; ++i)
    if (ct.child[i] >= n) {
      birth[ct.child[i] - n] = ct.lambda[i];
      cparent[ct.child[i] - n] = ct.parent[i];
      kids[ct.parent[i] - n].push_back(ct.child[i]);
    }
  for (size_t i = 0; i < rows; ++i)
    stab[ct.parent[i] - n] += (ct.lambda[i] - birth[ct.parent[i] - n]) * static_cast<double>(ct.size[i]);
  // 4. excess of mass, children before parents (descending ids); the root is never a cluster
  std::vector<char> sel(nc, 0);
  for (int64_t c = nc - 1; c >= 1; --c) sel[c] = 1;
  for (int64_t c = nc - 1; c >= 1; --c) {
    double sub = 0.0;
    for (int64_t k : kids[c]) sub += stab[k - n];
    if (sub > stab[c]) {
      sel[c] = 0;
      stab[c] = sub;
    } else {
      std::vector<int64_t> q(kids[c].begin(), kids[c].end());
      for (size_t i = 0; i < q.size(); ++i) {
        sel[q[i] - n] = 0;
        for (int64_t k : kids[q[i] - n]) q.push_back(k);
      }
    }
  }
  // 5. epsilon: a selected cluster born below distance eps is replaced by its lowest ancestor born above eps, or by
  //    the ancestor just under the root.  Distances here are 1 / lambda, as in scikit-learn.
  if (eps != 0.0 && nc > 1) {
    std::vector<char> out(nc, 0);
    for (int64_t c = 1; c < nc; ++c) {
      if (!sel[c]) continue;
      if (1.0 / birth[c] < eps) {
        int64_t x = c;
        while (true) {
          const int64_t p = cparent[x] - n;
          if (p == 0) break;
          if (1.0 / birth[p] > eps) { x = p; break; }
          x = p;
        }
        out[x] = 1;
      } else {
        out[c] = 1;
      }
    }
    sel.swap(out);
  }
  // 6. labels: selected clusters numbered in increasing id order; a point takes the label of its nearest selected
  //    ancestor in the condensed tree, noise (-1) if there is none
  std::vector<int64_t> lab(nc, -1);
  int64_t next = 0;
  for (int64_t c = 1; c < nc; ++c) {
    if (sel[c]) lab[c] = next++;
    else lab[c] = lab[cparent[c] - n];                   // a parent always has a smaller id than its children
  }
  for (int64_t i = 0; i < n; ++i) labels[i] = -1;
  for (size_t i = 0; i < rows; ++i)
    if (ct.child[i] < n) labels[ct.child[i]] = lab[ct.parent[i] - n];
  return 0;
}
