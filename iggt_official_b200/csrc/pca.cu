// PCA feature colours on the device (demo.py:372 and :380 -> iggt/utils/misc.py:272-332 apply_pca_colormap, which
// runs torch.pca_lowrank and torch.quantile, on the host in the demo) and an exact sort-free quantile.
//
// Stages, all over x [n, C] fp32 with 3 <= C <= 8:
//   1. moments: one pass computes the sums of d = x - x[0] and of d d^T in fp64 (the shift by the first point avoids
//      cancellation for features far from the origin) and counts non-finite values.  Every CTA of a persistent grid
//      writes its partial sums; a one-CTA kernel adds them in CTA order.  No float atomics: a given input on a given
//      device always gives bit-identical sums.
//   2. basis: the same one-CTA kernel forms the sample covariance and decomposes it by cyclic Jacobi in fp64
//      (sym_eig_jacobi, host + device; iggt_sym_eig exposes the host build), so the basis never leaves the GPU.
//   3. projection: y[j, i] = sum_c x[i, c] V[c, j] in fp32, fmas in channel order, of the UNcentred points as the
//      reference projects them; y is [3, n].
//   4. quantiles: torch.quantile's linear interpolation, restated exactly, with the order statistics found by a
//      three-pass radix selection (11 + 11 + 10 bits) over the order-preserving 32-bit key of each float.  Every target
//      rank of every row is selected in the same passes; the histograms hold integer counts, so the result does not
//      depend on scheduling.  No sort, so no 2^24-element limit.
//   5. stretch: out[i, j] = clamp((y[j, i] - lo_j) / (hi_j - lo_j), 0, 1), or 0.5 where hi_j <= lo_j.
// Every stage is bandwidth-bound or tiny; no tensor cores.  The streaming kernels stage tiles of 256 points through
// shared memory with 16-byte loads, so the loads stay vectorised for any C.
#include <cuda_runtime.h>
#include <float.h>
#include <math.h>
#include <stdint.h>

#include <algorithm>

#include "../../include/iggt_b200.h"
#include "launch.cuh"

namespace iggt {

constexpr int PCA_CMIN = 3, PCA_CMAX = 8;
constexpr int PCA_TILE = 256;         // points per tile = threads per CTA of the moments and projection kernels
constexpr int PCA_MAX_CTAS = 1024;    // partial-sum slots in the basis workspace
constexpr int PCA_JACOBI_SWEEPS = 64;
constexpr int pca_nv(int c) { return c + c * (c + 1) / 2; }   // sums of d, then of d d^T (upper triangle, row-major)

// ---- fp64 with one rounding per operation on the host and on the device.  nvcc would contract a * b + c into an
// fma in device code; the intrinsics keep the device build operation for operation equal to the host build (whose
// x86-64 baseline target has no fma to contract into), so both give bit-identical eigenvectors.
__host__ __device__ __forceinline__ double dmul(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dmul_rn(a, b);
#else
  return a * b;
#endif
}
__host__ __device__ __forceinline__ double dadd(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dadd_rn(a, b);
#else
  return a + b;
#endif
}
__host__ __device__ __forceinline__ double dsub(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dsub_rn(a, b);
#else
  return a - b;
#endif
}
__host__ __device__ __forceinline__ double ddiv(double a, double b) {
#ifdef __CUDA_ARCH__
  return __ddiv_rn(a, b);
#else
  return a / b;
#endif
}
__host__ __device__ __forceinline__ double dsqrt(double a) {
#ifdef __CUDA_ARCH__
  return __dsqrt_rn(a);
#else
  return sqrt(a);
#endif
}

__host__ __device__ __forceinline__ void jacobi_sync() {
#ifdef __CUDA_ARCH__
  __syncwarp();
#endif
}

// Symmetric eigendecomposition of a [C, C] (row-major fp64, upper triangle read) by cyclic Jacobi rotations.
// A pair (p, q) is rotated unless |a_pq| <= eps * sqrt(|a_pp a_qq|) (then it is set to 0); the sweeps stop when one
// rotates nothing.  evals [C] descending (ties: lower index first); evecs [C, C] row-major, eigenvector j in column j,
// its largest-magnitude component positive (the first one if several tie).  a and v: [PCA_CMAX][PCA_CMAX] scratch.
// `lanes` threads of one warp (lane = 0 .. lanes - 1; the host runs 1) share the row / column updates of every
// rotation; each element gets the same operations whatever `lanes` is, so the device result is the host result.
// Lane 0 writes evals / evecs.  Returns the number of sweeps.
__host__ __device__ inline int sym_eig_jacobi(const double* a_in, int C, double* evals, double* evecs,
                                              double (*a)[PCA_CMAX], double (*v)[PCA_CMAX], int lane, int lanes) {
  for (int i = lane; i < C * C; i += lanes) {
    const int p = i / C, q = i % C;
    a[p][q] = p <= q ? a_in[p * C + q] : a_in[q * C + p];
    v[p][q] = p == q ? 1.0 : 0.0;
  }
  jacobi_sync();
  int sweep = 0;
  while (sweep < PCA_JACOBI_SWEEPS) {
    ++sweep;
    bool rotated = false;
    for (int p = 0; p < C - 1; ++p)
      for (int q = p + 1; q < C; ++q) {
        const double apq = a[p][q], app = a[p][p], aqq = a[q][q];
        jacobi_sync();                                   // every lane has read the pair before it changes
        if (apq == 0.0) continue;
        if (fabs(apq) <= dmul(DBL_EPSILON, dsqrt(dmul(fabs(app), fabs(aqq))))) {
          if (lane == 0) a[p][q] = a[q][p] = 0.0;
          jacobi_sync();
          continue;
        }
        // Golub & Van Loan's symmetric 2x2 Schur decomposition: J = [[c, s], [-s, c]] zeroes a_pq in J^T A J
        const double theta = ddiv(dsub(aqq, app), dmul(2.0, apq));
        double t = fabs(theta) > 1e150 ? ddiv(0.5, fabs(theta))
                                       : ddiv(1.0, dadd(fabs(theta), dsqrt(dadd(1.0, dmul(theta, theta)))));
        if (theta < 0.0) t = -t;
        const double c = ddiv(1.0, dsqrt(dadd(1.0, dmul(t, t)))), s = dmul(t, c);
        for (int k = lane; k < C; k += lanes) {          // columns p, q of A J
          const double akp = a[k][p], akq = a[k][q];
          a[k][p] = dsub(dmul(c, akp), dmul(s, akq));
          a[k][q] = dadd(dmul(s, akp), dmul(c, akq));
        }
        jacobi_sync();
        for (int k = lane; k < C; k += lanes) {          // rows p, q of J^T (A J)
          const double apk = a[p][k], aqk = a[q][k];
          a[p][k] = dsub(dmul(c, apk), dmul(s, aqk));
          a[q][k] = dadd(dmul(s, apk), dmul(c, aqk));
        }
        jacobi_sync();
        if (lane == 0) a[p][q] = a[q][p] = 0.0;
        for (int k = lane; k < C; k += lanes) {          // V J
          const double vkp = v[k][p], vkq = v[k][q];
          v[k][p] = dsub(dmul(c, vkp), dmul(s, vkq));
          v[k][q] = dadd(dmul(s, vkp), dmul(c, vkq));
        }
        jacobi_sync();
        rotated = true;
      }
    if (!rotated) break;
  }
  if (lane != 0) return sweep;
  int order[PCA_CMAX];
  for (int i = 0; i < C; ++i) order[i] = i;
  for (int i = 1; i < C; ++i)                            // stable insertion sort, descending
    for (int j = i; j > 0 && a[order[j - 1]][order[j - 1]] < a[order[j]][order[j]]; --j) {
      const int tmp = order[j]; order[j] = order[j - 1]; order[j - 1] = tmp;
    }
  for (int j = 0; j < C; ++j) {
    const int src = order[j];
    evals[j] = a[src][src];
    int kmax = 0;
    for (int k = 1; k < C; ++k)
      if (fabs(v[k][src]) > fabs(v[kmax][src])) kmax = k;
    const double sgn = v[kmax][src] < 0.0 ? -1.0 : 1.0;
    for (int k = 0; k < C; ++k) evecs[k * C + j] = sgn * v[k][src];
  }
  return sweep;
}

// Tiles of 256 points staged in shared memory, double-buffered through registers: fetch() puts the 16-byte loads of a
// whole tile in flight (x 16-byte aligned: a tile starts at a multiple of 256*C floats), store() writes them to
// tile[0 .. cnt*C) between two barriers - by then the caller has fetched the next tile.  The last, partial tile is
// loaded float by float inside store().
template <int C>
struct TileLoader {
  static constexpr int NV4 = PCA_TILE * C / 4, PER = (NV4 + PCA_TILE - 1) / PCA_TILE;
  float4 r[PER];
  __device__ __forceinline__ void fetch(const float* __restrict__ x, int64_t n, int64_t tl, bool vec) {
    if (!vec || (tl + 1) * PCA_TILE > n) return;
    const float4* s4 = reinterpret_cast<const float4*>(x + tl * PCA_TILE * C);
#pragma unroll
    for (int k = 0; k < PER; ++k)
      if (threadIdx.x + k * PCA_TILE < NV4) r[k] = __ldg(s4 + threadIdx.x + k * PCA_TILE);
  }
  __device__ __forceinline__ int store(const float* __restrict__ x, int64_t n, int64_t tl, bool vec,
                                       float* __restrict__ tile) {
    const int64_t p0 = tl * PCA_TILE;
    const int cnt = static_cast<int>(n - p0 < PCA_TILE ? n - p0 : PCA_TILE);
    __syncthreads();                                     // the previous tile is consumed
    if (vec && cnt == PCA_TILE) {
#pragma unroll
      for (int k = 0; k < PER; ++k)
        if (threadIdx.x + k * PCA_TILE < NV4) reinterpret_cast<float4*>(tile)[threadIdx.x + k * PCA_TILE] = r[k];
    } else {
      for (int i = threadIdx.x; i < cnt * C; i += PCA_TILE) tile[i] = __ldg(x + p0 * C + i);
    }
    __syncthreads();
    return cnt;
  }
};

// Stage 1: per-CTA partial sums of d and d d^T (fp64) and of the non-finite count.
template <int C>
__global__ void __launch_bounds__(PCA_TILE, 1)
pca_moments_kernel(const float* __restrict__ x, int64_t n, bool vec, double* __restrict__ partial,
                   unsigned long long* __restrict__ partial_bad) {
  constexpr int NV = pca_nv(C);
  __shared__ __align__(16) float tile[PCA_TILE * C];
  __shared__ double red[PCA_TILE / 32][NV];
  __shared__ unsigned long long red_bad[PCA_TILE / 32];
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  float x0[C];
  double acc[NV];
#pragma unroll
  for (int c = 0; c < C; ++c) x0[c] = __ldg(x + c);
#pragma unroll
  for (int v = 0; v < NV; ++v) acc[v] = 0.0;
  unsigned bad = 0;                                      // < 2^26 per thread for n < 2^31
  const int64_t ntiles = (n + PCA_TILE - 1) / PCA_TILE;
  TileLoader<C> ld;
  if (blockIdx.x < ntiles) ld.fetch(x, n, blockIdx.x, vec);
  for (int64_t tl = blockIdx.x; tl < ntiles; tl += gridDim.x) {
    const int cnt = ld.store(x, n, tl, vec, tile);
    if (tl + gridDim.x < ntiles) ld.fetch(x, n, tl + gridDim.x, vec);
    if (t < cnt) {
      double d[C];
#pragma unroll
      for (int c = 0; c < C; ++c) {
        const float f = tile[t * C + c];
        bad += isfinite(f) ? 0 : 1;
        d[c] = static_cast<double>(f) - static_cast<double>(x0[c]);
        acc[c] += d[c];
      }
      int m = C;
#pragma unroll
      for (int c = 0; c < C; ++c)
#pragma unroll
        for (int k = c; k < C; ++k) acc[m++] += d[c] * d[k];
    }
  }
  // fixed-order reduction: a butterfly within each warp, then the warps in order
#pragma unroll
  for (int v = 0; v < NV; ++v)
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc[v] += __shfl_xor_sync(0xffffffffu, acc[v], o);
  const unsigned long long warp_bad = __reduce_add_sync(0xffffffffu, bad);
  if (lane == 0) {
#pragma unroll
    for (int v = 0; v < NV; ++v) red[warp][v] = acc[v];
    red_bad[warp] = warp_bad;
  }
  __syncthreads();
  if (t < NV) {
    double s = red[0][t];
#pragma unroll
    for (int w = 1; w < PCA_TILE / 32; ++w) s += red[w][t];
    partial[static_cast<int64_t>(blockIdx.x) * NV + t] = s;
  } else if (t == NV) {
    unsigned long long s = 0;
#pragma unroll
    for (int w = 0; w < PCA_TILE / 32; ++w) s += red_bad[w];
    partial_bad[blockIdx.x] = s;
  }
}

// Stage 2 (one CTA): the partials in CTA order -> moments, covariance, Jacobi (one warp), V [C, 3] fp32.
template <int C>
__global__ void __launch_bounds__(64, 1)
pca_basis_kernel(int64_t n, const double* __restrict__ partial, const unsigned long long* __restrict__ partial_bad,
                 int nparts, double* __restrict__ moments, double* __restrict__ cov, double* __restrict__ evals,
                 double* __restrict__ evecs, float* __restrict__ V, int64_t* __restrict__ nonfinite) {
  constexpr int NV = pca_nv(C);
  __shared__ double mom[NV], a[C * C], ev[C], vec[C * C], work_a[PCA_CMAX][PCA_CMAX], work_v[PCA_CMAX][PCA_CMAX];
  __shared__ unsigned long long nbad;
  const int t = threadIdx.x;
  if (t < NV) {
    double s = 0.0;
    for (int b = 0; b < nparts; ++b) s += partial[static_cast<int64_t>(b) * NV + t];
    mom[t] = s;
    moments[t] = s;
  } else if (t == NV) {
    unsigned long long s = 0;
    for (int b = 0; b < nparts; ++b) s += partial_bad[b];
    nbad = s;
    *nonfinite = static_cast<int64_t>(s);
  }
  __syncthreads();
  if (t >= 32) return;
  // sample covariance (S2 - S1 S1^T / n) / (n - 1) of the shifted points (= that of the points); all zero when
  // there are non-finite values (the caller rejects the input) so that the rotations stay finite
  if (t == 0) {
    const double nn = static_cast<double>(n), den = static_cast<double>(n > 1 ? n - 1 : 1);
    int m = C;
    for (int c = 0; c < C; ++c)
      for (int k = c; k < C; ++k, ++m) {
        const double s = nbad ? 0.0 : ddiv(dsub(mom[m], ddiv(dmul(mom[c], mom[k]), nn)), den);
        a[c * C + k] = a[k * C + c] = s;
      }
    for (int i = 0; i < C * C; ++i) cov[i] = a[i];
  }
  __syncwarp();
  sym_eig_jacobi(a, C, ev, vec, work_a, work_v, t, 32);
  if (t != 0) return;
  for (int j = 0; j < C; ++j) evals[j] = ev[j];
  for (int i = 0; i < C * C; ++i) evecs[i] = vec[i];
  for (int c = 0; c < C; ++c)
    for (int j = 0; j < 3; ++j) V[c * 3 + j] = static_cast<float>(vec[c * C + j]);
}

// Stage 3: y[j, i] = sum_c x[i, c] V[c, j], fp32 fmas in channel order.
template <int C>
__global__ void __launch_bounds__(PCA_TILE)
pca_project_kernel(const float* __restrict__ x, int64_t n, bool vec, const float* __restrict__ V,
                   float* __restrict__ y, int64_t ldy) {
  __shared__ __align__(16) float tile[PCA_TILE * C];
  __shared__ float w[C][3];
  const int t = threadIdx.x;
  if (t < C * 3) w[t / 3][t % 3] = V[t];                 // store()'s first barrier publishes it
  const int64_t ntiles = (n + PCA_TILE - 1) / PCA_TILE;
  TileLoader<C> ld;
  if (blockIdx.x < ntiles) ld.fetch(x, n, blockIdx.x, vec);
  for (int64_t tl = blockIdx.x; tl < ntiles; tl += gridDim.x) {
    const int cnt = ld.store(x, n, tl, vec, tile);
    if (tl + gridDim.x < ntiles) ld.fetch(x, n, tl + gridDim.x, vec);
    if (t < cnt) {
      const int64_t i = tl * PCA_TILE + t;
#pragma unroll
      for (int j = 0; j < 3; ++j) {
        float acc = tile[t * C] * w[0][j];
#pragma unroll
        for (int c = 1; c < C; ++c) acc = __fmaf_rn(tile[t * C + c], w[c][j], acc);
        y[j * ldy + i] = acc;
      }
    }
  }
}

// Stage 5: out [n, 3] (flat: element f is point f / 3, channel f % 3) from y [3, n] and qv [3, 2] = (lo, hi) per
// row.  Four output elements per thread and 16-byte stores; the y reads of a warp cover three short runs.  The IEEE
// division is the same correctly rounded quotient torch's div kernel computes.
__device__ __forceinline__ float stretch1(float v, float lo, float hi) {
  return hi > lo ? fminf(fmaxf(__fdiv_rn(__fsub_rn(v, lo), __fsub_rn(hi, lo)), 0.f), 1.f) : 0.5f;
}
__global__ void __launch_bounds__(256)
pca_stretch_kernel(const float* __restrict__ y, int64_t n, int64_t ldy, const float* __restrict__ qv, bool vec,
                   float* __restrict__ out) {
  __shared__ float lohi[6];
  if (threadIdx.x < 6) lohi[threadIdx.x] = qv[threadIdx.x];
  __syncthreads();
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  const int64_t g = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  const int64_t nv = vec ? 3 * n / 4 : 0;
  for (int64_t i = g; i < nv; i += stride) {
    float r[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int64_t f = 4 * i + e, p = f / 3;
      const int j = static_cast<int>(f - 3 * p);
      r[e] = stretch1(__ldg(y + j * ldy + p), lohi[2 * j], lohi[2 * j + 1]);
    }
    reinterpret_cast<float4*>(out)[i] = make_float4(r[0], r[1], r[2], r[3]);
  }
  for (int64_t f = 4 * nv + g; f < 3 * n; f += stride) {
    const int64_t p = f / 3;
    const int j = static_cast<int>(f - 3 * p);
    out[f] = stretch1(__ldg(y + j * ldy + p), lohi[2 * j], lohi[2 * j + 1]);
  }
}

// ---- exact quantiles by radix selection
constexpr int QS_BINS = 2048;
constexpr int QS_SLOTS = 4;           // target ranks per row in one selection: floor and ceil of two q values
constexpr int QS_THREADS = 128;       // four warps: pass 0 gives each warp its own histogram

// Order-preserving key: a < b as floats <=> key(a) < key(b) (-0 just below +0); every NaN -> the largest key.
__device__ __forceinline__ uint32_t float_key(float f) {
  if (f != f) return 0xffffffffu;
  const uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float key_float(uint32_t k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

struct QsTargets {                    // one selection: QS_SLOTS target ranks, two quantiles
  int64_t rank[QS_SLOTS];             // targets 2i, 2i + 1 = floor and ceil rank of quantile i
  float weight[2];
  int nout;                           // quantiles written (1 or 2)
};
struct QsRow {                        // per-row selection state between passes
  uint32_t prefix[QS_SLOTS];          // distinct key prefixes still being refined
  int nslots;
  int slot[QS_SLOTS];                 // prefix slot of each target
  int64_t rank[QS_SLOTS];             // rank of each target within its prefix
  int has_nan;
};

// Histogram of one digit of every key (pass 0: bits 31..21) or of the keys under a slot's prefix (pass 1: bits
// 20..10 under 11 bits, pass 2: bits 9..0 under 22 bits).  Grid (x, rows); each CTA strides over its row with 16-byte
// loads.  Counts go to shared memory (32 KB: pass 0 one copy per warp, later passes one per slot), then to hist.
template <int PASS>
__global__ void __launch_bounds__(QS_THREADS)
qs_hist_kernel(const float* __restrict__ y, int64_t n, int64_t ld, const QsRow* __restrict__ state,
               uint32_t* __restrict__ hist) {
  __shared__ uint32_t h[QS_SLOTS][QS_BINS];
  const int row = blockIdx.y, t = threadIdx.x, warp = t >> 5;
  for (int i = t; i < QS_SLOTS * QS_BINS; i += QS_THREADS) (&h[0][0])[i] = 0;
  uint32_t pre[QS_SLOTS] = {0, 0, 0, 0};
  int ns = 1;
  if (PASS > 0) {
    ns = state[row].nslots;
#pragma unroll
    for (int s = 0; s < QS_SLOTS; ++s) pre[s] = state[row].prefix[s];
  }
  __syncthreads();
  auto count = [&](float f) {
    const uint32_t k = float_key(f);
    if (PASS == 0) {
      atomicAdd(&h[warp][k >> 21], 1u);
    } else {
      const uint32_t p = PASS == 1 ? k >> 21 : k >> 10;
      const uint32_t d = PASS == 1 ? (k >> 10) & 0x7ffu : k & 0x3ffu;
#pragma unroll
      for (int s = 0; s < QS_SLOTS; ++s)
        if (s < ns && p == pre[s]) atomicAdd(&h[s][d], 1u);
    }
  };
  const float* r = y + static_cast<int64_t>(row) * ld;
  const int64_t g = static_cast<int64_t>(blockIdx.x) * QS_THREADS + t;
  const int64_t stride = static_cast<int64_t>(gridDim.x) * QS_THREADS;
  const int64_t head = min(n, static_cast<int64_t>(((16 - (reinterpret_cast<uintptr_t>(r) & 15)) & 15) / 4));
  if (g < head) count(r[g]);
  const int64_t nv = (n - head) / 4;
  const float4* r4 = reinterpret_cast<const float4*>(r + head);
#pragma unroll 4
  for (int64_t i = g; i < nv; i += stride) {
    const float4 v = __ldg(r4 + i);
    count(v.x); count(v.y); count(v.z); count(v.w);
  }
  for (int64_t i = head + 4 * nv + g; i < n; i += stride) count(r[i]);
  __syncthreads();
  uint32_t* gh = hist + static_cast<int64_t>(row) * QS_SLOTS * QS_BINS;
  if (PASS == 0) {
    for (int b = t; b < QS_BINS; b += QS_THREADS) {
      const uint32_t s = h[0][b] + h[1][b] + h[2][b] + h[3][b];
      if (s) atomicAdd(gh + b, s);
    }
  } else {
    for (int i = t; i < ns * QS_BINS; i += QS_THREADS) {
      const uint32_t s = (&h[0][0])[i];
      if (s) atomicAdd(gh + i, s);
    }
  }
}

// One warp per row: the bin of every target rank in its slot's histogram; the refined prefixes become the next
// pass's slots.  After pass 2 the keys are complete: lerp of the floor / ceil order statistics, as ATen's lerp
// (Lerp.h) computes it - the small-weight and large-weight branches, each a single fma as nvcc contracts them.
template <int PASS>
__global__ void __launch_bounds__(32)
qs_select_kernel(const uint32_t* __restrict__ hist, QsRow* __restrict__ state, QsTargets tg, float* __restrict__ out,
                 int64_t ldo) {
  constexpr int BITS = PASS == 2 ? 10 : 11;
  constexpr int BINS = 1 << BITS;
  constexpr int PER_LANE = BINS / 32;
  const int row = blockIdx.x, lane = threadIdx.x;
  QsRow st;
  if (PASS == 0) {
    st.nslots = 1;
    st.prefix[0] = 0;
#pragma unroll
    for (int i = 0; i < QS_SLOTS; ++i) { st.slot[i] = 0; st.rank[i] = tg.rank[i]; }
    st.has_nan = hist[static_cast<int64_t>(row) * QS_SLOTS * QS_BINS + QS_BINS - 1] != 0;   // NaN keys only
  } else {
    st = state[row];
  }
  uint32_t key[QS_SLOTS];
  int64_t rank[QS_SLOTS];
  for (int i = 0; i < QS_SLOTS; ++i) {
    const int s = st.slot[i];
    const uint32_t* h = hist + (static_cast<int64_t>(row) * QS_SLOTS + s) * QS_BINS + lane * PER_LANE;
    uint32_t c[PER_LANE];
    int64_t local = 0;
#pragma unroll
    for (int b = 0; b < PER_LANE; ++b) { c[b] = h[b]; local += c[b]; }
    int64_t incl = local;                                // inclusive scan over the lanes
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int64_t u = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += u;
    }
    int64_t base = incl - local;
    const int64_t k = st.rank[i];
    const bool mine = k >= base && k < incl;
    int bin = 0;
    int64_t below = 0;
    bool found = !mine;
#pragma unroll
    for (int b = 0; b < PER_LANE; ++b) {
      if (!found && k < base + c[b]) { bin = lane * PER_LANE + b; below = base; found = true; }
      base += c[b];
    }
    const int src = __ffs(__ballot_sync(0xffffffffu, mine)) - 1;   // the rank lies in exactly one lane's bins
    bin = __shfl_sync(0xffffffffu, bin, src < 0 ? 0 : src);
    below = __shfl_sync(0xffffffffu, below, src < 0 ? 0 : src);
    key[i] = (PASS == 0 ? 0u : st.prefix[s] << BITS) | static_cast<uint32_t>(bin);
    rank[i] = k - below;
  }
  if (lane != 0) return;
  if (PASS < 2) {
    QsRow nx;
    nx.has_nan = st.has_nan;
    nx.nslots = 0;
    for (int i = 0; i < QS_SLOTS; ++i) {
      int s = 0;
      while (s < nx.nslots && nx.prefix[s] != key[i]) ++s;
      if (s == nx.nslots) nx.prefix[nx.nslots++] = key[i];
      nx.slot[i] = s;
      nx.rank[i] = rank[i];
    }
    state[row] = nx;
  } else {
    for (int q = 0; q < tg.nout; ++q) {
      float r;
      if (st.has_nan) {
        r = __uint_as_float(0x7fc00000u);
      } else {
        const float self = key_float(key[2 * q]), end = key_float(key[2 * q + 1]), w = tg.weight[q];
        r = fabsf(w) < 0.5f ? __fmaf_rn(w, __fsub_rn(end, self), self)
                            : __fmaf_rn(-__fsub_rn(end, self), __fsub_rn(1.f, w), end);
      }
      out[static_cast<int64_t>(row) * ldo + q] = r;
    }
  }
}

inline int grid_for(const void* kernel, int threads, int64_t work_ctas) {
  int per_sm = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, threads, 0) != cudaSuccess || per_sm < 1)
    per_sm = 1;
  const int64_t g = static_cast<int64_t>(device_sm_count()) * per_sm;
  return static_cast<int>(work_ctas < g ? (work_ctas > 0 ? work_ctas : 1) : g);
}

template <int C>
int pca_basis_launch(const float* x, int64_t n, void* workspace, double* moments, double* cov, double* evals,
                     double* evecs, float* V, int64_t* nonfinite, cudaStream_t st) {
  const bool vec = (reinterpret_cast<uintptr_t>(x) & 15) == 0;
  int grid = grid_for(reinterpret_cast<const void*>(pca_moments_kernel<C>), PCA_TILE, (n + PCA_TILE - 1) / PCA_TILE);
  if (grid > PCA_MAX_CTAS) grid = PCA_MAX_CTAS;
  double* partial = static_cast<double*>(workspace);
  unsigned long long* bad = reinterpret_cast<unsigned long long*>(partial + static_cast<int64_t>(PCA_MAX_CTAS) * pca_nv(C));
  pca_moments_kernel<C><<<grid, PCA_TILE, 0, st>>>(x, n, vec, partial, bad);
  pca_basis_kernel<C><<<1, 64, 0, st>>>(n, partial, bad, grid, moments, cov, evals, evecs, V, nonfinite);
  return (int)cudaGetLastError();
}

template <int C>
int pca_project_launch(const float* x, int64_t n, const float* V, float* y, int64_t ldy, cudaStream_t st) {
  const bool vec = (reinterpret_cast<uintptr_t>(x) & 15) == 0;
  const int grid = grid_for(reinterpret_cast<const void*>(pca_project_kernel<C>), PCA_TILE, (n + PCA_TILE - 1) / PCA_TILE);
  pca_project_kernel<C><<<grid, PCA_TILE, 0, st>>>(x, n, vec, V, y, ldy);
  return (int)cudaGetLastError();
}

constexpr int64_t qs_hist_bytes(int64_t rows) { return rows * QS_SLOTS * QS_BINS * 4; }

}  // namespace iggt

using namespace iggt;

extern "C" int iggt_sym_eig(const double* a, int C, double* evals, double* evecs) {
  if (!a || !evals || !evecs || C < 1 || C > PCA_CMAX) return -1;
  for (int i = 0; i < C * C; ++i)
    if (!isfinite(a[i])) return -1;
  double work_a[PCA_CMAX][PCA_CMAX], work_v[PCA_CMAX][PCA_CMAX];
  sym_eig_jacobi(a, C, evals, evecs, work_a, work_v, 0, 1);
  return 0;
}

extern "C" int iggt_pca_basis_workspace(int C, int64_t* bytes) {
  if (!bytes || C < PCA_CMIN || C > PCA_CMAX) return -1;
  *bytes = static_cast<int64_t>(PCA_MAX_CTAS) * (pca_nv(C) + 1) * 8;
  return 0;
}

extern "C" int iggt_pca_basis(const float* x, int64_t n, int C, void* workspace, double* moments, double* cov,
                              double* evals, double* evecs, float* V, int64_t* nonfinite, iggt_stream_t stream) {
  if (!x || !workspace || !moments || !cov || !evals || !evecs || !V || !nonfinite || n <= 0) return -1;
  cudaStream_t st = (cudaStream_t)stream;
  switch (C) {
    case 3: return pca_basis_launch<3>(x, n, workspace, moments, cov, evals, evecs, V, nonfinite, st);
    case 4: return pca_basis_launch<4>(x, n, workspace, moments, cov, evals, evecs, V, nonfinite, st);
    case 5: return pca_basis_launch<5>(x, n, workspace, moments, cov, evals, evecs, V, nonfinite, st);
    case 6: return pca_basis_launch<6>(x, n, workspace, moments, cov, evals, evecs, V, nonfinite, st);
    case 7: return pca_basis_launch<7>(x, n, workspace, moments, cov, evals, evecs, V, nonfinite, st);
    case 8: return pca_basis_launch<8>(x, n, workspace, moments, cov, evals, evecs, V, nonfinite, st);
    default: return -1;
  }
}

extern "C" int iggt_pca_project(const float* x, int64_t n, int C, const float* V, float* y, int64_t ldy,
                                iggt_stream_t stream) {
  if (!x || !V || !y || n <= 0 || ldy < n) return -1;
  cudaStream_t st = (cudaStream_t)stream;
  switch (C) {
    case 3: return pca_project_launch<3>(x, n, V, y, ldy, st);
    case 4: return pca_project_launch<4>(x, n, V, y, ldy, st);
    case 5: return pca_project_launch<5>(x, n, V, y, ldy, st);
    case 6: return pca_project_launch<6>(x, n, V, y, ldy, st);
    case 7: return pca_project_launch<7>(x, n, V, y, ldy, st);
    case 8: return pca_project_launch<8>(x, n, V, y, ldy, st);
    default: return -1;
  }
}

extern "C" int iggt_quantile_workspace(int64_t rows, int64_t* bytes) {
  if (!bytes || rows <= 0 || rows > 65535) return -1;
  *bytes = 3 * qs_hist_bytes(rows) + rows * static_cast<int64_t>(sizeof(QsRow));
  return 0;
}

extern "C" int iggt_quantile(const float* y, int64_t rows, int64_t n, int64_t ld, const float* q, int nq,
                             void* workspace, float* out, iggt_stream_t stream) {
  if (!y || !q || !workspace || !out || rows <= 0 || rows > 65535 || n <= 0 || n >= (1LL << 32) || ld < n || nq <= 0)
    return -1;
  for (int i = 0; i < nq; ++i)
    if (!(q[i] >= 0.f && q[i] <= 1.f)) return -1;
  cudaStream_t st = (cudaStream_t)stream;
  uint32_t* hist = static_cast<uint32_t*>(workspace);
  const int64_t hb = qs_hist_bytes(rows);
  QsRow* state = reinterpret_cast<QsRow*>(static_cast<char*>(workspace) + 3 * hb);
  const int64_t chunks = (n / 4 + QS_THREADS - 1) / QS_THREADS;
  const int gx = std::max<int64_t>(1, grid_for(reinterpret_cast<const void*>(qs_hist_kernel<0>), QS_THREADS,
                                               chunks * rows) / rows);
  const dim3 hgrid(static_cast<unsigned>(std::min<int64_t>(gx, std::max<int64_t>(chunks, 1))), static_cast<unsigned>(rows));
  const int R = static_cast<int>(rows);
  for (int q0 = 0; q0 < nq; q0 += 2) {
    // torch.quantile: rank = float32(q) * float32(n - 1) in fp32; floor / ceil order statistics; weight = rank - floor
    QsTargets tg;
    tg.nout = nq - q0 < 2 ? nq - q0 : 2;
    for (int i = 0; i < 2; ++i) {
      const float r = q[q0 + (i < tg.nout ? i : 0)] * static_cast<float>(n - 1);
      const int64_t lo = static_cast<int64_t>(r), hi = static_cast<int64_t>(ceilf(r));
      tg.rank[2 * i] = lo < n - 1 ? lo : n - 1;          // float32(n - 1) may round above n - 1 for n > 2^24
      tg.rank[2 * i + 1] = hi < n - 1 ? hi : n - 1;
      tg.weight[i] = r - static_cast<float>(lo);
    }
    cudaError_t e = cudaMemsetAsync(hist, 0, 3 * hb, st);
    if (e != cudaSuccess) return (int)e;
    qs_hist_kernel<0><<<hgrid, QS_THREADS, 0, st>>>(y, n, ld, state, hist);
    qs_select_kernel<0><<<R, 32, 0, st>>>(hist, state, tg, out + q0, nq);
    qs_hist_kernel<1><<<hgrid, QS_THREADS, 0, st>>>(y, n, ld, state, hist + hb / 4);
    qs_select_kernel<1><<<R, 32, 0, st>>>(hist + hb / 4, state, tg, out + q0, nq);
    qs_hist_kernel<2><<<hgrid, QS_THREADS, 0, st>>>(y, n, ld, state, hist + hb / 2);
    qs_select_kernel<2><<<R, 32, 0, st>>>(hist + hb / 2, state, tg, out + q0, nq);
    e = cudaGetLastError();
    if (e != cudaSuccess) return (int)e;
  }
  return 0;
}

extern "C" int iggt_pca_stretch(const float* y, int64_t n, int64_t ldy, const float* qv, float* out,
                                iggt_stream_t stream) {
  if (!y || !qv || !out || n <= 0 || ldy < n) return -1;
  const bool vec = (reinterpret_cast<uintptr_t>(y) & 15) == 0 && (ldy & 3) == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0;
  const int grid = grid_for(reinterpret_cast<const void*>(pca_stretch_kernel), 256, (n / 4 + 255) / 256);
  pca_stretch_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(y, n, ldy, qv, vec, out);
  return (int)cudaGetLastError();
}
