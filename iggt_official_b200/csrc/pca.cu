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
#include "fpops.cuh"
#include "launch.cuh"

namespace iggt {

constexpr int PCA_CMIN = 3, PCA_CMAX = 8;
constexpr int PCA_TILE = 256;         // points per tile = threads per CTA of the moments and projection kernels
constexpr int PCA_MAX_CTAS = 1024;    // partial-sum slots in the basis workspace
constexpr int PCA_JACOBI_SWEEPS = 64;
constexpr int pca_nv(int c) { return c + c * (c + 1) / 2; }   // sums of d, then of d d^T (upper triangle, row-major)

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

// ---- rank and interpolation rules of the selection (IGGT_QRULE_* in the header), shared by the device selection and
// the host entry point iggt_quantile_rule, with one rounding per operation on both sides (fpops.cuh; fmaf below is an
// explicit, correctly rounded fma on both).
struct QsRank {
  int64_t lo, hi;                     // order statistics (0-based ranks among the `count` selected values)
  float w;                            // interpolation weight
};

// Ranks of quantile q among `count` > 0 values.
//   TORCH: torch.quantile, q in [0, 1]: r = q * float32(n - 1) in fp32, floor / ceil, w = r - floor (clamped to n - 1).
//   NUMPY, NUMPY_NAN: np.percentile / np.nanpercentile, method "linear", q in percent, as numpy 2.3 runs them for
//     float32 data: q / float32(100) in fp32 (percentile divides by a.dtype.type(100)); virtual index
//     v = float32(n - 1) * q in fp32 (n - 1 is a weak Python int); v >= n - 1 takes the last value twice with
//     w = v - (-1) (numpy's index -1); otherwise lo = floor(v), hi = float32(lo + 1) (both still fp32, so above 2^24
//     hi can round to lo or to lo + 2), w = v - lo.  hi is clamped to n - 1 where numpy would index past the end.
//   MEDIAN: np.median: the middle value, or the two middle values of an even count.
__host__ __device__ inline QsRank qs_rank(int rule, int64_t count, float q) {
  QsRank k;
  const int64_t last = count - 1;
  if (rule == IGGT_QRULE_TORCH) {
    const float r = fmul(q, static_cast<float>(last));
    const int64_t lo = static_cast<int64_t>(r), hi = static_cast<int64_t>(ceilf(r));
    k.lo = lo < last ? lo : last;                        // float32(n - 1) may round above n - 1 for n > 2^24
    k.hi = hi < last ? hi : last;
    k.w = fsub(r, static_cast<float>(lo));
  } else if (rule == IGGT_QRULE_MEDIAN) {
    k.lo = (count - 1) / 2;
    k.hi = count / 2;
    k.w = 0.f;
  } else {
    const float fl = static_cast<float>(last);
    const float v = fmul(fl, fdiv(q, 100.f));
    if (v >= fl) {
      k.lo = k.hi = last;
      k.w = fadd(v, 1.f);
    } else {
      const float lo = floorf(v), hi = fadd(lo, 1.f);
      k.lo = static_cast<int64_t>(lo);
      k.hi = static_cast<int64_t>(hi) < last ? static_cast<int64_t>(hi) : last;
      k.w = fsub(v, lo);
    }
  }
  return k;
}

// The quantile from the order statistics a (rank lo) and b (rank hi).
//   TORCH: ATen's lerp (Lerp.h): the small-weight and large-weight branches, each a single fma as nvcc contracts them.
//   NUMPY*: numpy's _lerp, no fma: d = b - a; a + d * w, or b - d * (1 - w) where w >= 0.5.
//   MEDIAN: np.mean of the middle value(s) in fp32: a, or (a + b) / 2.
__host__ __device__ inline float qs_interp(int rule, int64_t lo, int64_t hi, float a, float b, float w) {
  if (rule == IGGT_QRULE_TORCH)
    return fabsf(w) < 0.5f ? fmaf(w, fsub(b, a), a) : fmaf(-fsub(b, a), fsub(1.f, w), b);
  if (rule == IGGT_QRULE_MEDIAN) return lo == hi ? a : fdiv(fadd(a, b), 2.f);
  const float d = fsub(b, a);
  return w >= 0.5f ? fsub(b, fmul(d, fsub(1.f, w))) : fadd(a, fmul(d, w));
}

struct QsTargets {                    // one selection: two quantiles (floor and ceil rank of each = QS_SLOTS targets)
  float q[2];
  int rule;
  int nout;                           // quantiles written (1 or 2)
};
struct QsRow {                        // per-row selection state between passes
  uint32_t prefix[QS_SLOTS];          // distinct key prefixes still being refined
  int nslots;
  int slot[QS_SLOTS];                 // prefix slot of each target
  int64_t rank[QS_SLOTS];             // rank of each target within its prefix
  int64_t order[QS_SLOTS];            // rank of each target among the selected values
  float weight[2];
  int nan_out;                        // the row's result is NaN (a NaN the rule propagates, or nothing selected)
};

// Histogram of one digit of every key (pass 0: bits 31..21) or of the keys under a slot's prefix (pass 1: bits
// 20..10 under 11 bits, pass 2: bits 9..0 under 22 bits).  Grid (x, rows); each CTA strides over its row with 16-byte
// loads.  Counts go to shared memory (32 KB: pass 0 one copy per warp, later passes one per slot), then to hist.
template <int PASS>
__global__ void __launch_bounds__(QS_THREADS)
qs_hist_kernel(const float* __restrict__ y, int64_t n, int64_t ld, const uint8_t* __restrict__ mask, int64_t ldm,
               const QsRow* __restrict__ state, uint32_t* __restrict__ hist) {
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
  const uint8_t* m = mask ? mask + static_cast<int64_t>(row) * ldm : nullptr;
  auto count = [&](float f, int64_t i) {
    if (m && !m[i]) return;
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
  if (g < head) count(r[g], g);
  const int64_t nv = (n - head) / 4;
  const float4* r4 = reinterpret_cast<const float4*>(r + head);
#pragma unroll 4
  for (int64_t i = g; i < nv; i += stride) {
    const float4 v = __ldg(r4 + i);
    const int64_t e = head + 4 * i;
    count(v.x, e); count(v.y, e + 1); count(v.z, e + 2); count(v.w, e + 3);
  }
  for (int64_t i = head + 4 * nv + g; i < n; i += stride) count(r[i], i);
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
// pass's slots.  Pass 0 first counts the row's selected values (all bins; NaN keys sit in the last bin alone) and
// derives the target ranks from that count by qs_rank.  After pass 2 the keys are complete: qs_interp of the order
// statistics.
template <int PASS>
__global__ void __launch_bounds__(32)
qs_select_kernel(const uint32_t* __restrict__ hist, QsRow* __restrict__ state, QsTargets tg, float* __restrict__ out,
                 int64_t ldo, int64_t* __restrict__ count_out) {
  constexpr int BITS = PASS == 2 ? 10 : 11;
  constexpr int BINS = 1 << BITS;
  constexpr int PER_LANE = BINS / 32;
  const int row = blockIdx.x, lane = threadIdx.x;
  QsRow st;
  if (PASS == 0) {
    const uint32_t* h0 = hist + static_cast<int64_t>(row) * QS_SLOTS * QS_BINS;
    int64_t total = 0;
    for (int b = lane; b < QS_BINS; b += 32) total += h0[b];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) total += __shfl_xor_sync(0xffffffffu, total, o);
    const int64_t nans = h0[QS_BINS - 1];                // NaN keys only
    const int64_t count = tg.rule == IGGT_QRULE_NUMPY_NAN ? total - nans : total;
    st.nslots = 1;
    st.prefix[0] = 0;
    st.nan_out = count == 0 || (tg.rule != IGGT_QRULE_NUMPY_NAN && nans != 0);
    for (int q = 0; q < 2; ++q) {
      const QsRank k = count > 0 ? qs_rank(tg.rule, count, tg.q[q]) : QsRank{0, 0, 0.f};
      st.order[2 * q] = k.lo;
      st.order[2 * q + 1] = k.hi;
      st.weight[q] = k.w;
    }
#pragma unroll
    for (int i = 0; i < QS_SLOTS; ++i) { st.slot[i] = 0; st.rank[i] = st.order[i]; }
    if (count_out && lane == 0) count_out[row] = count;
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
    QsRow nx = st;
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
      const float r = st.nan_out ? __uint_as_float(0x7fc00000u)
                                 : qs_interp(tg.rule, st.order[2 * q], st.order[2 * q + 1], key_float(key[2 * q]),
                                             key_float(key[2 * q + 1]), st.weight[q]);
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

// The radix selection behind iggt_quantile and iggt_select: every row, one pair of quantiles per three passes.
static int qs_run(const float* y, int64_t rows, int64_t n, int64_t ld, const uint8_t* mask, int64_t ldm, int rule,
                  const float* q, int nq, void* workspace, float* out, int64_t* count, cudaStream_t st) {
  uint32_t* hist = static_cast<uint32_t*>(workspace);
  const int64_t hb = qs_hist_bytes(rows);
  QsRow* state = reinterpret_cast<QsRow*>(static_cast<char*>(workspace) + 3 * hb);
  const int64_t chunks = (n / 4 + QS_THREADS - 1) / QS_THREADS;
  const int gx = std::max<int64_t>(1, grid_for(reinterpret_cast<const void*>(qs_hist_kernel<0>), QS_THREADS,
                                               chunks * rows) / rows);
  const dim3 hgrid(static_cast<unsigned>(std::min<int64_t>(gx, std::max<int64_t>(chunks, 1))), static_cast<unsigned>(rows));
  const int R = static_cast<int>(rows);
  for (int q0 = 0; q0 < nq; q0 += 2) {
    QsTargets tg;
    tg.rule = rule;
    tg.nout = nq - q0 < 2 ? nq - q0 : 2;
    for (int i = 0; i < 2; ++i) tg.q[i] = q[q0 + (i < tg.nout ? i : 0)];
    cudaError_t e = cudaMemsetAsync(hist, 0, 3 * hb, st);
    if (e != cudaSuccess) return (int)e;
    qs_hist_kernel<0><<<hgrid, QS_THREADS, 0, st>>>(y, n, ld, mask, ldm, state, hist);
    qs_select_kernel<0><<<R, 32, 0, st>>>(hist, state, tg, out + q0, nq, q0 == 0 ? count : nullptr);
    qs_hist_kernel<1><<<hgrid, QS_THREADS, 0, st>>>(y, n, ld, mask, ldm, state, hist + hb / 4);
    qs_select_kernel<1><<<R, 32, 0, st>>>(hist + hb / 4, state, tg, out + q0, nq, nullptr);
    qs_hist_kernel<2><<<hgrid, QS_THREADS, 0, st>>>(y, n, ld, mask, ldm, state, hist + hb / 2);
    qs_select_kernel<2><<<R, 32, 0, st>>>(hist + hb / 2, state, tg, out + q0, nq, nullptr);
    e = cudaGetLastError();
    if (e != cudaSuccess) return (int)e;
  }
  return 0;
}

extern "C" int iggt_quantile(const float* y, int64_t rows, int64_t n, int64_t ld, const float* q, int nq,
                             void* workspace, float* out, iggt_stream_t stream) {
  if (!y || !q || !workspace || !out || rows <= 0 || rows > 65535 || n <= 0 || n >= (1LL << 32) || ld < n || nq <= 0)
    return -1;
  for (int i = 0; i < nq; ++i)
    if (!(q[i] >= 0.f && q[i] <= 1.f)) return -1;
  return qs_run(y, rows, n, ld, nullptr, 0, IGGT_QRULE_TORCH, q, nq, workspace, out, nullptr, (cudaStream_t)stream);
}

extern "C" int iggt_select(const float* y, int64_t rows, int64_t n, int64_t ld, const uint8_t* mask, int64_t ldm,
                           int rule, const float* q, int nq, void* workspace, float* out, int64_t* count,
                           iggt_stream_t stream) {
  if (!y || !workspace || !out || rows <= 0 || rows > 65535 || n <= 0 || n >= (1LL << 32) || ld < n ||
      (mask && ldm != 0 && ldm < n) || rule < IGGT_QRULE_TORCH || rule > IGGT_QRULE_MEDIAN)   // ldm 0: one shared row
    return -1;
  const float median_q = 0.f;
  if (rule == IGGT_QRULE_MEDIAN) {
    if (nq != 1) return -1;
    q = &median_q;
  } else {
    if (!q || nq <= 0) return -1;
    const float qmax = rule == IGGT_QRULE_TORCH ? 1.f : 100.f;
    for (int i = 0; i < nq; ++i)
      if (!(q[i] >= 0.f && q[i] <= qmax)) return -1;
  }
  return qs_run(y, rows, n, ld, mask, ldm, rule, q, nq, workspace, out, count, (cudaStream_t)stream);
}

extern "C" int iggt_quantile_rule(const float* sorted, int64_t count, int rule, float q, float* out) {
  if (!out || count < 0 || (count > 0 && !sorted) || rule < IGGT_QRULE_TORCH || rule > IGGT_QRULE_MEDIAN) return -1;
  if (rule != IGGT_QRULE_MEDIAN && !(q >= 0.f && q <= (rule == IGGT_QRULE_TORCH ? 1.f : 100.f))) return -1;
  int64_t nans = 0;                                      // NaNs sort last, as np.sort puts them
  while (nans < count && isnan(sorted[count - 1 - nans])) ++nans;
  const int64_t n = rule == IGGT_QRULE_NUMPY_NAN ? count - nans : count;
  if (n == 0 || (rule != IGGT_QRULE_NUMPY_NAN && nans != 0)) {
    *out = NAN;
    return 0;
  }
  const QsRank k = qs_rank(rule, n, q);
  *out = qs_interp(rule, k.lo, k.hi, sorted[k.lo], sorted[k.hi], k.w);
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
