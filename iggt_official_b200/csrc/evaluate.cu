// Scene evaluation on the device (iggt/metrics.py:257-671, run per frame in numpy by demo.py:145-163) and the
// ground-truth depth helpers (iggt/datasets/utils/misc.py:488-541 threshold_depth_map, iggt/utils/geometry.py:238-268).
//
//   resize:   nearest-neighbour [S, Hi, Wi] -> [S, Ho, Wo] with scipy.ndimage.zoom(order=0, grid_mode=True)'s index
//             map, which skimage.transform.resize(order=0) runs (zoom_nearest_index, host + device).
//   metrics:  one pass per frame over (gt, pred, mask) restating the reference's fp32 per-pixel arithmetic; fp64 sums,
//             per-CTA partials added in CTA order by a second kernel (no float atomics: bit-identical on repeated
//             calls).  Least-squares alignment runs the same scheme once more before, for sum g p and sum p^2.
//   poses:    fp64 translation norm and scipy's rotation magnitude (pose_errors, host + device).
//   threshold / camera coordinates: elementwise.
// The medians and percentiles come from the radix selection in pca.cu (iggt_select).
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include <algorithm>

#include "../../include/iggt_b200.h"
#include "fpops.cuh"
#include "launch.cuh"

namespace iggt {

constexpr int EV_THREADS = 256;
constexpr int EV_MAX_CTAS = 128;       // partial-sum slots per frame
constexpr int EV_NM = 10;              // metric sums (record fields 0..9)
constexpr int EV_NL = 2;               // least-squares sums

// scipy's ni_interpolation.c (NI_ZoomShift, grid_mode, order 0): cc = (k + 0.5) * zoom - 0.5 with
// zoom = n_in / n_out, source = floor(cc + 0.5).  cc stays inside (-0.5, n_in - 0.5), where every boundary mode
// leaves the index as it is; the clamp only guards the last bit.
__host__ __device__ inline int zoom_nearest_index(int k, int n_in, int n_out) {
  const double z = ddiv(static_cast<double>(n_in), static_cast<double>(n_out));
  const double cc = dsub(dmul(dadd(static_cast<double>(k), 0.5), z), 0.5);
  const double s = floor(dadd(cc, 0.5));
  return s < 0.0 ? 0 : (s > n_in - 1 ? n_in - 1 : static_cast<int>(s));
}

__global__ void __launch_bounds__(256)
resize_nearest_kernel(const float* __restrict__ src, int Hi, int Wi, float* __restrict__ dst, int Ho, int Wo) {
  const int s = blockIdx.y;
  const int64_t n = static_cast<int64_t>(Ho) * Wo;
  const float* in = src + static_cast<int64_t>(s) * Hi * Wi;
  float* out = dst + static_cast<int64_t>(s) * n;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int y = static_cast<int>(i / Wo), x = static_cast<int>(i - static_cast<int64_t>(y) * Wo);
    out[i] = __ldg(in + static_cast<int64_t>(zoom_nearest_index(y, Hi, Ho)) * Wi + zoom_nearest_index(x, Wi, Wo));
  }
}

__global__ void __launch_bounds__(256)
valid_mask_kernel(const float* __restrict__ gt, const float* __restrict__ pred, int64_t total, int sparse,
                  uint8_t* __restrict__ mask) {
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x)
    mask[i] = __ldg(gt + i) > 0.f && (!sparse || __ldg(pred + i) != 0.f);
}

// Fixed-order CTA reduction of NF per-thread sums: a butterfly within each warp, then the warps in order.
template <int NF>
__device__ __forceinline__ void cta_partials(double (&acc)[NF], double* __restrict__ out) {
  __shared__ double red[EV_THREADS / 32][NF];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int f = 0; f < NF; ++f)
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc[f] += __shfl_xor_sync(0xffffffffu, acc[f], o);
  if (lane == 0)
#pragma unroll
    for (int f = 0; f < NF; ++f) red[warp][f] = acc[f];
  __syncthreads();
  if (threadIdx.x < NF) {
    double s = red[0][threadIdx.x];
#pragma unroll
    for (int w = 1; w < EV_THREADS / 32; ++w) s += red[w][threadIdx.x];
    out[threadIdx.x] = s;
  }
}

// Least-squares sums over the mask: gt * pred and pred ** 2, fp32 products as numpy forms them.
__global__ void __launch_bounds__(EV_THREADS)
lsq_sums_kernel(const float* __restrict__ gt, const float* __restrict__ pred, const uint8_t* __restrict__ mask,
                int64_t n, double* __restrict__ partial) {
  const int s = blockIdx.y;
  const int64_t off = static_cast<int64_t>(s) * n;
  double acc[EV_NL] = {0.0, 0.0};
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * EV_THREADS + threadIdx.x; i < n;
       i += static_cast<int64_t>(gridDim.x) * EV_THREADS) {
    if (!mask[off + i]) continue;
    const float g = __ldg(gt + off + i), p = __ldg(pred + off + i);
    acc[0] += static_cast<double>(__fmul_rn(g, p));
    acc[1] += static_cast<double>(__fmul_rn(p, p));
  }
  cta_partials<EV_NL>(acc, partial + (static_cast<int64_t>(s) * gridDim.x + blockIdx.x) * EV_NL);
}

// One thread per (frame, field): the partials of the frame's CTAs in CTA order -> out[s * ldo + f].
__global__ void reduce_partials_kernel(const double* __restrict__ partial, int nblk, int nf, int S,
                                       double* __restrict__ out, int ldo) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= S * nf) return;
  const int s = t / nf, f = t - s * nf;
  double acc = 0.0;
  for (int b = 0; b < nblk; ++b) acc += partial[(static_cast<int64_t>(s) * nblk + b) * nf + f];
  out[static_cast<int64_t>(s) * ldo + f] = acc;
}

// Per frame: the ratio (record fields 10..13), metrics.py:328-357.
__global__ void align_scale_kernel(int alignment, const float* __restrict__ medians, int S, double* __restrict__ rec) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= S) return;
  double* r = rec + static_cast<int64_t>(s) * IGGT_EVAL_RECORD;
  float ratio = 1.f;
  bool ok = false;
  if (alignment == IGGT_ALIGN_MEDIAN) {
    const float g = medians[s], p = medians[S + s];
    ratio = __fdiv_rn(g, p);
    ok = isfinite(ratio);
    r[12] = g;
    r[13] = p;
  } else if (alignment == IGGT_ALIGN_LSQ) {                // r[12], r[13] hold the two sums
    ratio = static_cast<float>(__ddiv_rn(r[12], r[13]));
    ok = isfinite(ratio) && ratio > 0.f;
  } else {
    r[12] = r[13] = 0.0;
  }
  r[10] = ok ? ratio : 1.0;
  r[11] = ok ? 1.0 : 0.0;
}

// The aligned / clipped prediction and the metric sums of one frame per grid row.
__global__ void __launch_bounds__(EV_THREADS)
depth_metrics_kernel(const float* __restrict__ gt, const float* __restrict__ pred, const uint8_t* __restrict__ mask,
                     int64_t n, const double* __restrict__ rec, int clip, float clip_lo, float clip_hi, int sparse,
                     float* __restrict__ aligned, double* __restrict__ partial) {
  const int s = blockIdx.y;
  const int64_t off = static_cast<int64_t>(s) * n;
  const bool apply = rec[static_cast<int64_t>(s) * IGGT_EVAL_RECORD + 11] != 0.0;
  const float ratio = static_cast<float>(rec[static_cast<int64_t>(s) * IGGT_EVAL_RECORD + 10]);
  const float miss = static_cast<float>(1.03 + 1.0);     // nan_to_num(gt / pred, nan=thresh + 1, ...)
  double acc[EV_NM];
#pragma unroll
  for (int f = 0; f < EV_NM; ++f) acc[f] = 0.0;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * EV_THREADS + threadIdx.x; i < n;
       i += static_cast<int64_t>(gridDim.x) * EV_THREADS) {
    const float p0 = __ldg(pred + off + i);
    float p = apply ? __fmul_rn(p0, ratio) : p0;
    if (clip) {
      if (!isnan(p)) p = fminf(fmaxf(p, clip_lo), clip_hi);
      p = __fmul_rn(p, (!sparse || p0 != 0.f) ? 1.f : 0.f);
    }
    if (aligned) aligned[off + i] = p;
    if (!mask[off + i]) continue;
    acc[0] += 1.0;
    if (sparse && p == 0.f) continue;
    const float g = __ldg(gt + off + i);
    acc[1] += 1.0;
    const float rel = __fdiv_rn(fabsf(__fsub_rn(p, g)), g);
    acc[2] += isfinite(rel) ? static_cast<double>(rel) : 0.0;
    const float gp = __fdiv_rn(g, p), pg = __fdiv_rn(p, g);
    const float r1 = isfinite(gp) ? gp : miss, r2 = isfinite(pg) ? pg : 0.f;
    const float mx = fmaxf(r1, r2);
    acc[3] += (0.f < mx && mx < 1.03f) ? 1.0 : 0.0;
    const float d = __fsub_rn(g, p);
    acc[4] += static_cast<double>(fabsf(d));
    acc[5] += static_cast<double>(__fmul_rn(d, d));
    const float rr = (isnan(gp) || isnan(pg)) ? gp + pg : fmaxf(gp, pg);   // np.maximum propagates NaN
    if (isfinite(rr)) {
      acc[6] += 1.0;
      acc[7] += rr < 1.25f ? 1.0 : 0.0;
      acc[8] += rr < 1.5625f ? 1.0 : 0.0;
      acc[9] += rr < 1.953125f ? 1.0 : 0.0;
    }
  }
  cta_partials<EV_NM>(acc, partial + (static_cast<int64_t>(s) * gridDim.x + blockIdx.x) * EV_NM);
}

// ---- poses
__host__ __device__ inline double det3(const double (&m)[3][3]) {
  return dadd(dsub(dmul(m[0][0], dsub(dmul(m[1][1], m[2][2]), dmul(m[1][2], m[2][1]))),
                   dmul(m[0][1], dsub(dmul(m[1][0], m[2][2]), dmul(m[1][2], m[2][0])))),
              dmul(m[0][2], dsub(dmul(m[1][0], m[2][1]), dmul(m[1][1], m[2][0]))));
}

// Orthogonal polar factor of m (det > 0) by the scaled Newton iteration X <- (g X + X^-T / g) / 2, g = |det X|^-1/3;
// it equals scipy's U V^T of the SVD to rounding.
__host__ __device__ inline void polar3(double (&m)[3][3]) {
  for (int it = 0; it < 100; ++it) {
    const double det = det3(m);
    const double g = pow(fabs(det), -1.0 / 3.0);
    double cof[3][3];                                    // X^-T = cofactor(X) / det
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) {
        const int i1 = (i + 1) % 3, i2 = (i + 2) % 3, j1 = (j + 1) % 3, j2 = (j + 2) % 3;
        cof[i][j] = dsub(dmul(m[i1][j1], m[i2][j2]), dmul(m[i1][j2], m[i2][j1]));
      }
    double change = 0.0;
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) {
        const double x = dmul(0.5, dadd(dmul(g, m[i][j]), ddiv(cof[i][j], dmul(g, det))));
        change = fmax(change, fabs(dsub(x, m[i][j])));
        m[i][j] = x;
      }
    if (change <= 1e-15) break;
  }
}

// Rotation angle of m in radians, as scipy 1.18's Rotation.from_matrix(m).magnitude(); NaN for det(m) <= 0.
__host__ __device__ inline double rotation_magnitude(double (&m)[3][3]) {
  if (!(det3(m) > 0.0)) return NAN;
  bool ortho = true;                                     // isclose(m m^T, I, atol=1e-12) (rtol 1e-5)
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      const double g = dadd(dadd(dmul(m[i][0], m[j][0]), dmul(m[i][1], m[j][1])), dmul(m[i][2], m[j][2]));
      const double e = i == j ? 1.0 : 0.0;
      if (!(fabs(dsub(g, e)) <= dadd(1e-12, dmul(1e-5, e)))) ortho = false;
    }
  if (!ortho) polar3(m);
  const double tr = dadd(dadd(m[0][0], m[1][1]), m[2][2]);
  const double dec[4] = {m[0][0], m[1][1], m[2][2], tr};
  int c = 0;
  for (int k = 1; k < 4; ++k)
    if (dec[k] > dec[c]) c = k;
  double q[4];
  if (c < 3) {
    const int i = c, j = (i + 1) % 3, k = (j + 1) % 3;
    q[i] = dadd(dsub(1.0, tr), dmul(2.0, m[i][i]));
    q[j] = dadd(m[j][i], m[i][j]);
    q[k] = dadd(m[k][i], m[i][k]);
    q[3] = dsub(m[k][j], m[j][k]);
  } else {
    q[0] = dsub(m[2][1], m[1][2]);
    q[1] = dsub(m[0][2], m[2][0]);
    q[2] = dsub(m[1][0], m[0][1]);
    q[3] = dadd(1.0, tr);
  }
  const double nrm = dsqrt(dadd(dadd(dadd(dmul(q[0], q[0]), dmul(q[1], q[1])), dmul(q[2], q[2])), dmul(q[3], q[3])));
  for (int k = 0; k < 4; ++k) q[k] = ddiv(q[k], nrm);
  const double sin_half = dsqrt(dadd(dadd(dmul(q[0], q[0]), dmul(q[1], q[1])), dmul(q[2], q[2])));
  return dmul(2.0, atan2(sin_half, fabs(q[3])));
}

// Frame i of gt, pred [N, 3, 4]: t_err = |t_gt - t_pred|, r_err = magnitude(R_gt^T R_pred) in degrees.
__host__ __device__ inline void pose_error(const double* g, const double* p, double* t_err, double* r_err) {
  const double dx = dsub(g[3], p[3]), dy = dsub(g[7], p[7]), dz = dsub(g[11], p[11]);
  *t_err = dsqrt(dadd(dadd(dmul(dx, dx), dmul(dy, dy)), dmul(dz, dz)));
  double m[3][3];
  for (int a = 0; a < 3; ++a)
    for (int b = 0; b < 3; ++b)
      m[a][b] = dadd(dadd(dmul(g[a], p[b]), dmul(g[4 + a], p[4 + b])), dmul(g[8 + a], p[8 + b]));
  *r_err = dmul(rotation_magnitude(m), 180.0 / M_PI);   // np.degrees: x * (180 / pi)
}

__global__ void pose_errors_kernel(const double* __restrict__ gt, const double* __restrict__ pred, int N,
                                   double* __restrict__ t_err, double* __restrict__ r_err) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < N) pose_error(gt + 12 * i, pred + 12 * i, t_err + i, r_err + i);
}

__global__ void __launch_bounds__(256)
zero_outside_kernel(float* __restrict__ depth, int64_t n, const float* __restrict__ thr, int use_hi, int use_lo,
                    float max_depth) {
  const int s = blockIdx.y;
  float* d = depth + static_cast<int64_t>(s) * n;
  const float hi = thr ? thr[2 * s] : max_depth, lo = thr ? thr[2 * s + 1] : 0.f;
  const bool zhi = thr ? (use_hi && hi > 0.f) : true, zlo = thr && use_lo && lo > 0.f;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const float x = d[i];
    if ((zhi && x > hi) || (zlo && x < lo)) d[i] = 0.f;
  }
}

// cam = ((u - cu) d / fu, (v - cv) d / fv, d): numpy's int64 grid minus a float scalar is float64.
__global__ void __launch_bounds__(256)
depth_to_cam_kernel(const float* __restrict__ depth, const double* __restrict__ intr, int H, int W,
                    float* __restrict__ cam) {
  const int s = blockIdx.y;
  const double* K = intr + 9 * s;
  const double fu = K[0], fv = K[4], cu = K[2], cv = K[5];
  const int64_t hw = static_cast<int64_t>(H) * W;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < hw;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const float d = __ldg(depth + static_cast<int64_t>(s) * hw + i);
    const int v = static_cast<int>(i / W), u = static_cast<int>(i - static_cast<int64_t>(v) * W);
    float* o = cam + (static_cast<int64_t>(s) * hw + i) * 3;
    o[0] = static_cast<float>(__ddiv_rn(__dmul_rn(__dsub_rn(u, cu), d), fu));
    o[1] = static_cast<float>(__ddiv_rn(__dmul_rn(__dsub_rn(v, cv), d), fv));
    o[2] = d;
  }
}

inline int ev_blocks(int64_t work, int per_frame_max) {
  const int64_t b = (work + 4 * 256 - 1) / (4 * 256);
  return static_cast<int>(std::max<int64_t>(1, std::min<int64_t>(b, per_frame_max)));
}

}  // namespace iggt

using namespace iggt;

extern "C" int iggt_zoom_nearest_index(int n_in, int n_out, int32_t* idx) {
  if (n_in <= 0 || n_out <= 0 || !idx) return -1;
  for (int k = 0; k < n_out; ++k) idx[k] = zoom_nearest_index(k, n_in, n_out);
  return 0;
}

extern "C" int iggt_resize_nearest(const float* src, int S, int Hi, int Wi, float* dst, int Ho, int Wo,
                                   iggt_stream_t stream) {
  if (!src || !dst || S <= 0 || S > 65535 || Hi <= 0 || Wi <= 0 || Ho <= 0 || Wo <= 0) return -1;
  const int gx = ev_blocks(static_cast<int64_t>(Ho) * Wo, std::max(1, 4 * device_sm_count() / S));
  resize_nearest_kernel<<<dim3(gx, S), 256, 0, (cudaStream_t)stream>>>(src, Hi, Wi, dst, Ho, Wo);
  return (int)cudaGetLastError();
}

extern "C" int iggt_depth_valid_mask(const float* gt, const float* pred, int64_t S, int64_t n, int sparse,
                                     uint8_t* mask, iggt_stream_t stream) {
  if (!gt || !pred || !mask || S <= 0 || n <= 0) return -1;
  const int g = ev_blocks(S * n, 8 * device_sm_count());
  valid_mask_kernel<<<g, 256, 0, (cudaStream_t)stream>>>(gt, pred, S * n, sparse, mask);
  return (int)cudaGetLastError();
}

extern "C" int iggt_depth_metrics_workspace(int64_t S, int64_t* bytes) {
  if (!bytes || S <= 0 || S > 65535) return -1;
  *bytes = S * EV_MAX_CTAS * EV_NM * static_cast<int64_t>(sizeof(double));
  return 0;
}

extern "C" int iggt_depth_metrics(const float* gt, const float* pred, const uint8_t* mask, int64_t S, int64_t n,
                                  int alignment, const float* medians, int clip, float clip_lo, float clip_hi,
                                  int sparse, void* workspace, double* records, float* aligned,
                                  iggt_stream_t stream) {
  if (!gt || !pred || !mask || !workspace || !records || S <= 0 || S > 65535 || n <= 0 ||
      alignment < IGGT_ALIGN_NONE || alignment > IGGT_ALIGN_LSQ || (alignment == IGGT_ALIGN_MEDIAN && !medians))
    return -1;
  cudaStream_t st = (cudaStream_t)stream;
  const int Si = static_cast<int>(S);
  const int gx = ev_blocks(n, std::min(EV_MAX_CTAS, std::max(1, 2 * device_sm_count() / Si)));
  double* partial = static_cast<double*>(workspace);
  if (alignment == IGGT_ALIGN_LSQ) {
    lsq_sums_kernel<<<dim3(gx, Si), EV_THREADS, 0, st>>>(gt, pred, mask, n, partial);
    reduce_partials_kernel<<<(Si * EV_NL + 127) / 128, 128, 0, st>>>(partial, gx, EV_NL, Si, records + 12,
                                                                   IGGT_EVAL_RECORD);
  }
  align_scale_kernel<<<(Si + 127) / 128, 128, 0, st>>>(alignment, medians, Si, records);
  depth_metrics_kernel<<<dim3(gx, Si), EV_THREADS, 0, st>>>(gt, pred, mask, n, records, clip, clip_lo, clip_hi,
                                                            sparse, aligned, partial);
  reduce_partials_kernel<<<(Si * EV_NM + 127) / 128, 128, 0, st>>>(partial, gx, EV_NM, Si, records, IGGT_EVAL_RECORD);
  return (int)cudaGetLastError();
}

extern "C" int iggt_pose_errors(const double* gt, const double* pred, int N, double* t_err, double* r_err,
                                iggt_stream_t stream) {
  if (!gt || !pred || !t_err || !r_err || N <= 0) return -1;
  pose_errors_kernel<<<(N + 127) / 128, 128, 0, (cudaStream_t)stream>>>(gt, pred, N, t_err, r_err);
  return (int)cudaGetLastError();
}

extern "C" int iggt_pose_errors_host(const double* gt, const double* pred, int N, double* t_err, double* r_err) {
  if (!gt || !pred || !t_err || !r_err || N <= 0) return -1;
  for (int i = 0; i < N; ++i) pose_error(gt + 12 * i, pred + 12 * i, t_err + i, r_err + i);
  return 0;
}

extern "C" int iggt_depth_zero_outside(float* depth, int64_t S, int64_t n, const float* thr, int use_hi, int use_lo,
                                       float max_depth, iggt_stream_t stream) {
  if (!depth || S <= 0 || S > 65535 || n <= 0 || (!thr && !(max_depth > 0.f))) return -1;
  const int gx = ev_blocks(n, std::max(1, 4 * device_sm_count() / static_cast<int>(S)));
  zero_outside_kernel<<<dim3(gx, static_cast<unsigned>(S)), 256, 0, (cudaStream_t)stream>>>(depth, n, thr, use_hi,
                                                                                            use_lo, max_depth);
  return (int)cudaGetLastError();
}

extern "C" int iggt_depth_to_cam(const float* depth, const double* intr, int S, int H, int W, float* cam,
                                 iggt_stream_t stream) {
  if (!depth || !intr || !cam || S <= 0 || S > 65535 || H <= 0 || W <= 0) return -1;
  const int gx = ev_blocks(static_cast<int64_t>(H) * W, std::max(1, 4 * device_sm_count() / S));
  depth_to_cam_kernel<<<dim3(gx, S), 256, 0, (cudaStream_t)stream>>>(depth, intr, H, W, cam);
  return (int)cudaGetLastError();
}
