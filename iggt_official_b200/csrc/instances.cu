// Instance-mask evaluation (iggt/metrics.py:16-80 calculate_iou / evaluate_matched_instances).
//
//   overlaps:    the K x P intersection counts of 0/1 byte masks are one integer GEMM, I = G P^T, with G [K, n] and
//                P [P, n] row-major byte stacks (K-major operands, as 8-bit wgmma reads them).  TMA -> 128B-swizzled
//                shared memory -> mbarrier ring -> wgmma m64nNk32.s32.u8.u8.  The pixel range is split across CTAs;
//                each CTA keeps s32 accumulators (a count over its slice is <= n < 2^31) and adds them into the int64
//                totals with integer atomics, so every count is exact and repeated calls are bit-identical.  The row
//                sizes |g_i| and |p_j| come from the same staged tiles, multiplied by an all-ones operand in shared
//                memory (G 1 and 1 P^T), so the stacks are read once.  TMA zero-fills rows past K / P and pixels past
//                n; zero bytes change no count.
//   assignment:  scipy's linear_sum_assignment on the host (Crouse's shortest augmenting path for rectangular
//                matrices, with scipy's column scan order and tie rule), iggt_linear_sum_assignment.
#include <cuda.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include <algorithm>
#include <numeric>
#include <vector>

#include "../../include/iggt_b200.h"
#include "launch.cuh"
#include "ptx.cuh"
#include "tmap.cuh"

namespace iggt {

constexpr int MO_BM = 128;                   // gt rows per CTA: 64 per consumer warpgroup
constexpr int MO_BK = 128;                   // pixels (bytes) per stage: one 128-byte swizzle row
constexpr int MO_STAGES = 6;
constexpr int MO_THREADS = 384;              // TMA producer warpgroup + two consumer warpgroups
constexpr int MO_ONES_BYTES = 64 * MO_BK;    // all-ones operand: 64 rows of 128 bytes (8 KB)
constexpr int MO_MIN_KB_PER_SPLIT = 16;      // pixel blocks per CTA at least (bounds the atomics per count)

template <int BN>
struct MoSmem {
  static constexpr int A_BYTES = MO_BM * MO_BK;
  static constexpr int B_BYTES = BN * MO_BK;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int ONES_OFF = MO_STAGES * STAGE_BYTES;
  static constexpr int BAR_OFF = ONES_OFF + MO_ONES_BYTES;
  static constexpr int TOTAL = BAR_OFF + 2 * MO_STAGES * 8 + 1024;   // + slack for the 1024-byte alignment
};

struct MoParams {
  int64_t K, P;
  int kb_total, splits, tiles_n, tiles;
  int64_t* inter;
  int64_t* gsize;
  int64_t* psize;
};

__device__ __forceinline__ void add_count(int64_t* dst, uint32_t v) {
  if (v) atomicAdd(reinterpret_cast<unsigned long long*>(dst), static_cast<unsigned long long>(v));
}

template <int BN, bool GS, bool PS>
__device__ __forceinline__ void mo_consume(uint8_t* smem, const MoParams& p, int wg, int nt, int64_t m0, int kb0,
                                           int kb1, uint64_t* full_bar, uint64_t* empty_bar);

// One CTA: gt rows [mt * 128, +128) x pred rows [nt * BN, +BN) over pixel blocks [kb0, kb1).  Warpgroup 0 is the TMA
// producer; consumer warpgroup w takes gt rows mt * 128 + 64 w + [0, 64).  CTAs with nt == 0 also count the gt rows
// (A times 64 x 8 ones), CTAs with mt == 0 the pred rows (consumer 0: 64 x 128 ones times B; every row of that product
// is the row-size vector).
template <int BN>
__global__ void __launch_bounds__(MO_THREADS, 1)
mask_overlaps_kernel(const __grid_constant__ CUtensorMap tmG, const __grid_constant__ CUtensorMap tmP,
                     const MoParams p) {
  using SM = MoSmem<BN>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);   // swizzled tiles: 1024-byte aligned
  uint8_t* ones = smem + SM::ONES_OFF;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + SM::BAR_OFF);
  uint64_t* empty_bar = full_bar + MO_STAGES;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tile = static_cast<int>(blockIdx.x % p.tiles), split = static_cast<int>(blockIdx.x / p.tiles);
  const int mt = tile / p.tiles_n, nt = tile % p.tiles_n;
  const int kb0 = static_cast<int>(static_cast<int64_t>(split) * p.kb_total / p.splits);
  const int kb1 = static_cast<int>(static_cast<int64_t>(split + 1) * p.kb_total / p.splits);
  const int64_t m0 = static_cast<int64_t>(mt) * MO_BM;
  const int consumers = m0 + 64 < p.K ? 2 : 1;      // a warpgroup whose 64 rows all lie past K issues nothing

  for (int i = threadIdx.x; i < MO_ONES_BYTES / 4; i += MO_THREADS) reinterpret_cast<uint32_t*>(ones)[i] = 0x01010101u;
  fence_proxy_async_smem();                         // generic-proxy writes -> visible to wgmma's async proxy
  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tmG);
    tma_prefetch_desc(&tmP);
  }
  if (warp == 1 && lane == 0) {
    for (int i = 0; i < MO_STAGES; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], consumers);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp < 4) {
    // ------------------------------------------------------------ TMA producer
    reg_dealloc<40>();
    if (warp == 0 && lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait(&empty_bar[stage], phase ^ 1);
        uint8_t* st = smem + stage * SM::STAGE_BYTES;
        mbar_expect_tx(&full_bar[stage], SM::STAGE_BYTES);
        tma_load_2d(st, &tmG, &full_bar[stage], kb * MO_BK, static_cast<int32_t>(m0));
        tma_load_2d(st + SM::A_BYTES, &tmP, &full_bar[stage], kb * MO_BK, nt * BN);
        if (++stage == MO_STAGES) { stage = 0; phase ^= 1; }
      }
    }
    return;
  }
  // -------------------------------------------------------------- consumers
  reg_alloc<232>();
  const int wg = (warp - 4) >> 2;                   // consumer warpgroup
  if (wg >= consumers) return;
  // the row-size products as compile-time variants (no wgmma on a divergent path)
  const bool do_gs = nt == 0, do_ps = mt == 0 && wg == 0;
  if (do_ps) {
    if (do_gs) mo_consume<BN, true, true>(smem, p, wg, nt, m0, kb0, kb1, full_bar, empty_bar);
    else mo_consume<BN, false, true>(smem, p, wg, nt, m0, kb0, kb1, full_bar, empty_bar);
  } else {
    if (do_gs) mo_consume<BN, true, false>(smem, p, wg, nt, m0, kb0, kb1, full_bar, empty_bar);
    else mo_consume<BN, false, false>(smem, p, wg, nt, m0, kb0, kb1, full_bar, empty_bar);
  }
}

// Consumer warpgroup wg of a CTA: main loop over pixel blocks [kb0, kb1), then its counts into the int64 totals.
template <int BN, bool GS, bool PS>
__device__ __forceinline__ void mo_consume(uint8_t* smem, const MoParams& p, int wg, int nt, int64_t m0, int kb0,
                                           int kb1, uint64_t* full_bar, uint64_t* empty_bar) {
  using SM = MoSmem<BN>;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int ew = (warp - 4) & 3;                    // warp inside the warpgroup
  const int gtid = ew * 32 + lane;
  uint8_t* ones = smem + SM::ONES_OFF;
  uint32_t acc[BN / 2], ps[BN / 2], gs[4];          // ps / gs stay unused (and unallocated) without PS / GS
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) acc[i] = ps[i] = 0u;
#pragma unroll
  for (int i = 0; i < 4; ++i) gs[i] = 0u;
  const uint32_t ones_addr = smem_u32(ones);
  int stage = 0, prev_stage = -1;
  uint32_t phase = 0;
  for (int kb = kb0; kb < kb1; ++kb) {
    mbar_wait(&full_bar[stage], phase);
    const uint32_t a_addr = smem_u32(smem + stage * SM::STAGE_BYTES) + wg * (64 * MO_BK);
    const uint32_t b_addr = smem_u32(smem + stage * SM::STAGE_BYTES + SM::A_BYTES);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < MO_BK / 32; ++k) {
      const uint64_t da = make_desc_sw128(a_addr + k * 32, 1024);
      const uint64_t db = make_desc_sw128(b_addr + k * 32, 1024);
      const uint64_t d1 = make_desc_sw128(ones_addr + k * 32, 1024);
      if constexpr (BN == 128) wgmma_m64n128k32_u8(acc, da, db);
      else wgmma_m64n64k32_u8(acc, da, db);
      if constexpr (GS) wgmma_m64n8k32_u8(gs, da, d1);
      if constexpr (PS) {
        if constexpr (BN == 128) wgmma_m64n128k32_u8(ps, d1, db);
        else wgmma_m64n64k32_u8(ps, d1, db);
      }
    }
    wgmma_commit();
    wgmma_wait<1>();                                // the previous block's MMAs have retired: free its stage
    if (prev_stage >= 0 && gtid == 0) mbar_arrive(&empty_bar[prev_stage]);
    prev_stage = stage;
    if (++stage == MO_STAGES) { stage = 0; phase ^= 1; }
  }
  wgmma_wait<0>();
  reg_fence(acc);
  reg_fence(ps);
  reg_fence(gs);
  if (prev_stage >= 0 && gtid == 0) mbar_arrive(&empty_bar[prev_stage]);

  // ---- fragments -> int64 totals: thread (ew, lane) holds rows 16 ew + lane / 4 (+ 8), columns 8 j + 2 (lane % 4) + {0, 1}
  const int64_t g0 = m0 + wg * 64 + ew * 16 + (lane >> 2), g1 = g0 + 8;
  const int64_t pc = static_cast<int64_t>(nt) * BN + 2 * (lane & 3);
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    const int64_t c0 = pc + 8 * j, c1 = c0 + 1;
    if (g0 < p.K && c0 < p.P) add_count(p.inter + g0 * p.P + c0, acc[4 * j]);
    if (g0 < p.K && c1 < p.P) add_count(p.inter + g0 * p.P + c1, acc[4 * j + 1]);
    if (g1 < p.K && c0 < p.P) add_count(p.inter + g1 * p.P + c0, acc[4 * j + 2]);
    if (g1 < p.K && c1 < p.P) add_count(p.inter + g1 * p.P + c1, acc[4 * j + 3]);
  }
  if (GS && (lane & 3) == 0) {                      // every column of G 1 is the row size
    if (g0 < p.K) add_count(p.gsize + g0, gs[0]);
    if (g1 < p.K) add_count(p.gsize + g1, gs[2]);
  }
  if (PS && ew == 0 && lane < 4) {                  // row 0 of 1 P^T
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      const int64_t c0 = pc + 8 * j;
      if (c0 < p.P) add_count(p.psize + c0, ps[4 * j]);
      if (c0 + 1 < p.P) add_count(p.psize + c0 + 1, ps[4 * j + 1]);
    }
  }
}

template <int BN>
int launch_mask_overlaps(const uint8_t* g, int64_t K, int64_t ldg, const uint8_t* pm, int64_t P, int64_t ldp,
                         int64_t n, int64_t* inter, int64_t* gsize, int64_t* psize, cudaStream_t st) {
  using SM = MoSmem<BN>;
  static DeviceOnce once;
  if (once.first()) {
    const cudaError_t e = cudaFuncSetAttribute(mask_overlaps_kernel<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                               SM::TOTAL);
    if (e != cudaSuccess) {
      once.reset_current();
      return (int)e;
    }
  }
  CUtensorMap tmG, tmP;
  const uint64_t gdims[2] = {static_cast<uint64_t>(n), static_cast<uint64_t>(K)};
  const uint64_t gstr[1] = {static_cast<uint64_t>(ldg)};
  const uint32_t gbox[2] = {MO_BK, MO_BM};
  const uint64_t pdims[2] = {static_cast<uint64_t>(n), static_cast<uint64_t>(P)};
  const uint64_t pstr[1] = {static_cast<uint64_t>(ldp)};
  const uint32_t pbox[2] = {MO_BK, BN};
  if (make_tmap(&tmG, TM_U8, 2, g, gdims, gstr, gbox) || make_tmap(&tmP, TM_U8, 2, pm, pdims, pstr, pbox)) return -3;

  MoParams prm;
  prm.K = K;
  prm.P = P;
  prm.kb_total = static_cast<int>((n + MO_BK - 1) / MO_BK);
  prm.tiles_n = static_cast<int>((P + BN - 1) / BN);
  const int64_t tiles = ((K + MO_BM - 1) / MO_BM) * prm.tiles_n;
  if (tiles > (1 << 24)) return -1;
  prm.tiles = static_cast<int>(tiles);
  // persistent-sized grid: about one CTA per SM, the pixel range split evenly across the CTAs of each tile
  const int64_t want = std::max<int64_t>(1, device_sm_count() / tiles);
  prm.splits = static_cast<int>(std::max<int64_t>(1, std::min<int64_t>(want, prm.kb_total / MO_MIN_KB_PER_SPLIT)));
  prm.inter = inter;
  prm.gsize = gsize;
  prm.psize = psize;

  cudaError_t e = cudaMemsetAsync(inter, 0, static_cast<size_t>(K * P) * sizeof(int64_t), st);
  if (e == cudaSuccess) e = cudaMemsetAsync(gsize, 0, static_cast<size_t>(K) * sizeof(int64_t), st);
  if (e == cudaSuccess) e = cudaMemsetAsync(psize, 0, static_cast<size_t>(P) * sizeof(int64_t), st);
  if (e != cudaSuccess) return (int)e;
  mask_overlaps_kernel<BN><<<static_cast<unsigned>(tiles * prm.splits), MO_THREADS, SM::TOTAL, st>>>(tmG, tmP, prm);
  return (int)cudaGetLastError();
}

// ---- scipy.optimize.linear_sum_assignment (host)
// Crouse, "On implementing 2D rectangular assignment algorithms" (IEEE TAES 2016), as scipy runs it on a cost
// matrix with nr <= nc: rows are added one at a time, each by a Dijkstra-style shortest augmenting path over the
// reduced costs minVal + c[i, j] - u[i] - v[j].  The scan keeps the columns not yet reached in a list that starts
// as nc-1, ..., 0 and is compacted by moving its last entry into the slot of the column just reached; among equal
// path costs the first one in that list wins unless a later one is an unassigned column (a sink).
struct Lsap {
  int64_t nr, nc;
  const double* c;
  std::vector<double> u, v, dist;
  std::vector<int64_t> path, col4row, row4col, remaining;
  std::vector<char> SR, SC;

  Lsap(int64_t r, int64_t cc, const double* cost)
      : nr(r), nc(cc), c(cost), u(r, 0.0), v(cc, 0.0), dist(cc), path(cc, -1), col4row(r, -1), row4col(cc, -1),
        remaining(cc), SR(r), SC(cc) {}

  // the sink column of the shortest augmenting path from row i, or -1 if every remaining cost is infinite
  int64_t augment(int64_t i, double* min_out) {
    double minval = 0.0;
    int64_t left = nc;
    for (int64_t it = 0; it < nc; ++it) remaining[it] = nc - it - 1;
    std::fill(SR.begin(), SR.end(), 0);
    std::fill(SC.begin(), SC.end(), 0);
    std::fill(dist.begin(), dist.end(), INFINITY);
    int64_t sink = -1;
    while (sink == -1) {
      int64_t index = -1;
      double lowest = INFINITY;
      SR[i] = 1;
      for (int64_t it = 0; it < left; ++it) {
        const int64_t j = remaining[it];
        const double r = minval + c[i * nc + j] - u[i] - v[j];
        if (r < dist[j]) {
          path[j] = i;
          dist[j] = r;
        }
        if (dist[j] < lowest || (dist[j] == lowest && row4col[j] == -1)) {
          lowest = dist[j];
          index = it;
        }
      }
      minval = lowest;
      if (minval == INFINITY) return -1;
      const int64_t j = remaining[index];
      if (row4col[j] == -1) sink = j;
      else i = row4col[j];
      SC[j] = 1;
      remaining[index] = remaining[--left];
    }
    *min_out = minval;
    return sink;
  }

  int solve() {
    for (int64_t cur = 0; cur < nr; ++cur) {
      double minval = 0.0;
      const int64_t sink = augment(cur, &minval);
      if (sink < 0) return -3;
      u[cur] += minval;
      for (int64_t i = 0; i < nr; ++i)
        if (SR[i] && i != cur) u[i] += minval - dist[col4row[i]];
      for (int64_t j = 0; j < nc; ++j)
        if (SC[j]) v[j] -= minval - dist[j];
      for (int64_t j = sink;;) {                    // augment along the path back to row cur
        const int64_t i = path[j];
        row4col[j] = i;
        std::swap(col4row[i], j);
        if (i == cur) break;
      }
    }
    return 0;
  }
};

}  // namespace iggt

using namespace iggt;

extern "C" int iggt_mask_overlaps(const uint8_t* g, int64_t K, int64_t ldg, const uint8_t* p, int64_t P, int64_t ldp,
                                  int64_t n, int64_t* inter, int64_t* gsize, int64_t* psize, iggt_stream_t stream) {
  if (!g || !p || !inter || !gsize || !psize || K <= 0 || P <= 0 || n <= 0 || K >= (1ll << 31) ||
      P >= (1ll << 31) || n > (1ll << 31) - MO_BK)
    return -1;
  if (ldg < n || ldp < n || (ldg & 15) || (ldp & 15) || (reinterpret_cast<uintptr_t>(g) & 15) ||
      (reinterpret_cast<uintptr_t>(p) & 15))
    return -2;
  cudaStream_t st = (cudaStream_t)stream;
  return P <= 64 ? launch_mask_overlaps<64>(g, K, ldg, p, P, ldp, n, inter, gsize, psize, st)
                 : launch_mask_overlaps<128>(g, K, ldg, p, P, ldp, n, inter, gsize, psize, st);
}

extern "C" int iggt_linear_sum_assignment(const double* cost, int64_t nr, int64_t nc, int64_t* rows, int64_t* cols) {
  if (nr < 0 || nc < 0 || (nr * nc > 0 && (!cost || !rows || !cols))) return -1;
  if (nr == 0 || nc == 0) return 0;
  for (int64_t i = 0; i < nr * nc; ++i)
    if (!std::isfinite(cost[i])) return -2;
  const bool transpose = nc < nr;                    // a tall matrix is solved as its transpose
  std::vector<double> t;
  if (transpose) {
    t.resize(nr * nc);
    for (int64_t i = 0; i < nr; ++i)
      for (int64_t j = 0; j < nc; ++j) t[j * nr + i] = cost[i * nc + j];
  }
  Lsap s(transpose ? nc : nr, transpose ? nr : nc, transpose ? t.data() : cost);
  const int st = s.solve();
  if (st) return st;
  if (transpose) {                                   // pairs (col4row[k], k) sorted by their row col4row[k]
    std::vector<int64_t> order(s.nr);
    std::iota(order.begin(), order.end(), 0);
    std::sort(order.begin(), order.end(), [&](int64_t a, int64_t b) { return s.col4row[a] < s.col4row[b]; });
    for (int64_t k = 0; k < s.nr; ++k) {
      rows[k] = s.col4row[order[k]];
      cols[k] = order[k];
    }
  } else {
    for (int64_t i = 0; i < nr; ++i) {
      rows[i] = i;
      cols[i] = s.col4row[i];
    }
  }
  return 0;
}
