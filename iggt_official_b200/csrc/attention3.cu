// Flash-attention forward for head_dim 64 on sm_90a.  Replaces F.scaled_dot_product_attention at
// iggt/layers/attention.py:61-66.
//
// Persistent CTAs over work items (sequence, head, pair of 128-row query tiles A / B), 3 warpgroups:
//   WG0      : warp 0 TMA producer (Q double-buffered per tile, a K / V ring shared by both tiles)
//   WG1, WG2 : one consumer per query tile (A, B), each working its 128 rows as two 64-row halves
// For every kv tile and half, a consumer computes S = Q K^T (wgmma, both operands from 128B-swizzled shared memory,
// fp32 in registers), runs the online softmax on the register fragment (row max / sum across the 4 threads of a row),
// packs P to 16 bit straight into the A-operand registers of O += P V (wgmma with A from registers, V read MN-major
// from shared memory) and keeps O in registers.  Inside a consumer, the softmax of one 64 x 64 slice runs while the
// P V of the slice before it is in flight (attn3_tile), and the two consumers run free, interleaving their softmax
// phases with each other's MMAs.  Registers: setmaxnreg gives the producer warpgroup 40, the consumers 232.
// Item schedule: Attn3Items below.
#include <stdlib.h>
#include "ptx.cuh"
#include "tmap.cuh"
#include "launch.cuh"
#include "../../include/iggt_b200.h"

namespace iggt {

constexpr int A3_BQ = 128;
constexpr int A3_BK = 128;
constexpr int A3_D = 64;
constexpr int A3_STAGES = 4;
constexpr int A3_THREADS = 384;
constexpr int A3_TILE = A3_BK * A3_D * 2;     // 16 KB
constexpr int A3_SMEM = A3_TILE * (4 + 2 * A3_STAGES) + 512;   // Q is double-buffered per tile
static_assert(A3_SMEM <= 232448, "shared memory budget");

struct Attn3Params {
  int Lq, Lk, H, num_seq;
  int q_pairs;
  int total_items;
  int64_t ldo;
  void* o;
  float scale_log2;
  int light_tail;       // the last query pair of every (sequence, head) has no rows for tile B (Lq = 1374: 94 rows)
  // split-KV (view-sharded ranks: 88 work items for 132 SMs): the kv tiles of every item are cut into `kv_splits` ranges
  // of `tiles_per_split`; each (item, split) writes its un-normalised fp32 O and (m, l) to the workspace and
  // attention3_merge_kernel combines the splits.  kv_splits == 1: the kernel writes the normalised 16-bit output itself.
  int kv_splits, tiles_per_split;
  float* ws_o;          // [split][num_seq * Lq][H * 64]
  float* ws_ml;         // [split][num_seq * Lq][H][2]  (running max in log2-scaled units' source scale, row sum)
};

// Work items = (query-tile pair, head, sequence).  When the last pair of every (sequence, head) has no rows for tile B
// (Lq = 1374: 10.7 tiles) that pair is a half-weight item: tile B's MMAs and softmax are skipped outright for it, and
// the static schedule is longest-processing-time-first - every CTA first takes its full items round-robin, then the
// halves go (twice) to the CTAs that got one full item fewer, then round-robin again.  8 x 16 x (5 + 1/2) items on
// 132 CTAs finish in 5.5 item-times instead of 6.0.  All roles of a CTA walk the same sequence.
struct Attn3Items {
  int n_full, n_half, full_pairs, G, c, r;
  int k;          // position in this CTA's sequence
  const Attn3Params& p;
  // G CTAs in the grid, this is CTA c (host-callable so that the schedule itself is unit-tested without a GPU)
  __host__ __device__ Attn3Items(const Attn3Params& p_, int G_, int c_) : p(p_) {
    G = G_; c = c_; k = 0; split = 0;
    if (p.light_tail) {
      full_pairs = p.q_pairs - 1;
      n_half = p.H * p.num_seq * p.kv_splits;
      n_full = full_pairs * n_half;
    } else {
      full_pairs = p.q_pairs; n_full = p.total_items; n_half = 0;
    }
    r = n_full % G;
  }
  // next item of this CTA: false when done; b_active = tile B has rows
  int split;      // kv split of the item returned last by next() / peek()
  __host__ __device__ bool next(int& qp, int& head, int& seq, bool& b_active) {
    const int my_full = (n_full - c + G - 1) / G;            // full items of this CTA (c, c + G, ...)
    int sh;
    if (k < my_full) {
      const int item = c + k * G;
      qp = item % full_pairs; sh = item / full_pairs; b_active = true;
    } else {
      int m = k - my_full;                                   // m-th half item of this CTA
      int h;
      if (r > 0) {
        const int short_ctas = G - r;                        // CTAs [r, G) have one full item fewer
        if (c >= r) {
          if (m < 2) h = (c - r) + m * short_ctas;
          else h = 2 * short_ctas + c + (m - 2) * G;
          // a CTA whose first-round half does not exist has no later one either (h grows with m)
        } else {
          h = 2 * short_ctas + c + m * G;
        }
      } else {
        h = c + m * G;
      }
      if (h >= n_half) return false;
      qp = full_pairs; sh = h; b_active = false;
    }
    ++k;
    head = sh % p.H;
    const int rest = sh / p.H;
    seq = rest % p.num_seq;
    split = rest / p.num_seq;
    return true;
  }
  // kv tile range [j0, j1) of the current item
  __host__ __device__ void kv_range(int n_kv, int& j0, int& j1) const {
    j0 = split * p.tiles_per_split;
    j1 = j0 + p.tiles_per_split < n_kv ? j0 + p.tiles_per_split : n_kv;
  }
  // the item that follows the current one (for the Q prefetch), without advancing
  __host__ __device__ bool peek(int& qp, int& head, int& seq, bool& b_active) {
    const int k0 = k, split0 = split;
    const bool ok = next(qp, head, seq, b_active);
    k = k0; split = split0;
    return ok;
  }
};

// Register state of a consumer warpgroup for one work item.  A slice is 64 query rows (half hh of the query tile)
// x 64 keys (half kh of the kv tile).
struct Attn3Frag {
  float o[2][32];
  float m[2][2], l[2][2];            // [half][row r / r + 8]: running max (raw score units), partial sum
  float s[32];                       // S of the next slice, then its unpacked P
  uint32_t pa[4][4];                 // P of the current slice as the A fragments of the 4 k16 steps of P V
  float fac[2];                      // the current slice's rescale factors of O (rows r / r + 8)
};

struct Attn3Bars {
  uint64_t *k_full, *k_empty, *v_full, *v_empty, *q_empty;
};

// S = Q K^T of one slice: rows [64 hh, +64) of the query tile at q_addr, keys [64 kh, +64) of the kv tile at k_addr
template <bool BF16>
__device__ __forceinline__ void attn3_issue_s(float (&d)[32], uint32_t q_addr, int hh, uint32_t k_addr, int kh) {
  wgmma_fence();
#pragma unroll
  for (int kk = 0; kk < A3_D / 16; ++kk)
    wgmma_m64n64k16_ss<BF16>(d, make_desc_sw128(q_addr + hh * (64 * 128) + kk * 32, 1024),
                             make_desc_sw128(k_addr + kh * (64 * 128) + kk * 32, 1024), kk != 0 ? 1u : 0u);
  wgmma_commit();
}

// Online softmax of a completed S fragment (each row is spread over the 4 threads of a quad): masks the keys past
// kvalid, updates the running max m and sum l of its half, leaves the rescale factors of O in fac (first: the half's
// first slice, which rescales nothing) and the unpacked P in s.
__device__ __forceinline__ void attn3_softmax(float (&s)[32], float (&m)[2], float (&l)[2], float (&fac)[2], int kvalid,
                                              bool first, float c, int quad) {
  if (kvalid < 64) {                                   // only the ragged last kv tile
#pragma unroll
    for (int jj = 0; jj < 8; ++jj) {
      const int col = 8 * jj + 2 * quad;
      if (col >= kvalid) { s[4 * jj] = -INFINITY; s[4 * jj + 2] = -INFINITY; }
      if (col + 1 >= kvalid) { s[4 * jj + 1] = -INFINITY; s[4 * jj + 3] = -INFINITY; }
    }
  }
  float mx0 = s[0], mx1 = s[2];
#pragma unroll
  for (int jj = 0; jj < 8; ++jj) {
    mx0 = fmaxf(mx0, fmaxf(s[4 * jj], s[4 * jj + 1]));
    mx1 = fmaxf(mx1, fmaxf(s[4 * jj + 2], s[4 * jj + 3]));
  }
  mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
  mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
  mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
  mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
  const float mn0 = fmaxf(m[0], mx0), mn1 = fmaxf(m[1], mx1);
  if (!first) {
    // a fully masked slice leaves the running max in place (mn == m): f = 1
    fac[0] = ex2_approx((m[0] - mn0) * c);
    fac[1] = ex2_approx((m[1] - mn1) * c);
    // its own rounding: contracted with the sum below into one fma, l (and so the output) would change in the last bit
    l[0] = __fmul_rn(l[0], fac[0]);
    l[1] = __fmul_rn(l[1], fac[1]);
  }
  m[0] = mn0; m[1] = mn1;
  const float nmc0 = -mn0 * c, nmc1 = -mn1 * c;
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int jj = 2 * kk + h;
      s[4 * jj] = ex2_approx(fmaf(s[4 * jj], c, nmc0));
      s[4 * jj + 1] = ex2_approx(fmaf(s[4 * jj + 1], c, nmc0));
      s[4 * jj + 2] = ex2_approx(fmaf(s[4 * jj + 2], c, nmc1));
      s[4 * jj + 3] = ex2_approx(fmaf(s[4 * jj + 3], c, nmc1));
    }
    const float* e = s + 8 * kk;
    l[0] += (e[0] + e[1]) + (e[4] + e[5]);
    l[1] += (e[2] + e[3]) + (e[6] + e[7]);
  }
}

// P to 16 bit, as the A fragments of the 4 k16 steps of P V
template <bool BF16>
__device__ __forceinline__ void attn3_pack_p(uint32_t (&pa)[4][4], const float (&s)[32]) {
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) {
    const float* e = s + 8 * kk;
    pa[kk][0] = pack16x2<BF16>(e[0], e[1]);      // row r,     keys 16 kk + 2 quad + {0, 1}
    pa[kk][1] = pack16x2<BF16>(e[2], e[3]);      // row r + 8
    pa[kk][2] = pack16x2<BF16>(e[4], e[5]);      // row r,     keys 16 kk + 8 + 2 quad + {0, 1}
    pa[kk][3] = pack16x2<BF16>(e[6], e[7]);      // row r + 8
  }
}

// One kv tile j of a consumer's item.  Its slices run (kh, hh) = (0,0), (0,1), (1,0), (1,1): each half still sees its
// keys in order, and consecutive slices use different O halves.  On entry the P of the tile's first slice is packed
// in f.pa; per slice n the consumer issues S_{n+1}, rescales its O half and issues PV_n, waits for S_{n+1} only, runs
// the softmax of slice n + 1 while PV_n is in flight, then waits for PV_n and packs P_{n+1}.  No wgmma is in flight
// between slices, so P needs one register buffer.  In the item's first kv tile the halves' first slices rescale
// nothing; LAST (the item's last kv tile, whose last slice has no S_{n+1}) is compile-time, so that no wgmma is issued
// under a runtime condition.
template <bool BF16, bool LAST>
__device__ __forceinline__ void attn3_tile(Attn3Frag& f, int j, bool first, int& st, uint32_t& ph,
                                           const Attn3Bars& b, const uint8_t* sK, const uint8_t* sV, uint32_t q_addr,
                                           int Lk, float c, int quad, int gtid) {
  const uint32_t k_addr = smem_u32(sK + st * A3_TILE);
  const uint32_t v_addr = smem_u32(sV + st * A3_TILE);
  int nst = st + 1; uint32_t nph = ph;                     // stage of kv tile j + 1
  if (nst == A3_STAGES) { nst = 0; nph ^= 1; }
#pragma unroll
  for (int sl = 0; sl < 4; ++sl) {
    const int kh = sl >> 1, hh = sl & 1;
    const bool has_next = sl < 3 || !LAST;
    const int nkh = sl < 3 ? (sl + 1) >> 1 : 0, nhh = hh ^ 1;
    // ---- S of the next slice (after the tile's last slice: the next kv tile's first)
    if (sl < 3) {
      attn3_issue_s<BF16>(f.s, q_addr, nhh, k_addr, nkh);
    } else if (!LAST) {
      mbar_wait(&b.k_full[nst], nph);
      attn3_issue_s<BF16>(f.s, q_addr, 0, smem_u32(sK + nst * A3_TILE), 0);
    }
    // ---- O += P V of this slice  (V rows [64 kh, +64) of the kv tile)
    float (&o)[32] = f.o[hh];
    if (!first || kh > 0) {
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) {
        o[4 * jj] *= f.fac[0]; o[4 * jj + 1] *= f.fac[0]; o[4 * jj + 2] *= f.fac[1]; o[4 * jj + 3] *= f.fac[1];
      }
    }
    if (sl == 0) mbar_wait(&b.v_full[st], ph);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk)
      wgmma_m64n64k16_rs_tb<BF16>(o, f.pa[kk], make_desc_sw128(v_addr + kh * (64 * 128) + kk * 2048, 1024), 1u);
    wgmma_commit();
    if (has_next) {
      // ---- softmax of the next slice while P V runs
      wgmma_wait<1>();
      reg_fence(f.s);
      if (sl == 2 && gtid == 0) {
        mbar_arrive(&b.k_empty[st]);                     // all four S of this kv tile are complete
        if (LAST) mbar_arrive(b.q_empty);                // last use of this item's Q
      }
      const int nj = sl < 3 ? j : j + 1;
      attn3_softmax(f.s, f.m[nhh], f.l[nhh], f.fac, Lk - nj * A3_BK - nkh * 64, first && sl == 0, c, quad);
    }
    wgmma_wait<0>();
    reg_fence(o);
    if (sl == 3 && gtid == 0) mbar_arrive(&b.v_empty[st]);   // the last P V of this kv tile has retired
    if (has_next) attn3_pack_p<BF16>(f.pa, f.s);
  }
  st = nst; ph = nph;
}

template <bool BF16>
__global__ void __launch_bounds__(A3_THREADS, 1)
attention3_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                  const __grid_constant__ CUtensorMap tmV, const Attn3Params p) {
  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* sQ = smem;                      // [2 buffers][2 tiles]: the next item's Q lands while this one runs
  uint8_t* sK = sQ + 4 * A3_TILE;
  uint8_t* sV = sK + A3_STAGES * A3_TILE;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sV + A3_STAGES * A3_TILE);
  uint64_t* q_full = bars;                 // [2 buffers][2 tiles]
  uint64_t* q_empty = q_full + 4;          // [2 buffers][2 tiles]
  uint64_t* k_full = q_empty + 4;          // [A3_STAGES]
  uint64_t* k_empty = k_full + A3_STAGES;
  uint64_t* v_full = k_empty + A3_STAGES;
  uint64_t* v_empty = v_full + A3_STAGES;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int n_kv = (p.Lk + A3_BK - 1) / A3_BK;

  if (warp == 0 && lane == 0) {
    if ((smem_u32(smem) & 1023u) != 0) __trap();
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmK);
    tma_prefetch_desc(&tmV);
  }
  if (warp == 1 && lane == 0) {
    for (int i = 0; i < 4; ++i) { mbar_init(&q_full[i], 1); mbar_init(&q_empty[i], 1); }
    for (int i = 0; i < A3_STAGES; ++i) {
      mbar_init(&k_full[i], 1); mbar_init(&k_empty[i], 2);   // K / V: released by both consumers
      mbar_init(&v_full[i], 1); mbar_init(&v_empty[i], 2);
    }
    fence_barrier_init();
  }
  __syncthreads();
  griddep_wait();
  griddep_launch();

  if (warp < 4) {
    reg_dealloc<40>();
    if (warp == 0 && lane == 0) {
      // ------------------------------------------------------------------ TMA producer
      int st = 0; uint32_t ph = 0;
      uint32_t q_cnt[2] = {0, 0};             // per tile: Q loads issued (= items in which the tile takes part)
      // Q of item n of a tile goes to buffer n & 1; it is requested one item ahead (after the first K/V tile of the
      // previous item has been requested), so a short item (frame attention: 11 kv tiles) never waits for its Q
      auto load_q = [&](int qp, int head, int seq, bool b_active) {
#pragma unroll
        for (int t = 0; t < 2; ++t) {
          if (t == 1 && !b_active) continue;
          const uint32_t buf = q_cnt[t] & 1, par = (q_cnt[t] >> 1) & 1;
          mbar_wait(&q_empty[buf * 2 + t], par ^ 1);
          mbar_expect_tx(&q_full[buf * 2 + t], A3_TILE);
          tma_load_2d(sQ + (buf * 2 + t) * A3_TILE, &tmQ, &q_full[buf * 2 + t], head * A3_D,
                      seq * p.Lq + (qp * 2 + t) * A3_BQ);
          ++q_cnt[t];
        }
      };
      Attn3Items items(p, static_cast<int>(gridDim.x), static_cast<int>(blockIdx.x));
      int qp, head, seq, nqp, nhead, nseq;
      bool b_active, nb;
      if (items.peek(qp, head, seq, b_active)) load_q(qp, head, seq, b_active);
      while (items.next(qp, head, seq, b_active)) {
        int j0, j1;
        items.kv_range(n_kv, j0, j1);
        const bool has_next = items.peek(nqp, nhead, nseq, nb);
        const int col = head * A3_D;
        for (int j = j0; j < j1; ++j) {
          mbar_wait(&k_empty[st], ph ^ 1);
          mbar_expect_tx(&k_full[st], A3_TILE);
          tma_load_3d(sK + st * A3_TILE, &tmK, &k_full[st], col, j * A3_BK, seq);
          mbar_wait(&v_empty[st], ph ^ 1);
          mbar_expect_tx(&v_full[st], A3_TILE);
          tma_load_3d(sV + st * A3_TILE, &tmV, &v_full[st], col, j * A3_BK, seq);
          if (++st == A3_STAGES) { st = 0; ph ^= 1; }
          if (j == j0 && has_next) load_q(nqp, nhead, nseq, nb);
        }
      }
    }
  } else {
    // -------------------------------------------------------------------- consumers (one warpgroup per query tile)
    reg_alloc<232>();
    const int t = (warp - 4) >> 2;                 // query tile
    const int gtid = threadIdx.x & 127;
    const int ew = (warp - 4) & 3;                 // warp inside the warpgroup: fragment rows [16 ew, 16 ew + 16) of a half
    const int quad = lane & 3;
    const float c = p.scale_log2;
    int st = 0; uint32_t ph = 0;                   // K / V ring stage and parity of the current kv tile
    uint32_t item_cnt = 0;                         // items in which THIS tile took part
    Attn3Items items(p, static_cast<int>(gridDim.x), static_cast<int>(blockIdx.x));
    int qp, head, seq;
    bool b_active;
    while (items.next(qp, head, seq, b_active)) {
      int j0, j1;
      items.kv_range(n_kv, j0, j1);
      const int split = items.split;
      if (!b_active && t == 1) {
        // tile B has no rows in this item: only keep the shared K/V ring turning
        for (int j = j0; j < j1; ++j) {
          mbar_wait(&k_full[st], ph);
          if (gtid == 0) mbar_arrive(&k_empty[st]);
          mbar_wait(&v_full[st], ph);
          if (gtid == 0) mbar_arrive(&v_empty[st]);
          if (++st == A3_STAGES) { st = 0; ph ^= 1; }
        }
        continue;
      }
      const uint32_t qbuf = item_cnt & 1, qbpar = (item_cnt >> 1) & 1;
      ++item_cnt;
      const uint32_t q_addr = smem_u32(sQ + (qbuf * 2 + t) * A3_TILE);
      mbar_wait(&q_full[qbuf * 2 + t], qbpar);
      Attn3Frag f;
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
#pragma unroll
        for (int i = 0; i < 32; ++i) f.o[hh][i] = 0.f;
        f.m[hh][0] = f.m[hh][1] = -INFINITY;
        f.l[hh][0] = f.l[hh][1] = 0.f;
      }
      const Attn3Bars bars_t{k_full, k_empty, v_full, v_empty, &q_empty[qbuf * 2 + t]};
      // the item's first slice: S, softmax and P before the pipelined kv tiles
      mbar_wait(&k_full[st], ph);
      attn3_issue_s<BF16>(f.s, q_addr, 0, smem_u32(sK + st * A3_TILE), 0);
      wgmma_wait<0>();
      reg_fence(f.s);
      attn3_softmax(f.s, f.m[0], f.l[0], f.fac, p.Lk - j0 * A3_BK, true, c, quad);
      attn3_pack_p<BF16>(f.pa, f.s);
      for (int j = j0; j < j1 - 1; ++j)
        attn3_tile<BF16, false>(f, j, j == j0, st, ph, bars_t, sK, sV, q_addr, p.Lk, c, quad, gtid);
      attn3_tile<BF16, true>(f, j1 - 1, j1 - 1 == j0, st, ph, bars_t, sK, sV, q_addr, p.Lk, c, quad, gtid);
      const float (&o)[2][32] = f.o;
      const float (&m)[2][2] = f.m;
      const float (&l)[2][2] = f.l;
      // ---- epilogue of the item
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          float lt = l[hh][h];
          lt += __shfl_xor_sync(0xffffffffu, lt, 1);
          lt += __shfl_xor_sync(0xffffffffu, lt, 2);
          const int qrow = (qp * 2 + t) * A3_BQ + hh * 64 + ew * 16 + (lane >> 2) + 8 * h;
          if (qrow >= p.Lq) continue;
          if (p.kv_splits > 1) {
            // partial result of this kv split: un-normalised O (relative to this split's running max m) + (m, l)
            const int64_t grow = static_cast<int64_t>(split) * p.num_seq * p.Lq + static_cast<int64_t>(seq) * p.Lq + qrow;
            float* dst = p.ws_o + grow * (p.H * A3_D) + head * A3_D + 2 * quad;
#pragma unroll
            for (int jj = 0; jj < 8; ++jj)
              *reinterpret_cast<float2*>(dst + 8 * jj) = make_float2(o[hh][4 * jj + 2 * h], o[hh][4 * jj + 2 * h + 1]);
            if (quad == 0) *reinterpret_cast<float2*>(p.ws_ml + (grow * p.H + head) * 2) = make_float2(m[hh][h], lt);
          } else {
            const float inv = 1.0f / lt;
            uint16_t* dst = reinterpret_cast<uint16_t*>(p.o) + (static_cast<int64_t>(seq) * p.Lq + qrow) * p.ldo +
                            head * A3_D + 2 * quad;
#pragma unroll
            for (int jj = 0; jj < 8; ++jj)
              *reinterpret_cast<uint32_t*>(dst + 8 * jj) =
                  pack16x2<BF16>(o[hh][4 * jj + 2 * h] * inv, o[hh][4 * jj + 2 * h + 1] * inv);
          }
        }
      }
    }
  }
}

// Combines the kv splits of attention3_kernel: one warp per (query row, head), lane = two of the 64 columns.
//   m = max_s m_s,  w_s = 2^((m_s - m) * scale_log2),  out = sum_s w_s O_s / sum_s w_s l_s
template <bool BF16>
__global__ void __launch_bounds__(256)
attention3_merge_kernel(const float* __restrict__ ws_o, const float* __restrict__ ws_ml, void* __restrict__ out, int64_t ldo,
                        int64_t rows, int H, int splits, float scale_log2) {
  griddep_wait();
  griddep_launch();
  const int64_t item = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;     // (row, head)
  if (item >= rows * H) return;
  const int lane = threadIdx.x & 31;
  const int64_t row = item / H;
  const int head = static_cast<int>(item % H);
  float m = -INFINITY;
  for (int s = 0; s < splits; ++s) m = fmaxf(m, __ldg(ws_ml + ((s * rows + row) * H + head) * 2));
  float2 acc = make_float2(0.f, 0.f);
  float l = 0.f;
  for (int s = 0; s < splits; ++s) {
    const float2 ml = __ldg(reinterpret_cast<const float2*>(ws_ml + ((s * rows + row) * H + head) * 2));
    const float w = ex2_approx((ml.x - m) * scale_log2);
    const float2 o = __ldg(reinterpret_cast<const float2*>(ws_o + (s * rows + row) * (static_cast<int64_t>(H) * A3_D) +
                                                             head * A3_D + lane * 2));
    acc.x = fmaf(w, o.x, acc.x);
    acc.y = fmaf(w, o.y, acc.y);
    l = fmaf(w, ml.y, l);
  }
  const float inv = 1.0f / l;
  uint32_t* dst = reinterpret_cast<uint32_t*>(reinterpret_cast<uint16_t*>(out) + row * ldo + head * A3_D + lane * 2);
  *dst = pack16x2<BF16>(acc.x * inv, acc.y * inv);
}

template <bool BF16>
int launch_attention3(const CUtensorMap& tQ, const CUtensorMap& tK, const CUtensorMap& tV, const Attn3Params& p,
                      cudaStream_t stream) {
  auto kern = attention3_kernel<BF16>;
  static DeviceOnce once;
  if (once.first()) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, A3_SMEM);
    if (e != cudaSuccess) { once.reset_current(); return (int)e; }
  }
  const int sms = device_sm_count();
  const int grid = p.total_items < sms ? p.total_items : sms;
  return (int)launch_pdl(kern, dim3(grid), dim3(A3_THREADS), A3_SMEM, stream, tQ, tK, tV, p);
}

}  // namespace iggt

using namespace iggt;

namespace {
// Cost (in kv-tile steps of one CTA) of running the launch with `splits` kv ranges on `sms` CTAs: rounds x (tiles per
// split + a fixed per-item overhead: Q load, pipeline fill, first-tile max, O read-out) + the merge pass over the fp32
// workspace.  Model constants (estimates, not fitted on this kernel): 7 steps per item, 8 steps + workspace traffic for
// the merge launch.
double attn3_cost(int num_seq, int Lq, int Lk, int H, int splits, int sms) {
  const int q_tiles = (Lq + A3_BQ - 1) / A3_BQ, n_kv = (Lk + A3_BK - 1) / A3_BK;
  const int tps = (n_kv + splits - 1) / splits, se = (n_kv + tps - 1) / tps;
  const double full = static_cast<double>(num_seq) * H * (q_tiles / 2) * se;       // items with both query tiles
  const double half = (q_tiles & 1) ? static_cast<double>(num_seq) * H * se : 0.0;  // items whose tile B has no rows
  const double weight = full + 0.5 * half;
  double rounds;
  if (full + half <= sms) rounds = full > 0 ? 1.0 : 0.5;
  else {   // longest-first: the busiest CTA carries ceil(full / sms) full items, or the average rounded up to a half item
    const double by_weight = static_cast<double>(static_cast<long>(2.0 * weight / sms + 0.999999)) / 2.0;
    const double by_full = static_cast<double>(static_cast<long>(full / sms + 0.999999));
    rounds = by_weight > by_full ? by_weight : by_full;
  }
  double cost = rounds * (tps + 7.0);
  if (se > 1) {
    const double ws_bytes = 2.0 * se * num_seq * Lq * H * A3_D * 4;     // written + read back
    cost += 8.0 + ws_bytes / 8.0e12 / 1.4e-6;                            // workspace stays in L2 (model constants)
  }
  return cost;
}
// kv splits that minimise attn3_cost (1 = no split); IGGT_ATTN_SPLITS forces a value
int attn3_plan_splits(int num_seq, int Lq, int Lk, int H, int sms) {
  static const int forced = [] { const char* e = getenv("IGGT_ATTN_SPLITS"); return e ? atoi(e) : 0; }();
  const int n_kv = (Lk + A3_BK - 1) / A3_BK;
  int best = 1;
  if (forced > 0) {
    best = forced < n_kv ? forced : n_kv;
  } else {
    double bc = attn3_cost(num_seq, Lq, Lk, H, 1, sms);
    for (int s = 2; s <= 8 && s <= n_kv; ++s) {
      const double c = attn3_cost(num_seq, Lq, Lk, H, s, sms);
      if (c < 0.95 * bc) { bc = c; best = s; }        // a split must buy at least 5 %
    }
  }
  const int tps = (n_kv + best - 1) / best;
  return (n_kv + tps - 1) / tps;                       // effective splits (no empty range)
}
void attn3_shape(Attn3Params& p, int num_seq, int Lq, int Lk, int H, int splits = 1) {
  p.Lq = Lq; p.Lk = Lk; p.H = H; p.num_seq = num_seq;
  const int q_tiles = (Lq + A3_BQ - 1) / A3_BQ;
  const int n_kv = (Lk + A3_BK - 1) / A3_BK;
  p.q_pairs = (q_tiles + 1) / 2;
  p.kv_splits = splits < 1 ? 1 : splits;
  p.tiles_per_split = (n_kv + p.kv_splits - 1) / p.kv_splits;
  p.ws_o = nullptr; p.ws_ml = nullptr;
  p.total_items = num_seq * H * p.q_pairs * p.kv_splits;
  static const int lpt = [] { const char* e = getenv("IGGT_ATTN_LPT"); return e ? atoi(e) : 1; }();
  p.light_tail = (lpt && (q_tiles & 1) && p.q_pairs > 1) ? 1 : 0;    // odd tile count: the last pair has no tile B
}
}  // namespace

// Host-side view of the kernel's static work schedule (no GPU needed): the items CTA `cta` of a `grid`-CTA launch
// processes, in order, as (query pair, head, sequence, tile-B-active) quadruples.  Returns the item count (which may
// exceed max_items; only the first max_items are written) or a negative argument error.
extern "C" int iggt_attention_schedule(int num_seq, int Lq, int Lk, int H, int grid, int cta, int* items,
                                       int max_items) {
  if (num_seq <= 0 || Lq <= 0 || Lk <= 0 || H <= 0 || grid <= 0 || cta < 0 || cta >= grid) return -1;
  Attn3Params p{};
  attn3_shape(p, num_seq, Lq, Lk, H);
  Attn3Items it(p, grid, cta);
  int n = 0, qp, head, seq;
  bool b_active;
  while (it.next(qp, head, seq, b_active)) {
    if (items && n < max_items) {
      items[4 * n] = qp; items[4 * n + 1] = head; items[4 * n + 2] = seq; items[4 * n + 3] = b_active ? 1 : 0;
    }
    ++n;
  }
  return n;
}

// As iggt_attention_schedule, for a launch with `splits` kv ranges: quintuples (query pair, head, sequence, tile-B-active,
// kv split); also returns the kv tiles per split through *tiles_per_split.
extern "C" int iggt_attention_schedule_splits(int num_seq, int Lq, int Lk, int H, int splits, int grid, int cta, int* items,
                                              int max_items, int* tiles_per_split) {
  if (num_seq <= 0 || Lq <= 0 || Lk <= 0 || H <= 0 || splits <= 0 || grid <= 0 || cta < 0 || cta >= grid) return -1;
  Attn3Params p{};
  attn3_shape(p, num_seq, Lq, Lk, H, splits);
  if (tiles_per_split) *tiles_per_split = p.tiles_per_split;
  Attn3Items it(p, grid, cta);
  int n = 0, qp, head, seq;
  bool b_active;
  while (it.next(qp, head, seq, b_active)) {
    if (items && n < max_items) {
      items[5 * n] = qp; items[5 * n + 1] = head; items[5 * n + 2] = seq; items[5 * n + 3] = b_active ? 1 : 0;
      items[5 * n + 4] = it.split;
    }
    ++n;
  }
  return n;
}

namespace {
int attention_launch(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv, void* o,
                     int64_t ldo, int num_seq, int Lq, int Lk, int H, int head_dim, float scale, int dtype, int splits,
                     void* ws, int64_t ws_bytes, cudaStream_t s) {
  if (head_dim != 64) return -1;
  if (num_seq <= 0 || Lq <= 0 || Lk <= 0 || H <= 0 || splits < 1) return -1;
  if ((ldq % 8) || (ldk % 8) || (ldv % 8) || (ldo % 8)) return -2;
  if (dtype != 0 && dtype != 1) return -3;
  const TmDtype dt = dtype ? TM_BF16 : TM_F16;
  CUtensorMap tQ, tK, tV;
  if (make_tmap_2d(&tQ, dt, q, (uint64_t)num_seq * Lq, (uint64_t)H * 64, ldq, 64, A3_BQ)) return -4;
  // K and V are 3-D {H*64 columns, Lk rows, num_seq sequences}: the ragged last key tile of a sequence reads zeros past
  // row Lk (TMA fill), never the next sequence's rows.  The mask gives those keys P = 0, but 0 * V is NaN where V is inf,
  // so with a 2-D map over all sequences one sequence's output could depend on its neighbour's values.
  {
    const uint64_t dims[3] = {(uint64_t)H * 64, (uint64_t)Lk, (uint64_t)num_seq};
    const uint32_t box[3] = {64, A3_BK, 1};
    const uint64_t kstr[2] = {(uint64_t)ldk * 2, (uint64_t)Lk * ldk * 2};
    const uint64_t vstr[2] = {(uint64_t)ldv * 2, (uint64_t)Lk * ldv * 2};
    if (make_tmap(&tK, dt, 3, k, dims, kstr, box)) return -4;
    if (make_tmap(&tV, dt, 3, v, dims, vstr, box)) return -4;
  }
  Attn3Params p;
  attn3_shape(p, num_seq, Lq, Lk, H, splits);
  const int n_kv = (Lk + A3_BK - 1) / A3_BK;
  if ((p.kv_splits - 1) * p.tiles_per_split >= n_kv) return -5;        // an empty kv range: use iggt_attention_plan's count
  const int64_t rows = static_cast<int64_t>(num_seq) * Lq;
  if (p.kv_splits > 1) {
    const int64_t need = p.kv_splits * rows * H * (A3_D + 2) * 4;
    if (!ws || ws_bytes < need || (reinterpret_cast<uintptr_t>(ws) & 15)) return -6;
    p.ws_o = reinterpret_cast<float*>(ws);
    p.ws_ml = p.ws_o + p.kv_splits * rows * H * A3_D;
  }
  p.ldo = ldo; p.o = o;
  p.scale_log2 = scale * 1.4426950408889634f;
  const int st = dtype ? launch_attention3<true>(tQ, tK, tV, p, s) : launch_attention3<false>(tQ, tK, tV, p, s);
  if (st != 0 || p.kv_splits == 1) return st;
  const int64_t warps = rows * H;
  const unsigned grid = static_cast<unsigned>((warps + 7) / 8);
  if (dtype) return (int)launch_pdl(attention3_merge_kernel<true>, dim3(grid), dim3(256), 0, s, (const float*)p.ws_o, (const float*)p.ws_ml, o, ldo, rows, H, p.kv_splits, p.scale_log2);
  return (int)launch_pdl(attention3_merge_kernel<false>, dim3(grid), dim3(256), 0, s, (const float*)p.ws_o, (const float*)p.ws_ml, o, ldo, rows, H, p.kv_splits, p.scale_log2);
}
}  // namespace

extern "C" int iggt_attention_plan(int num_seq, int Lq, int Lk, int H, int sms, int* splits, int64_t* ws_bytes) {
  if (num_seq <= 0 || Lq <= 0 || Lk <= 0 || H <= 0 || !splits || !ws_bytes) return -1;
  const int s = attn3_plan_splits(num_seq, Lq, Lk, H, sms > 0 ? sms : device_sm_count());
  *splits = s;
  *ws_bytes = s > 1 ? static_cast<int64_t>(s) * num_seq * Lq * H * (A3_D + 2) * 4 : 0;
  return 0;
}

extern "C" int iggt_attention_fwd_ws(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v, int64_t ldv,
                                     void* o, int64_t ldo, int num_seq, int Lq, int Lk, int H, int head_dim, float scale,
                                     int dtype, int splits, void* ws, int64_t ws_bytes, iggt_stream_t stream) {
  return attention_launch(q, ldq, k, ldk, v, ldv, o, ldo, num_seq, Lq, Lk, H, head_dim, scale, dtype, splits, ws, ws_bytes,
                          (cudaStream_t)stream);
}

extern "C" int iggt_attention_fwd(const void* q, int64_t ldq, const void* k, int64_t ldk, const void* v,
                                  int64_t ldv, void* o, int64_t ldo, int num_seq, int Lq, int Lk, int H,
                                  int head_dim, float scale, int dtype, iggt_stream_t stream) {
  return attention_launch(q, ldq, k, ldk, v, ldv, o, ldo, num_seq, Lq, Lk, H, head_dim, scale, dtype, 1, nullptr, 0,
                          (cudaStream_t)stream);
}
