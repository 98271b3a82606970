// Persistent, warp-specialised wgmma GEMM / implicit-GEMM convolution for sm_90a.
//
//   D[M,N] = epilogue( A[M,K] (16-bit, K-major) x W[N,K]^T (16-bit, K-major), fp32 accumulate in registers )
//
// One CTA per SM loops over 128 x BN output tiles (BN = 64 or 128). Work is handed out by WorkIter (whole tiles
// round-robin, or stream-K ranges of k-blocks for the residual epilogue). Warp roles:
//   warp 0       TMA producer: fills a ring of 128B-swizzled A / W stages in segment order (setmaxnreg: 40 registers)
//   warpgroups 1 and 2: "ping-pong" consumers (setmaxnreg: 232 registers). Consumer warpgroup w owns segments w, w+2,
//                w+4, ... of this CTA: it issues the wgmma of the whole 128 x BN tile (two m64 halves, BN fp32
//                accumulator registers per thread), spills the accumulator to a shared fp32 tile and runs the epilogue
//                (one row per thread: registers -> swizzled smem staging -> TMA store / TMA reduce-add, the two staging
//                buffers alternating between column chunks).
// Named barriers keep the two consumers in segment order, once for the main loops and once for the epilogues, so the
// epilogue of segment s runs while the other warpgroup's main loop of segment s+1 keeps the tensor cores busy, and
// one accumulator tile and one pair of staging buffers serve both warpgroups.
//
// Reference call sites this replaces (all via torch.nn on the reference side, SURVEY.md §2.2):
//   qkv   iggt/layers/attention.py:52-58   (+ q/k LayerNorm(64) and 2-D RoPE, rope.py:154-188)
//   proj  iggt/layers/attention.py:74-75 + layer_scale.py:27 + block.py:105 (residual)
//   fc1   iggt/layers/mlp.py:35-36 (exact-erf GELU)      fc2  mlp.py:38 + block.py:106
//   1x1 / 3x3 convolutions of the dense heads, iggt/heads/dpt_head.py:234-316
#pragma once
#include "ptx.cuh"
#include "launch.cuh"

namespace iggt {

enum GemmEpi : int {
  EPI_STORE16 = 0,   // out16 = act(acc + bias) [+ addend]
  EPI_RESID32 = 1,   // out32 += gamma * (acc + bias)           (TMA reduce-add into the fp32 residual)
  EPI_QKV = 2,       // out16 = [rope(ln(q)) | rope(ln(k)) | v]  (per 64-wide head)
  EPI_STORE32 = 3,   // out32 = acc + bias
  EPI_QKV_GATHER = 4,  // EPI_QKV + the K | V chunks also stored into every rank's gathered buffer (view sharding); a separate
                       // instantiation so that the single-GPU qkv kernel carries none of it (it cost 22 % when it did)
};
__host__ __device__ constexpr bool epi_is_qkv(int e) { return e == EPI_QKV || e == EPI_QKV_GATHER; }

struct GemmParams {
  int M, N, K;
  int num_m_tiles, num_n_tiles, num_k_blocks;
  const float* bias;   // [N] or nullptr
  const float* gamma;  // [N] (EPI_RESID32) or nullptr (=1)
  int act;             // 0 none, 1 exact GELU, 2 ReLU, 3 LeakyReLU(0.01)
  // EPI_QKV
  int qk_norm;         // apply LayerNorm(64) (eps 1e-5, affine) + RoPE to the q and k column ranges
  int C;               // embedding width: q = cols [0,C), k = [C,2C), v = [2C,3C)
  const float* qn_w; const float* qn_b; const float* kn_w; const float* kn_b;  // [64]
  const float* rope_cos; const float* rope_sin;  // [npos][16]
  const int* pos_yx;   // [T][2] (y,x) RoPE positions of one view's tokens
  int T;               // tokens per view (row r of A is token r % T)
  // optional elementwise addend (EPI_STORE16): out += addend[(row % add_rows) * add_ld + col] (16-bit)
  const void* addend; int add_rows; int add_ld;
  // convolution mode (A is an NHWC tensor; K loop runs taps x C/64)
  int conv_taps;       // 1 (1x1 through the 4-D path) or 9 (3x3, pad 1)
  int conv_C;          // input channels
  int H, W, NB;        // spatial size / images
  int tiles_x, tiles_y;
  // residuals for the conv epilogue: out = act_post(act(acc+bias) + resid16[pixel,col] + resid2_16[pixel,col])
  // (NHWC, same H,W, ld = N)
  const void* resid;
  const void* resid2;
  int act_post;
  // EPI_RESID32: round (acc + bias) to 16 bit before the LayerScale multiply (autocast Linear output)
  int round_out16;
  // EPI_QKV, view sharding: the K | V column chunks (col >= gather_col0) of every tile are ALSO stored through these
  // tensor maps (device array; one per rank of the box, each describing THIS rank's row window of that rank's gathered
  // K|V buffer, reached over NVLink peer mappings): the all-gather of the global attention's keys and values is fused
  // into the producing GEMM, tile by tile (parallel.py, FusedKVGather)
  // The maps are 3-D {2048 columns, rows of one scene, scenes}: the rank's rows (scene, view, token) land at
  // (scene, rank, view, token) in the gathered buffer.  The TMA store of a 128-row tile is clipped to the scene of the
  // tile's first row; rows of a tile that belong to a later scene (B - 1 tiles per GEMM) are written by their epilogue
  // threads with plain 16-byte stores through the raw peer pointers that follow the maps in the device array
  // ([n maps][n pointers][ld, scene_ld as int64]).
  const CUtensorMap* gather_maps;
  int n_gather;
  int gather_col0;
  int gather_rows;     // rows of this rank per scene (S_loc * T)
  // stream-K (EPI_RESID32 only): the (tile, k-block) space is cut into gridDim.x equal contiguous ranges; every
  // CTA reduce-adds the partial product of each tile segment it owns (fp32 atomics in L2 make the pieces add up)
  int stream_k;
};

constexpr int GEMM_BM = 128;
constexpr int GEMM_BK = 64;
constexpr int GEMM_THREADS = 384;
constexpr int CONV_TW = 16;
constexpr int CONV_TH = 8;

template <int BN>
struct GemmSmem {
  static constexpr int A_BYTES = GEMM_BM * GEMM_BK * 2;   // 16 KB
  static constexpr int B_BYTES = BN * GEMM_BK * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int STG_BYTES = 16384;                 // 128 rows x 128 B staging tile
  static constexpr int ACC_LD = BN + 8;                   // fp32 accumulator tile row pitch (conflict-free fragment stores)
  static constexpr int ACC_BYTES = GEMM_BM * ACC_LD * 4;
  static constexpr int STAGES = BN == 128 ? 3 : 6;
  static constexpr int VEC_BYTES = BN * 4 + (BN * 4 > 1024 ? BN * 4 : 1024);   // bias[BN] + (gamma[BN] | q/k-norm vectors [4][64])
  static constexpr int TOTAL = STAGES * STAGE_BYTES + ACC_BYTES + 2 * STG_BYTES + 256 /*barriers*/ + VEC_BYTES;
};

template <bool BF16>
__device__ __forceinline__ float cvt16_to_f32(uint16_t h) {
  if constexpr (BF16) return __uint_as_float(static_cast<uint32_t>(h) << 16);
  else return __half2float(__ushort_as_half(h));
}
template <bool BF16>
__device__ __forceinline__ float round16(float x) {
  if constexpr (BF16) return __bfloat162float(__float2bfloat16_rn(x));
  else return __half2float(__float2half_rn(x));
}

__device__ __forceinline__ float apply_act(float x, int act) {
  if (act == 1) return gelu_fast(x);
  if (act == 2) return relu_nan(x);
  if (act == 3) return x > 0.0f ? x : 0.01f * x;
  return x;
}

// Work iterator shared by the three warp roles.  Default: whole tiles, static round-robin over the CTAs.
// stream_k: CTA b owns k-blocks [b*per, (b+1)*per) of the linearised (tile, k-block) space.
struct WorkIter {
  int pos, end, step, kb_per_tile, num_tiles;
  bool sk;
  // `worker` of `workers`: the CTA (or CTA pair) index and count
  __device__ WorkIter(const GemmParams& p, int worker, int workers) {
    kb_per_tile = p.num_k_blocks;
    num_tiles = p.num_m_tiles * p.num_n_tiles;
    sk = p.stream_k != 0;
    if (sk) {
      const long total = static_cast<long>(num_tiles) * kb_per_tile;
      const long per = (total + workers - 1) / workers;
      const long b = static_cast<long>(worker) * per;
      pos = static_cast<int>(b < total ? b : total);
      end = static_cast<int>(b + per < total ? b + per : total);
      step = 0;
    } else {
      pos = worker; end = num_tiles; step = workers;
    }
  }
  // next segment: tile index and k-block range [kb0, kb1)
  __device__ bool next(int& tile, int& kb0, int& kb1) {
    if (pos >= end) return false;
    if (sk) {
      tile = pos / kb_per_tile;
      kb0 = pos - tile * kb_per_tile;
      const int room = end - pos;
      kb1 = kb0 + room < kb_per_tile ? kb0 + room : kb_per_tile;
      pos += kb1 - kb0;
    } else {
      tile = pos; kb0 = 0; kb1 = kb_per_tile; pos += step;
    }
    return true;
  }
};

// CONV: A operand comes from a 4-D NHWC tensor map (box {64, TW, TH, 1}); otherwise 2-D [M,K].
template <int BN, int EPI, bool BF16, bool CONV>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                  const __grid_constant__ CUtensorMap tmC, const GemmParams p) {
  using SM = GemmSmem<BN>;
  constexpr int STAGES = SM::STAGES;
  // named barriers: 1 + w = inside consumer warpgroup w; MMA_DONE + w = w has issued a segment's wgmma (the other
  // warpgroup may start waiting on the next ring stages); EPI_DONE + w = w is through an epilogue (acc_tile, the
  // per-column vectors and the staging buffers are free)
  constexpr uint32_t BAR_MMA_DONE = 3, BAR_EPI_DONE = 5;
  extern __shared__ __align__(1024) uint8_t smem[];   // 128B-swizzled tiles need 1024-byte alignment
  if ((smem_u32(smem) & 1023u) != 0) __trap();
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + STAGES * SM::A_BYTES;
  float* acc_tile = reinterpret_cast<float*>(smem + STAGES * SM::STAGE_BYTES);
  uint8_t* staging = smem + STAGES * SM::STAGE_BYTES + SM::ACC_BYTES;
  uint64_t* bars = reinterpret_cast<uint64_t*>(staging + 2 * SM::STG_BYTES);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + STAGES;
  float* epi_vec = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(bars) + 256);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int worker = static_cast<int>(blockIdx.x);
  const int workers = static_cast<int>(gridDim.x);

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    tma_prefetch_desc(&tmC);
  }
  if (warp == 1 && lane == 0) {
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 1);                     // each stage has one consumer warpgroup
    }
    fence_barrier_init();
  }
  __syncthreads();
  griddep_wait();      // PDL: everything above overlapped the previous kernel's tail
  griddep_launch();

  if (warp < 4) {
    // ------------------------------------------------------------ TMA producer
    reg_dealloc<40>();
    if (warp == 0 && lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      WorkIter work(p, worker, workers);
      int tile, kb0, kb1;
      while (work.next(tile, kb0, kb1)) {
        const int mt = tile / p.num_n_tiles;
        const int nt = tile % p.num_n_tiles;
        int img = 0, y0 = 0, x0 = 0;
        if constexpr (CONV) {
          const int per_img = p.tiles_x * p.tiles_y;
          img = mt / per_img;
          const int r = mt % per_img;
          y0 = (r / p.tiles_x) * CONV_TH;
          x0 = (r % p.tiles_x) * CONV_TW;
        }
        for (int kb = kb0; kb < kb1; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          int dy = 0, dx = 0, c0 = 0;
          if constexpr (CONV) {
            const int cblocks = p.conv_C / GEMM_BK;
            const int tap = kb / cblocks;
            c0 = (kb % cblocks) * GEMM_BK;
            if (p.conv_taps == 9) { dy = tap / 3 - 1; dx = tap % 3 - 1; }
          }
          mbar_expect_tx(&full_bar[stage], SM::STAGE_BYTES);
          if constexpr (CONV) tma_load_4d(smem_a + stage * SM::A_BYTES, &tmA, &full_bar[stage], c0, x0 + dx, y0 + dy, img);
          else tma_load_2d(smem_a + stage * SM::A_BYTES, &tmA, &full_bar[stage], kb * GEMM_BK, mt * GEMM_BM);
          tma_load_2d(smem_b + stage * SM::B_BYTES, &tmB, &full_bar[stage], kb * GEMM_BK, nt * BN);
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    // ------------------------------------------------------------ consumers: main loop, then epilogue (1 row / thread)
    reg_alloc<232>();
    const int wg = (warp - 4) >> 2;        // consumer warpgroup: owns segments wg, wg + 2, ...
    const int ew = (warp - 4) & 3;         // warp inside the warpgroup
    const int row = ew * 32 + lane;        // epilogue: row inside the tile
    const bool leader = (ew == 0 && lane == 0);
    constexpr int NBUF = 2;                // staging buffers, alternating between the column chunks of a tile
    const uint32_t bar_id = 1 + wg;
    const int gtid = ew * 32 + lane;       // thread index inside the warpgroup
    float* const vb = epi_vec;                  // this tile's bias   [BN]
    float* const vg = vb + BN;                  // this tile's gamma  [BN]  (EPI_RESID32)
    float* const vn = vb + BN;                  // q_norm w,b | k_norm w,b  [4][64]  (EPI_QKV, BN >= 128)
    if constexpr (epi_is_qkv(EPI)) {
      // written once; warpgroup 1 reads them only after warpgroup 0's first epilogue (BAR_EPI_DONE)
      if (p.qk_norm && wg == 0) {
        for (int i = gtid; i < 64; i += 128) {
          vn[i] = p.qn_w[i]; vn[64 + i] = p.qn_b[i]; vn[128 + i] = p.kn_w[i]; vn[192 + i] = p.kn_b[i];
        }
      }
    }
    uint32_t store_count = 0;
    WorkIter work(p, worker, workers);
    int tile, kb0, kb1, ntile, nkb0, nkb1;
    bool more = work.next(ntile, nkb0, nkb1);
    uint32_t ring = 0;                     // ring position of the segment's first k-block
    int seg_len = 0;
    for (int seg = 0; more; ++seg) {
      ring += seg_len;
      tile = ntile; kb0 = nkb0; kb1 = nkb1;
      seg_len = kb1 - kb0;
      more = work.next(ntile, nkb0, nkb1);   // segment seg + 1 exists: its warpgroup waits for this segment's signals
      if ((seg & 1) != wg) continue;
      const int mt = tile / p.num_n_tiles;
      const int nt = tile % p.num_n_tiles;
      const int n0 = nt * BN;
      // ---- main loop: the whole tile, rows [0, 64) into acc[0] and [64, 128) into acc[1].  It starts once segment
      // seg - 1 has waited for all of its stages: the full barriers of the ring are then at most one phase ahead of
      // this warpgroup's position, so the parity waits cannot alias.
      if (seg > 0) named_bar_sync(BAR_MMA_DONE + (wg ^ 1), 256);
      int stage = static_cast<int>(ring % STAGES);
      uint32_t phase = (ring / STAGES) & 1;
      float acc[2][BN / 2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc[h][i] = 0.f;
      }
      int prev_stage = -1;
      for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t a_addr = smem_u32(smem_a + stage * SM::A_BYTES);
        const uint32_t b_addr = smem_u32(smem_b + stage * SM::B_BYTES);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < GEMM_BK / 16; ++k) {
          const uint64_t db = make_desc_sw128(b_addr + k * 32, 1024);
          const uint32_t accumulate = (kb != kb0 || k != 0) ? 1u : 0u;
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const uint64_t da = make_desc_sw128(a_addr + h * (64 * 128) + k * 32, 1024);
            if constexpr (BN == 128) wgmma_m64n128k16_ss<BF16>(acc[h], da, db, accumulate);
            else wgmma_m64n64k16_ss<BF16>(acc[h], da, db, accumulate);
          }
        }
        wgmma_commit();
        // the previous k-block's MMAs have retired once at most this one is pending: free its smem slot
        wgmma_wait<1>();
        if (prev_stage >= 0 && gtid == 0) mbar_arrive(&empty_bar[prev_stage]);
        prev_stage = stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      if (more) named_bar_arrive(BAR_MMA_DONE + wg, 256);   // the other warpgroup's main loop may start
      wgmma_wait<0>();
      reg_fence(acc[0]);
      reg_fence(acc[1]);
      if (prev_stage >= 0 && gtid == 0) mbar_arrive(&empty_bar[prev_stage]);

      int img = 0, y0 = 0, x0 = 0;
      long grow;                           // global row (pixel) index of this thread, -1 if out of range
      if constexpr (CONV) {
        const int per_img = p.tiles_x * p.tiles_y;
        img = mt / per_img;
        const int r = mt % per_img;
        y0 = (r / p.tiles_x) * CONV_TH;
        x0 = (r % p.tiles_x) * CONV_TW;
        const int yy = y0 + row / CONV_TW, xx = x0 + row % CONV_TW;
        grow = (yy < p.H && xx < p.W && img < p.NB) ? ((long)img * p.H + yy) * p.W + xx : -1;
      } else {
        grow = (long)mt * GEMM_BM + row;
        if (grow >= p.M) grow = -1;
      }
      // ---- accumulator fragments -> fp32 tile in smem (one row per epilogue thread from here on), per-column vectors
      if (seg > 0) named_bar_sync(BAR_EPI_DONE + (wg ^ 1), 256);   // segment seg - 1's epilogue is done with them
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int r0 = h * 64 + ew * 16 + (lane >> 2);
        float* const d0 = acc_tile + r0 * SM::ACC_LD + 2 * (lane & 3);
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          *reinterpret_cast<float2*>(d0 + 8 * j) = make_float2(acc[h][4 * j], acc[h][4 * j + 1]);
          *reinterpret_cast<float2*>(d0 + 8 * SM::ACC_LD + 8 * j) = make_float2(acc[h][4 * j + 2], acc[h][4 * j + 3]);
        }
      }
      for (int i = gtid; i < BN; i += 128) {
        const int col = n0 + i;
        vb[i] = (p.bias && col < p.N && kb0 == 0) ? __ldg(p.bias + col) : 0.f;   // bias rides with the first K segment
        if constexpr (EPI == EPI_RESID32) vg[i] = (p.gamma && col < p.N) ? __ldg(p.gamma + col) : 1.f;
      }
      named_bar_sync(bar_id, 128);
      const float* const t_row = acc_tile + row * SM::ACC_LD;

      if constexpr (EPI == EPI_STORE16 || epi_is_qkv(EPI)) {
        const int nvalid = min(BN / 64, (p.N - n0 + 63) / 64);
#pragma unroll 1
        for (int c64 = 0; c64 < nvalid; ++c64) {
          const int col0 = n0 + c64 * 64;
          uint8_t* stg = staging + (store_count % NBUF) * SM::STG_BYTES;
          if (leader) tma_store_wait_read<NBUF - 1>();
          named_bar_sync(bar_id, 128);
          float v[64];
#pragma unroll
          for (int i = 0; i < 64; i += 4) {
            const float4 a = *reinterpret_cast<const float4*>(t_row + c64 * 64 + i);
            v[i] = a.x; v[i + 1] = a.y; v[i + 2] = a.z; v[i + 3] = a.w;
          }
          {
#pragma unroll
            for (int i = 0; i < 64; i += 4) {
              const float4 b = *reinterpret_cast<const float4*>(vb + c64 * 64 + i);
              const float2 lo = fadd2(make_float2(v[i], v[i + 1]), make_float2(b.x, b.y));
              const float2 hi = fadd2(make_float2(v[i + 2], v[i + 3]), make_float2(b.z, b.w));
              v[i] = lo.x; v[i + 1] = lo.y; v[i + 2] = hi.x; v[i + 3] = hi.y;
            }
          }
          if constexpr (epi_is_qkv(EPI)) {
            if (p.qk_norm && col0 < 2 * p.C) {
              const bool is_k = col0 >= p.C;
              const float* nw = vn + (is_k ? 128 : 0);
              const float* nb = nw + 64;
              // the reference rounds the Linear output to 16 bit before the fp32 LayerNorm (autocast)
              float s = 0.f;
#pragma unroll
              for (int i = 0; i < 64; ++i) { v[i] = round16<BF16>(v[i]); s += v[i]; }
              const float mean = s * (1.0f / 64.0f);
              float q = 0.f;
#pragma unroll
              for (int i = 0; i < 64; ++i) { const float d = v[i] - mean; q += d * d; }
              const float rstd = rsqrtf(q * (1.0f / 64.0f) + 1e-5f);
#pragma unroll
              for (int i = 0; i < 64; ++i) v[i] = (v[i] - mean) * rstd * nw[i] + nb[i];
              // 2-D RoPE: dims [0,32) rotate with the y position, [32,64) with x; halves of 16
              const int t = (grow >= 0) ? static_cast<int>(grow % p.T) : 0;
              const int py = __ldg(p.pos_yx + 2 * t), px = __ldg(p.pos_yx + 2 * t + 1);
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                const int ps = h == 0 ? py : px;
                const float* cs = p.rope_cos + ps * 16;
                const float* sn = p.rope_sin + ps * 16;
#pragma unroll
                for (int i = 0; i < 16; ++i) {
                  const float c = __ldg(cs + i), s_ = __ldg(sn + i);
                  const float a = v[h * 32 + i], b = v[h * 32 + 16 + i];
                  v[h * 32 + i] = a * c - b * s_;
                  v[h * 32 + 16 + i] = b * c + a * s_;
                }
              }
            }
          } else {
            if (p.act == 1) {
              // autocast: GELU is evaluated on the 16-bit Linear output (iggt/layers/mlp.py:35-36)
#pragma unroll
              for (int i = 0; i < 64; i += 2) {
                const float2 g = gelu_fast2(make_float2(round16<BF16>(v[i]), round16<BF16>(v[i + 1])));
                v[i] = g.x; v[i + 1] = g.y;
              }
            } else if (p.act) {
#pragma unroll
              for (int i = 0; i < 64; ++i) v[i] = apply_act(v[i], p.act);
            }
            if (p.addend && grow >= 0) {
              const uint16_t* ad = reinterpret_cast<const uint16_t*>(p.addend) +
                                   (grow % p.add_rows) * (long)p.add_ld + col0;
#pragma unroll
              for (int i = 0; i < 64; i += 8) {
                if (col0 + i < p.N) {
                  const uint4 u = __ldg(reinterpret_cast<const uint4*>(ad + i));
                  const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
                  for (int j = 0; j < 4; ++j) {
                    v[i + 2 * j] += cvt16_to_f32<BF16>(static_cast<uint16_t>(w[j] & 0xFFFF));
                    v[i + 2 * j + 1] += cvt16_to_f32<BF16>(static_cast<uint16_t>(w[j] >> 16));
                  }
                }
              }
            }
            if constexpr (CONV) {
#pragma unroll
              for (int rr = 0; rr < 2; ++rr) {
                const void* rp = rr == 0 ? p.resid : p.resid2;
                if (rp && grow >= 0) {
                  const uint16_t* ad = reinterpret_cast<const uint16_t*>(rp) + grow * (long)p.N + col0;
#pragma unroll
                  for (int i = 0; i < 64; i += 8) {
                    if (col0 + i < p.N) {
                      const uint4 u = __ldg(reinterpret_cast<const uint4*>(ad + i));
                      const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
                      for (int j = 0; j < 4; ++j) {
                        v[i + 2 * j] += cvt16_to_f32<BF16>(static_cast<uint16_t>(w[j] & 0xFFFF));
                        v[i + 2 * j + 1] += cvt16_to_f32<BF16>(static_cast<uint16_t>(w[j] >> 16));
                      }
                    }
                  }
                }
              }
              if (p.act_post) {
#pragma unroll
                for (int i = 0; i < 64; ++i) v[i] = apply_act(v[i], p.act_post);
              }
            }
          }
          // registers -> 128B-swizzled staging tile (row = 128 B = 64 x 16 bit)
          bool later_scene = false;                                       // EPI_QKV gather: this row is not in the tile's first scene
          if constexpr (EPI == EPI_QKV_GATHER) {
            if (p.n_gather > 0 && col0 >= p.gather_col0 && grow >= 0)
              later_scene = grow / p.gather_rows != (static_cast<long>(mt) * GEMM_BM) / p.gather_rows;
          }
#pragma unroll
          for (int c = 0; c < 8; ++c) {
            uint4 u;
            u.x = pack16x2<BF16>(v[c * 8 + 0], v[c * 8 + 1]);
            u.y = pack16x2<BF16>(v[c * 8 + 2], v[c * 8 + 3]);
            u.z = pack16x2<BF16>(v[c * 8 + 4], v[c * 8 + 5]);
            u.w = pack16x2<BF16>(v[c * 8 + 6], v[c * 8 + 7]);
            *reinterpret_cast<uint4*>(stg + row * 128 + ((c ^ (row & 7)) << 4)) = u;
            if constexpr (EPI == EPI_QKV_GATHER) {
              if (later_scene) {
                void* const* ptrs = reinterpret_cast<void* const*>(p.gather_maps + p.n_gather);
                const long* lds = reinterpret_cast<const long*>(ptrs + p.n_gather);
                const long scene = grow / p.gather_rows, rr = grow - scene * p.gather_rows;
                const long off = scene * __ldg(lds + 1) + rr * __ldg(lds) + (col0 - p.gather_col0) + c * 8;
                for (int r = 0; r < p.n_gather; ++r)
                  *reinterpret_cast<uint4*>(reinterpret_cast<uint16_t*>(ptrs[r]) + off) = u;
              }
            }
          }
          if constexpr (EPI == EPI_QKV_GATHER) {
            if (later_scene) __threadfence_system();                      // peer stores visible before the cross-rank barrier
          }
          fence_proxy_async_smem();
          named_bar_sync(bar_id, 128);
          if (leader) {
            if constexpr (CONV) tma_store_4d(&tmC, stg, col0, x0, y0, img);
            else tma_store_2d(&tmC, stg, col0, mt * GEMM_BM);
            if constexpr (EPI == EPI_QKV_GATHER) {
              if (p.n_gather > 0 && col0 >= p.gather_col0) {             // K | V chunk: to every rank's gathered buffer too
                const int row0 = mt * GEMM_BM, scene = row0 / p.gather_rows, r0 = row0 - scene * p.gather_rows;
                for (int r = 0; r < p.n_gather; ++r)
                  tma_store_3d(&p.gather_maps[r], stg, col0 - p.gather_col0, r0, scene);      // clipped to this scene's rows
              }
            }
            tma_store_commit();
          }
          ++store_count;
        }
      } else {
        // fp32 outputs: 32 columns (128 B) per staging tile
        const int nvalid = min(BN / 32, (p.N - n0 + 31) / 32);
#pragma unroll 1
        for (int c32 = 0; c32 < nvalid; ++c32) {
          const int col0 = n0 + c32 * 32;
          uint8_t* stg = staging + (store_count % NBUF) * SM::STG_BYTES;
          if (leader) tma_store_wait_read<NBUF - 1>();
          named_bar_sync(bar_id, 128);
          float v[32];
#pragma unroll
          for (int i = 0; i < 32; i += 4) {
            const float4 a = *reinterpret_cast<const float4*>(t_row + c32 * 32 + i);
            v[i] = a.x; v[i + 1] = a.y; v[i + 2] = a.z; v[i + 3] = a.w;
          }
#pragma unroll
          for (int i = 0; i < 32; i += 4) {
            const float4 b = *reinterpret_cast<const float4*>(vb + c32 * 32 + i);
            float2 lo = fadd2(make_float2(v[i], v[i + 1]), make_float2(b.x, b.y));
            float2 hi = fadd2(make_float2(v[i + 2], v[i + 3]), make_float2(b.z, b.w));
            if constexpr (EPI == EPI_RESID32) {
              if (p.round_out16 && !p.stream_k) {
                lo.x = round16<BF16>(lo.x); lo.y = round16<BF16>(lo.y);
                hi.x = round16<BF16>(hi.x); hi.y = round16<BF16>(hi.y);
              }
              const float4 g = *reinterpret_cast<const float4*>(vg + c32 * 32 + i);
              lo = fmul2(lo, make_float2(g.x, g.y));
              hi = fmul2(hi, make_float2(g.z, g.w));
            }
            v[i] = lo.x; v[i + 1] = lo.y; v[i + 2] = hi.x; v[i + 3] = hi.y;
          }
          if constexpr (EPI == EPI_STORE32) {
            if (p.act) {
#pragma unroll
              for (int i = 0; i < 32; ++i) v[i] = apply_act(v[i], p.act);
            }
          }
#pragma unroll
          for (int c = 0; c < 8; ++c) {
            float4 u = make_float4(v[c * 4], v[c * 4 + 1], v[c * 4 + 2], v[c * 4 + 3]);
            *reinterpret_cast<float4*>(stg + row * 128 + ((c ^ (row & 7)) << 4)) = u;
          }
          fence_proxy_async_smem();
          named_bar_sync(bar_id, 128);
          if (leader) {
            if constexpr (EPI == EPI_RESID32) tma_reduce_add_2d(&tmC, stg, col0, mt * GEMM_BM);
            else tma_store_2d(&tmC, stg, col0, mt * GEMM_BM);
            tma_store_commit();
          }
          ++store_count;
        }
      }
      if (leader) tma_store_wait_read<0>();   // the staging buffers are free for the other warpgroup's epilogue
      if (more) named_bar_arrive(BAR_EPI_DONE + wg, 256);
    }
    if (leader) {
      tma_store_wait_all<0>();
      if constexpr (EPI == EPI_QKV_GATHER) {
        if (p.n_gather > 0) __threadfence_system();      // peer stores visible before the cross-rank barrier
      }
    }
  }
}

}  // namespace iggt
