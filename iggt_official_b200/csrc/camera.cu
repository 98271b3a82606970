// The whole camera head (iggt/heads/camera_head.py:83-154 + head_act.py:12-35) as ONE persistent kernel.
//
// M = B*S <= 16 camera tokens against 216 M parameters, four refinement iterations: every Linear is a weight stream
// (1.7 GB of 16-bit weights per forward, 0.5 ms at the H100's 3.35 TB/s) with a few MFLOP of work, but as separate
// launches it is ~180 small dependent kernels (LayerNorm / skinny GEMM / tiny attention / AdaLN glue), i.e. launch- and
// latency-bound, and on view-sharded ranks the head is replicated.  Here the ~27 phases of an iteration run inside one grid of <= 128 CTAs with a device-wide barrier
// between phases:
//   * warp 8 is a TMA producer that walks the same phase program AHEAD of the consumers: weight stages (ONE 3-D box
//     {64 k, 16 columns, 16 k groups} = 1024 k x 16 columns = 32 KB per instruction, 128B-swizzled) of the next phases
//     stream into a 3-stage ring while the consumers are still in the barrier of the current one - weights do not depend on
//     activations - so HBM stays busy across phase boundaries; LayerNorm gamma | beta come through a 2-slot bulk-copy ring;
//   * activations are tiny and live in L2: after each barrier the 8 consumer warps pull the phase's input rows
//     ([M, <= 2048] fp32, 16-byte vectors), apply the LayerNorm that precedes the Linear (statistics over the row, two-pass
//     in registers) and store them as TWO 16-bit planes hi + lo = x (cam_split);
//   * the products run on the tensor cores (mma.sync.m16n8k16, fp32 accumulate): C[16 x 16] += (X_hi + X_lo) W^T, warp w
//     takes every 8th k step of a stage, fragments come straight from the swizzled stage / the padded planes (bank-conflict
//     free), the 8 warps' partial tiles meet in an 8 KB shared-memory reduction and thread (row, column) finishes one output.
//   * bias, exact-erf GELU / SiLU, LayerScale, residual and the pose accumulation + activation ride in the epilogue;
//   * the S x S attention (16 heads x 128) is a phase of its own: one warp per (row, head).
// fp32 accumulation, 16-bit weights, activations to ~2^-22 (fp16 weights) / 2^-16 (bf16) relative - within rounding of the
// arithmetic of iggt_skinny_gemm / iggt_small_attention, which this kernel replaces for M <= 16 (larger B*S keep the
// per-layer launches).
#include <stdlib.h>
#include "ptx.cuh"
#include "tmap.cuh"
#include "launch.cuh"
#include "../../include/iggt_b200.h"

namespace iggt {

constexpr int CAM_DIM = 2048, CAM_HEADS = 16, CAM_HD = 128;
constexpr int CAM_THREADS = 288;              // 8 consumer warps + 1 producer warp
constexpr int CAM_COLS = 16;                  // output columns per tile (two n-tiles of mma.m16n8k16)
constexpr int CAM_KS = 1024;                  // k per weight stage: ONE 3-D TMA box {64 k, 16 columns, 16 k groups} = 32 KB
constexpr int CAM_STAGES = 3;
constexpr int CAM_W_BYTES = CAM_COLS * CAM_KS * 2;       // 32 KB
constexpr int CAM_X_BYTES = 2 * 16 * (1024 + 8) * 2;     // activation planes (hi | lo) [rows][KX + 8] 16-bit: 8 x 2056 or 16 x 1032 per plane
constexpr int CAM_LN_FLOATS = 2 * 2 * CAM_DIM;           // LayerNorm gamma | beta of the next two LN phases (32 KB)
constexpr int CAM_RED_FLOATS = 8 * 16 * CAM_COLS;        // cross-warp reduction [8 warps][16 rows][16 cols] (8 KB)
constexpr int CAM_SMEM = CAM_STAGES * CAM_W_BYTES + CAM_X_BYTES + CAM_LN_FLOATS * 4 + CAM_RED_FLOATS * 4 + 512;
static_assert(CAM_SMEM <= 232448, "shared memory budget");
constexpr int CAM_MAX_PHASES = 32, CAM_MAX_MAPS = 24;

enum CamPhaseType : int { PH_GEMM = 0, PH_ATTN = 1, PH_MODULATE = 2, PH_LNROWS = 3 };
enum CamFlags : int { CF_EMBED_IN = 1, CF_POSE_OUT = 2, CF_ONCE = 4 };     // CF_ONCE: only before the first iteration

struct CamPhase {
  int type, tm, N, K;
  const float* x; long ldx;
  int ln;                      // 0 none, 1 LayerNorm (ln_w, ln_b), 2 LayerNorm without affine
  float ln_eps;
  const float* ln_w; const float* ln_b;
  const float* bias; const float* gamma; const float* resid; long ldr;
  float* out; long ldo;
  int act;                     // 0 none, 1 exact GELU, 4 SiLU
  int flags;
  const float* x2;             // CF_EMBED_IN: the empty pose token [16]; PH_MODULATE: ptn
  const float* x3;             // PH_MODULATE: pt
  float* out2;                 // CF_POSE_OUT: activated poses [iters][M][9]
};

struct CamProgram {
  CUtensorMap maps[CAM_MAX_MAPS];
  CamPhase ph[CAM_MAX_PHASES];
  int n_phases, iters, M, Mpad, B, S;
  unsigned* barrier;           // zeroed before the launch
  unsigned long long* dbg;     // optional (IGGT_CAMERA_DEBUG=1): CTA 0 stamps %globaltimer at 4 points of every phase
  int dbg_mode;                // 2: consumers skip the arithmetic (pure weight-streaming rate; results are garbage)
};

__device__ __forceinline__ unsigned long long cam_now() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
__device__ __forceinline__ unsigned ld_acquire_u32(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
// device-wide barrier of the consumer warps (256 threads per CTA; the producer warp never joins)
__device__ __forceinline__ void cam_grid_sync(unsigned* counter, unsigned& target) {
  named_bar_sync(1, 256);
  if (threadIdx.x == 0) {
    target += gridDim.x;
    __threadfence();
    atomicAdd(counter, 1u);
    while (ld_acquire_u32(counter) < target) { __nanosleep(20); }
    __threadfence();
  }
  named_bar_sync(1, 256);
}

// D (16 x 8, fp32) += A (16 x 16, row) * B (16 x 8, col), 16-bit operands
template <bool BF16>
__device__ __forceinline__ void cam_mma(float (&d)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
  if constexpr (BF16)
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]) : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
  else
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]) : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}
// x = hi + lo with hi, lo in the weights' 16-bit type: the fp32 activation enters the tensor cores as two operands
// (products with the 16-bit weights are exact in fp32, so the split only costs the ~2^-22 (fp16) / 2^-16 (bf16) of x it drops)
template <bool BF16>
__device__ __forceinline__ void cam_split(float x, uint16_t& hi, uint16_t& lo) {
  if constexpr (BF16) {
    const __nv_bfloat16 h = __float2bfloat16_rn(x);
    const __nv_bfloat16 l = __float2bfloat16_rn(x - __bfloat162float(h));
    hi = *reinterpret_cast<const uint16_t*>(&h); lo = *reinterpret_cast<const uint16_t*>(&l);
  } else {
    const __half h = __float2half_rn(x);
    const __half l = __float2half_rn(x - __half2float(h));
    hi = *reinterpret_cast<const uint16_t*>(&h); lo = *reinterpret_cast<const uint16_t*>(&l);
  }
}

__device__ __forceinline__ float warp_sum_f(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// MP = padded row count (8 or 16): xs is [k][MP]
template <bool BF16, int MP>
__global__ void __launch_bounds__(CAM_THREADS, 1)
camera_head_kernel(const __grid_constant__ CamProgram prog) {
  extern __shared__ __align__(1024) uint8_t cam_smem[];      // 128B-swizzled weight stages need 1024-byte alignment
  uint8_t* sW = cam_smem;
  uint16_t* xs = reinterpret_cast<uint16_t*>(cam_smem + CAM_STAGES * CAM_W_BYTES);     // hi plane, then lo plane
  float* lnbuf = reinterpret_cast<float*>(cam_smem + CAM_STAGES * CAM_W_BYTES + CAM_X_BYTES);     // [2 slots][gamma | beta][2048]
  float* red = lnbuf + CAM_LN_FLOATS;                     // [8 warps][16 rows][16 cols]
  uint64_t* full = reinterpret_cast<uint64_t*>(red + CAM_RED_FLOATS);
  uint64_t* empty = full + CAM_STAGES;
  uint64_t* ln_full = empty + CAM_STAGES;                 // [2]
  uint64_t* ln_empty = ln_full + 2;                       // [2]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int G = gridDim.x, cta = blockIdx.x;
  const int M = prog.M;
  constexpr int KX = 16384 / MP;                 // k extent of the staged activations (2048 for <= 8 rows, 1024 for <= 16)
  constexpr int KXP = KX + 8;                    // plane row pitch (16-bit elements): +16 B spreads the 8 rows of a fragment over all banks
  uint16_t* const xlo = xs + MP * KXP;
  if (threadIdx.x == 0) {
    for (int i = 0; i < CAM_STAGES; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], 8); }
    for (int i = 0; i < 2; ++i) { mbar_init(&ln_full[i], 1); mbar_init(&ln_empty[i], 8); }
    fence_barrier_init();
  }
  __syncthreads();
  griddep_wait();
  griddep_launch();

  if (warp == 8) {
    // ------------------------------------------------------------------ weight producer: runs ahead of the barriers
    if (lane == 0) {
      int st = 0; uint32_t ph = 0;
      int lslot = 0; uint32_t lph = 0;
      for (int it = 0; it < prog.iters; ++it)
        for (int p = 0; p < prog.n_phases; ++p) {
          const CamPhase& P = prog.ph[p];
          if (P.type != PH_GEMM || ((P.flags & CF_ONCE) && it > 0)) continue;
          const int tiles = (P.N + CAM_COLS - 1) / CAM_COLS;
          const int nst = (P.K + CAM_KS - 1) / CAM_KS;      // 32 KB stages per tile
          if (P.ln == 1 && cta < tiles) {                   // gamma / beta of this phase's LayerNorm, ahead of time
            mbar_wait(&ln_empty[lslot], lph ^ 1);
            mbar_expect_tx(&ln_full[lslot], 2 * CAM_DIM * 4);
            tma_bulk_load_1d(lnbuf + lslot * 2 * CAM_DIM, P.ln_w, CAM_DIM * 4, &ln_full[lslot]);
            tma_bulk_load_1d(lnbuf + lslot * 2 * CAM_DIM + CAM_DIM, P.ln_b, CAM_DIM * 4, &ln_full[lslot]);
            if (++lslot == 2) { lslot = 0; lph ^= 1; }
          }
          // the consumers' order: activation chunk (KX k = SPC stages) -> this CTA's tiles -> the chunk's stages
          constexpr int SPC = KX / CAM_KS;
          for (int s0 = 0; s0 < nst; s0 += SPC)
            for (int t = cta; t < tiles; t += G)
              for (int ks = s0; ks < min(s0 + SPC, nst); ++ks) {
                mbar_wait(&empty[st], ph ^ 1);
                mbar_expect_tx(&full[st], CAM_W_BYTES);     // the box is always 32 KB (out-of-range k groups / columns: zeros)
                tma_load_3d(sW + st * CAM_W_BYTES, &prog.maps[P.tm], &full[st], 0, t * CAM_COLS, ks * (CAM_KS / 64));
                if (++st == CAM_STAGES) { st = 0; ph ^= 1; }
              }
        }
    }
    return;
  }

  // -------------------------------------------------------------------- consumers (8 warps)
  const int tid = threadIdx.x;                   // 0..255
  unsigned target = 0;
  int st = 0; uint32_t ph = 0;
  int lslot = 0; uint32_t lph = 0;
  for (int it = 0; it < prog.iters; ++it)
    for (int p = 0; p < prog.n_phases; ++p) {
      const CamPhase& P = prog.ph[p];
      if ((P.flags & CF_ONCE) && it > 0) continue;
      unsigned long long* stamp = (prog.dbg && cta == 0 && tid == 0) ? prog.dbg + (it * CAM_MAX_PHASES + p) * 4 : nullptr;
      long long wait_clk = 0;
      if (stamp) stamp[0] = cam_now();
      if (P.type == PH_GEMM) {
        const int tiles = (P.N + CAM_COLS - 1) / CAM_COLS;
        const int nchunks = (P.K + KX - 1) / KX;                         // activation chunks of KX
        const bool embed0 = (P.flags & CF_EMBED_IN) && it == 0;
        // Tensor-core math: C[16 rows x 16 cols] += X[16 x k] W^T with mma.m16n8k16; the fp32 activations enter as two 16-bit
        // operands (hi + lo, cam_split), the weights straight from their 128B-swizzled TMA stage.  Warp w owns k steps
        // [8 w', 8 w' + 8) of every 128-step stage quarter...: each stage of 1024 k = 64 k steps of 16, 8 per warp.
        const int g = lane >> 2, tq = lane & 3;
        const float* gam = lnbuf + lslot * 2 * CAM_DIM;
        if (P.ln == 1 && cta < tiles) mbar_wait(&ln_full[lslot], lph);    // gamma | beta are in shared memory
        // chunk-major over this CTA's tiles (<= 4): an activation chunk is staged ONCE and every tile consumes its weight
        // stages of that chunk (the accumulators of all tiles live in registers across chunks)
        const int ntl = cta < tiles ? (tiles - cta + G - 1) / G : 0;
        float acc[4][2][4];
#pragma unroll
        for (int ti = 0; ti < 4; ++ti)
#pragma unroll
          for (int c = 0; c < 2; ++c)
#pragma unroll
            for (int i = 0; i < 4; ++i) acc[ti][c][i] = 0.f;
        if (ntl > 0) {
          for (int ch = 0; ch < nchunks; ++ch) {
            const int k0 = ch * KX;
            const int kn = min(KX, P.K - k0);                             // k of this chunk (16, 1024, 2048)
            const int kst = (kn + 15) & ~15;                              // staged extent: whole k steps
            {
              // ---- stage the activations as 16-bit planes hi | lo, [row][KXP], LayerNorm applied on the way
              named_bar_sync(2, 256);                                     // previous readers of xs are done
              for (int m = warp; m < MP; m += 8) {
                uint16_t* dh = xs + m * KXP;
                uint16_t* dl = xlo + m * KXP;
                if (m >= M) {
                  for (int k = lane * 4; k < kst; k += 128) { *reinterpret_cast<uint2*>(dh + k) = make_uint2(0u, 0u); *reinterpret_cast<uint2*>(dl + k) = make_uint2(0u, 0u); }
                  continue;
                }
                const float* row = embed0 ? P.x2 : P.x + m * P.ldx;
                auto put = [&](int k, const float4& y) {                  // 4 consecutive k -> 8 bytes in each plane
                  uint16_t h[4], l[4];
                  cam_split<BF16>(y.x, h[0], l[0]); cam_split<BF16>(y.y, h[1], l[1]);
                  cam_split<BF16>(y.z, h[2], l[2]); cam_split<BF16>(y.w, h[3], l[3]);
                  *reinterpret_cast<uint2*>(dh + k) = make_uint2(h[0] | (static_cast<uint32_t>(h[1]) << 16), h[2] | (static_cast<uint32_t>(h[3]) << 16));
                  *reinterpret_cast<uint2*>(dl + k) = make_uint2(l[0] | (static_cast<uint32_t>(l[1]) << 16), l[2] | (static_cast<uint32_t>(l[3]) << 16));
                };
                if (P.ln) {                                               // row length 2048; KX is 2048 or 1024
                  float4 v[CAM_DIM / 128];
                  float s = 0.f;
#pragma unroll
                  for (int i = 0; i < CAM_DIM / 128; ++i) {
                    v[i] = *reinterpret_cast<const float4*>(row + (lane + 32 * i) * 4);
                    s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
                  }
                  const float mean = warp_sum_f(s) * (1.0f / CAM_DIM);
                  float q = 0.f;
#pragma unroll
                  for (int i = 0; i < CAM_DIM / 128; ++i) {
                    const float a = v[i].x - mean, bq = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
                    q += (a * a + bq * bq) + (c * c + d * d);
                  }
                  const float rstd = rsqrtf(warp_sum_f(q) * (1.0f / CAM_DIM) + P.ln_eps);
#pragma unroll
                  for (int i = 0; i < CAM_DIM / 128; ++i) {
                    const int k = (lane + 32 * i) * 4;
                    if (k < k0 || k >= k0 + kn) continue;
                    float4 y = make_float4((v[i].x - mean) * rstd, (v[i].y - mean) * rstd, (v[i].z - mean) * rstd,
                                           (v[i].w - mean) * rstd);
                    if (P.ln == 1) {
                      const float4 ww = *reinterpret_cast<const float4*>(gam + k), bb = *reinterpret_cast<const float4*>(gam + CAM_DIM + k);
                      y.x = y.x * ww.x + bb.x; y.y = y.y * ww.y + bb.y; y.z = y.z * ww.z + bb.z; y.w = y.w * ww.w + bb.w;
                    }
                    put(k - k0, y);
                  }
                } else {
                  for (int k = lane * 4; k < kst; k += 128)              // P.K is a multiple of 4 (16, 1024, 2048, 8192)
                    put(k, (k0 + k < P.K) ? *reinterpret_cast<const float4*>(row + k0 + k) : make_float4(0.f, 0.f, 0.f, 0.f));
                }
              }
              named_bar_sync(2, 256);
              if (stamp && ch == 0) stamp[1] = cam_now();
            }
#pragma unroll
            for (int ti = 0; ti < 4; ++ti) {
              if (ti < ntl) {
            // ---- weight stages of this chunk (1024 k each)
            for (int ks = 0; ks < (kn + CAM_KS - 1) / CAM_KS; ++ks) {
              mbar_wait(&full[st], ph);
              if (prog.dbg_mode != 2) {
                const uint8_t* wst = sW + st * CAM_W_BYTES;
                const int steps = min(CAM_KS, kn - ks * CAM_KS + 15) / 16;      // k steps of 16 in this stage (64, or 1 for K = 16)
                for (int s16 = warp; s16 < steps; s16 += 8) {
                  const int kk = ks * CAM_KS + s16 * 16;                  // chunk-local k of this step
                  // A fragments: rows g (and g + 8 when more than 8 rows are staged), k = kk + 2 tq (+ 8)
                  const uint32_t ah0 = *reinterpret_cast<const uint32_t*>(xs + g * KXP + kk + 2 * tq);
                  const uint32_t ah2 = *reinterpret_cast<const uint32_t*>(xs + g * KXP + kk + 8 + 2 * tq);
                  const uint32_t al0 = *reinterpret_cast<const uint32_t*>(xlo + g * KXP + kk + 2 * tq);
                  const uint32_t al2 = *reinterpret_cast<const uint32_t*>(xlo + g * KXP + kk + 8 + 2 * tq);
                  uint32_t ah1 = 0, ah3 = 0, al1 = 0, al3 = 0;
                  if constexpr (MP == 16) {
                    ah1 = *reinterpret_cast<const uint32_t*>(xs + (g + 8) * KXP + kk + 2 * tq);
                    ah3 = *reinterpret_cast<const uint32_t*>(xs + (g + 8) * KXP + kk + 8 + 2 * tq);
                    al1 = *reinterpret_cast<const uint32_t*>(xlo + (g + 8) * KXP + kk + 2 * tq);
                    al3 = *reinterpret_cast<const uint32_t*>(xlo + (g + 8) * KXP + kk + 8 + 2 * tq);
                  }
                  // B fragments from the swizzled stage: k group (64 k) q64, 16-byte chunk (2 j) ^ (col & 7), + 4 tq bytes
                  const int q64 = s16 >> 2, j = (s16 & 3) * 2;
#pragma unroll
                  for (int c = 0; c < 2; ++c) {
                    const int col = c * 8 + g;
                    const uint8_t* wr = wst + q64 * (CAM_COLS * 128) + col * 128 + tq * 4;
                    const uint32_t b0 = *reinterpret_cast<const uint32_t*>(wr + ((j ^ (col & 7)) << 4));
                    const uint32_t b1 = *reinterpret_cast<const uint32_t*>(wr + (((j + 1) ^ (col & 7)) << 4));
                    cam_mma<BF16>(acc[ti][c], ah0, ah1, ah2, ah3, b0, b1);
                    cam_mma<BF16>(acc[ti][c], al0, al1, al2, al3, b0, b1);
                  }
                }
              }
              __syncwarp();
              if (lane == 0) mbar_arrive(&empty[st]);
              if (++st == CAM_STAGES) { st = 0; ph ^= 1; }
            }
              }
            }
          }
        }
#pragma unroll
        for (int ti = 0; ti < 4; ++ti) {
          if (ti >= ntl) break;
          const int t = cta + ti * G;
          // ---- reduce the 8 warps' k slices through shared memory; thread (m, c) finishes one output element
          named_bar_sync(2, 256);                                         // the previous tile's sums have been read
#pragma unroll
          for (int c = 0; c < 2; ++c) {
            float* r0 = red + (warp * 16 + g) * CAM_COLS + c * 8 + 2 * tq;
            *reinterpret_cast<float2*>(r0) = make_float2(acc[ti][c][0], acc[ti][c][1]);
            *reinterpret_cast<float2*>(r0 + 8 * CAM_COLS) = make_float2(acc[ti][c][2], acc[ti][c][3]);
          }
          named_bar_sync(2, 256);
          {
            const int m = tid / CAM_COLS, c = tid % CAM_COLS;
            float mine = 0.f;
#pragma unroll
            for (int wv = 0; wv < 8; ++wv) mine += red[(wv * 16 + m) * CAM_COLS + c];
            const int n = t * CAM_COLS + c;
            if (n < P.N && m < M) {
              float v = mine + (P.bias ? P.bias[n] : 0.f);
              if (P.act == 1) v = gelu_erf(v);
              else if (P.act == 4) v = v / (1.0f + expf(-v));
              if (P.gamma) v *= P.gamma[n];
              if (P.flags & CF_POSE_OUT) {
                if (it > 0) v += P.out[m * P.ldo + n];                    // pred += delta
                P.out2[(static_cast<long>(it) * M + m) * 9 + n] = n >= 7 ? relu_nan(v) : v;   // activate_pose
              } else if (P.resid) {
                v += P.resid[m * P.ldr + n];
              }
              P.out[m * P.ldo + n] = v;
            }
          }
        }
        if (P.ln == 1 && cta < tiles) {                                   // release the gamma | beta slot
          __syncwarp();
          if (lane == 0) mbar_arrive(&ln_empty[lslot]);
          if (++lslot == 2) { lslot = 0; lph ^= 1; }
        }
      } else if (P.type == PH_ATTN) {
        // one warp per (row, head): q . k_j over the S tokens of the row's scene, softmax, p . v
        const int items = M * CAM_HEADS;
        for (int i = cta * 8 + warp; i < items; i += G * 8) {
          const int m = i / CAM_HEADS, h = i % CAM_HEADS;
          const int b = m / prog.S;
          const float* qkv = P.x;
          const float4 q = *reinterpret_cast<const float4*>(qkv + m * P.ldx + h * CAM_HD + lane * 4);
          float s[16];
          float mx = -INFINITY;
#pragma unroll
          for (int j = 0; j < 16; ++j) {
            if (j < prog.S) {
              const float4 k = *reinterpret_cast<const float4*>(qkv + (b * prog.S + j) * P.ldx + CAM_DIM + h * CAM_HD + lane * 4);
              s[j] = warp_sum_f(q.x * k.x + q.y * k.y + q.z * k.z + q.w * k.w) * 0.08838834764831845f;   // 128^-0.5
              mx = fmaxf(mx, s[j]);
            }
          }
          float sum = 0.f;
          float4 o = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
          for (int j = 0; j < 16; ++j) {
            if (j < prog.S) {
              const float e = expf(s[j] - mx);
              sum += e;
              const float4 v = *reinterpret_cast<const float4*>(qkv + (b * prog.S + j) * P.ldx + 2 * CAM_DIM + h * CAM_HD + lane * 4);
              o.x = fmaf(e, v.x, o.x); o.y = fmaf(e, v.y, o.y); o.z = fmaf(e, v.z, o.z); o.w = fmaf(e, v.w, o.w);
            }
          }
          const float inv = 1.0f / sum;
          *reinterpret_cast<float4*>(P.out + m * P.ldo + h * CAM_HD + lane * 4) = make_float4(o.x * inv, o.y * inv, o.z * inv, o.w * inv);
        }
      } else if (P.type == PH_MODULATE) {
        // x = gate * (ptn * (1 + scale) + shift) + pt   (camera_head.py:119-121, modulate :157-161); mod = [shift|scale|gate]
        for (int i = cta * 256 + tid; i < M * CAM_DIM; i += G * 256) {
          const int m = i / CAM_DIM, k = i % CAM_DIM;
          const float* mod = P.x + m * P.ldx;
          P.out[m * P.ldo + k] = mod[2 * CAM_DIM + k] * (P.x2[i] * (1.0f + mod[CAM_DIM + k]) + mod[k]) + P.x3[i];
        }
      } else {   // PH_LNROWS: out[m] = LayerNorm(x[m]) over 2048, one warp per row
        for (int m = cta * 8 + warp; m < M; m += G * 8) {
          const float* row = P.x + m * P.ldx;
          float v[CAM_DIM / 32];
          float s = 0.f;
#pragma unroll
          for (int i = 0; i < CAM_DIM / 128; ++i) {
            const float4 a = *reinterpret_cast<const float4*>(row + (lane + 32 * i) * 4);
            v[4 * i] = a.x; v[4 * i + 1] = a.y; v[4 * i + 2] = a.z; v[4 * i + 3] = a.w;
            s += (a.x + a.y) + (a.z + a.w);
          }
          const float mean = warp_sum_f(s) * (1.0f / CAM_DIM);
          float q = 0.f;
#pragma unroll
          for (int i = 0; i < CAM_DIM / 32; ++i) { const float d = v[i] - mean; q += d * d; }
          const float rstd = rsqrtf(warp_sum_f(q) * (1.0f / CAM_DIM) + P.ln_eps);
#pragma unroll
          for (int i = 0; i < CAM_DIM / 128; ++i) {
            const int k = (lane + 32 * i) * 4;
            float4 y = make_float4((v[4 * i] - mean) * rstd, (v[4 * i + 1] - mean) * rstd, (v[4 * i + 2] - mean) * rstd,
                                   (v[4 * i + 3] - mean) * rstd);
            if (P.ln == 1) {
              const float4 ww = *reinterpret_cast<const float4*>(P.ln_w + k), bb = *reinterpret_cast<const float4*>(P.ln_b + k);
              y.x = y.x * ww.x + bb.x; y.y = y.y * ww.y + bb.y; y.z = y.z * ww.z + bb.z; y.w = y.w * ww.w + bb.w;
            }
            *reinterpret_cast<float4*>(P.out + m * P.ldo + k) = y;
          }
        }
      }
      if (stamp) stamp[2] = cam_now();
      cam_grid_sync(prog.barrier, target);
      if (stamp) stamp[3] = cam_now() | (static_cast<unsigned long long>(wait_clk >> 6) << 48);   // + cycles/64 spent waiting for weights
    }
}

}  // namespace iggt

using namespace iggt;

namespace {
struct CamWs {          // workspace layout (floats), M rows each
  float *pt, *ptn, *e, *mod, *x, *qkv, *o, *f, *hdn, *pred;
  unsigned* barrier;
};
int64_t cam_ws_floats(int M) { return static_cast<int64_t>(M) * (5 * CAM_DIM + 2 * 3 * CAM_DIM + 4 * CAM_DIM + 1024 + 16); }
}  // namespace

extern "C" int64_t iggt_camera_head_workspace(int M) {
  if (M <= 0) return -1;
  return cam_ws_floats(M) * 4 + 256 + 8 * CAM_MAX_PHASES * 4 * 8;     // + debug stamps [8 iters][32 phases][4]
}

extern "C" int iggt_camera_head(const iggt_camera_weights* w, const float* tokens, int64_t ld_tokens, float* out,
                                void* workspace, int64_t ws_bytes, int B, int S, int iters, int dtype,
                                iggt_stream_t stream) {
  if (!w || !tokens || !out || !workspace || B <= 0 || S <= 0 || iters <= 0) return -1;
  const int M = B * S;
  if (M > 16 || S > 16) return -7;                      // larger batches: the per-layer launches (iggt_skinny_gemm ...)
  if (dtype != 0 && dtype != 1) return -3;
  if (ws_bytes < iggt_camera_head_workspace(M) || (reinterpret_cast<uintptr_t>(workspace) & 15) || (ld_tokens % 4)) return -6;
  cudaStream_t s = (cudaStream_t)stream;
  CamWs ws;
  float* p = reinterpret_cast<float*>(workspace);
  ws.pt = p; p += M * CAM_DIM;
  ws.ptn = p; p += M * CAM_DIM;
  ws.e = p; p += M * CAM_DIM;
  ws.x = p; p += M * CAM_DIM;
  ws.o = p; p += M * CAM_DIM;
  ws.mod = p; p += M * 3 * CAM_DIM;
  ws.qkv = p; p += M * 3 * CAM_DIM;
  ws.f = p; p += M * 4 * CAM_DIM;
  ws.hdn = p; p += M * 1024;
  ws.pred = p; p += M * 16;
  ws.barrier = reinterpret_cast<unsigned*>((reinterpret_cast<uintptr_t>(p) + 127) & ~static_cast<uintptr_t>(127));
  static const int dbg_env = [] { const char* e = getenv("IGGT_CAMERA_DEBUG"); return e ? atoi(e) : 0; }();
  cudaError_t e = cudaMemsetAsync(ws.barrier, 0, 4, s);
  if (e != cudaSuccess) return (int)e;
  e = cudaMemsetAsync(ws.pred, 0, M * 16 * 4, s);       // columns 9..15 of `pred` are the zero padding of embed_pose's K
  if (e != cudaSuccess) return (int)e;

  CamProgram prog{};
  prog.iters = iters; prog.M = M; prog.Mpad = M <= 8 ? 8 : 16; prog.B = B; prog.S = S; prog.barrier = ws.barrier;
  prog.dbg = (dbg_env && iters <= 8) ? reinterpret_cast<unsigned long long*>(ws.barrier + 32) : nullptr;   // +128 B
  prog.dbg_mode = dbg_env;
  const TmDtype dt = dtype ? TM_BF16 : TM_F16;
  int nmaps = 0;
  // weights [N, K] row-major seen as {64 k, N, K / 64} (128B-swizzled rows of 64 k): one box = 16 columns x 1024 k
  auto add_map = [&](const void* W, int N, int K) -> int {
    const int k64 = K < 64 ? K : 64;                       // embed_pose: K = 16
    uint64_t dims[3] = {(uint64_t)k64, (uint64_t)N, (uint64_t)((K + 63) / 64)};
    uint64_t str[2] = {(uint64_t)K * 2, (uint64_t)128};
    uint32_t box[3] = {64, (uint32_t)CAM_COLS, (uint32_t)(CAM_KS / 64)};
    if (nmaps >= CAM_MAX_MAPS || make_tmap(&prog.maps[nmaps], dt, 3, W, dims, str, box, true)) return -1;
    return nmaps++;
  };
  int np = 0;
  bool bad = false;
  auto gemm = [&](const void* W, int N, int K, const float* x, long ldx, const float* bias, float* o, long ldo, int act) -> CamPhase& {
    CamPhase& P = prog.ph[np++];
    P = CamPhase{};
    P.type = PH_GEMM; P.N = N; P.K = K; P.x = x; P.ldx = ldx; P.bias = bias; P.out = o; P.ldo = ldo; P.act = act;
    P.tm = add_map(W, N, K);
    if (P.tm < 0) bad = true;
    return P;
  };
  auto ln = [](CamPhase& P, const float* lw, const float* lb, float eps) { P.ln = lw ? 1 : 2; P.ln_w = lw; P.ln_b = lb; P.ln_eps = eps; };
  {   // pose_tokens = token_norm(tokens[:, :, 0]); adaln_norm(pose_tokens)  (camera_head.py:99-100, :117)
    CamPhase& P0 = prog.ph[np++]; P0 = CamPhase{};
    P0.type = PH_LNROWS; P0.x = tokens; P0.ldx = ld_tokens; P0.out = ws.pt; P0.ldo = CAM_DIM; P0.flags = CF_ONCE;
    ln(P0, w->tok_w, w->tok_b, 1e-5f);
    CamPhase& P1 = prog.ph[np++]; P1 = CamPhase{};
    P1.type = PH_LNROWS; P1.x = ws.pt; P1.ldx = CAM_DIM; P1.out = ws.ptn; P1.ldo = CAM_DIM; P1.flags = CF_ONCE;
    ln(P1, nullptr, nullptr, 1e-6f);
  }
  {   // module_input = embed_pose(prev or empty); shift / scale / gate = Linear(SiLU(.))  (camera_head.py:105-115)
    CamPhase& E = gemm(w->emb_w, CAM_DIM, 16, ws.pred, 16, w->emb_b, ws.e, CAM_DIM, 4);
    E.flags = CF_EMBED_IN; E.x2 = w->empty;
    gemm(w->mod_w, 3 * CAM_DIM, CAM_DIM, ws.e, CAM_DIM, w->mod_b, ws.mod, 3 * CAM_DIM, 0);
    CamPhase& Mo = prog.ph[np++]; Mo = CamPhase{};
    Mo.type = PH_MODULATE; Mo.x = ws.mod; Mo.ldx = 3 * CAM_DIM; Mo.x2 = ws.ptn; Mo.x3 = ws.pt; Mo.out = ws.x; Mo.ldo = CAM_DIM;
  }
  for (int b = 0; b < 4; ++b) {   // trunk blocks (layers/block.py:105-106, LayerScale init 0.01)
    const auto& k = w->blk[b];
    CamPhase& Q = gemm(k.qkv_w, 3 * CAM_DIM, CAM_DIM, ws.x, CAM_DIM, k.qkv_b, ws.qkv, 3 * CAM_DIM, 0);
    ln(Q, k.n1w, k.n1b, 1e-5f);
    CamPhase& A = prog.ph[np++]; A = CamPhase{};
    A.type = PH_ATTN; A.x = ws.qkv; A.ldx = 3 * CAM_DIM; A.out = ws.o; A.ldo = CAM_DIM;
    CamPhase& Pr = gemm(k.proj_w, CAM_DIM, CAM_DIM, ws.o, CAM_DIM, k.proj_b, ws.x, CAM_DIM, 0);
    Pr.gamma = k.ls1; Pr.resid = ws.x; Pr.ldr = CAM_DIM;
    CamPhase& F1 = gemm(k.fc1_w, 4 * CAM_DIM, CAM_DIM, ws.x, CAM_DIM, k.fc1_b, ws.f, 4 * CAM_DIM, 1);
    ln(F1, k.n2w, k.n2b, 1e-5f);
    CamPhase& F2 = gemm(k.fc2_w, CAM_DIM, 4 * CAM_DIM, ws.f, 4 * CAM_DIM, k.fc2_b, ws.x, CAM_DIM, 0);
    F2.gamma = k.ls2; F2.resid = ws.x; F2.ldr = CAM_DIM;
  }
  {   // pose_branch(trunk_norm(.)) and the accumulation / activation  (camera_head.py:124-139)
    CamPhase& B1 = gemm(w->pb1_w, 1024, CAM_DIM, ws.x, CAM_DIM, w->pb1_b, ws.hdn, 1024, 1);
    ln(B1, w->trk_w, w->trk_b, 1e-5f);
    CamPhase& B2 = gemm(w->pb2_w, 9, 1024, ws.hdn, 1024, w->pb2_b, ws.pred, 16, 0);
    B2.flags = CF_POSE_OUT; B2.out2 = out;
  }
  if (bad || np > CAM_MAX_PHASES) return -4;
  prog.n_phases = np;

  const int sms = device_sm_count();
  const int grid = sms >= 128 ? 128 : sms;           // 128 | every tile count of the head (128 / 384 / 512): no ragged wave
  // the consumers keep at most 4 tiles of a phase in registers (acc[4]) while the producer streams the stages of every
  // tile it assigns to the CTA: below 128 SMs (fc1: 512 tiles) a CTA would own 5 and the weight ring would fall out of
  // step, so such devices take the per-layer launches
  int max_tiles = 0;
  for (int i = 0; i < np; ++i)
    if (prog.ph[i].type == PH_GEMM && (prog.ph[i].N + CAM_COLS - 1) / CAM_COLS > max_tiles)
      max_tiles = (prog.ph[i].N + CAM_COLS - 1) / CAM_COLS;
  if ((max_tiles + grid - 1) / grid > 4) return -7;
  void (*kern)(const CamProgram) = nullptr;
  if (prog.Mpad == 8) kern = dtype ? camera_head_kernel<true, 8> : camera_head_kernel<false, 8>;
  else kern = dtype ? camera_head_kernel<true, 16> : camera_head_kernel<false, 16>;
  static DeviceOnce once;
  if (once.first()) {
    cudaFuncSetAttribute(camera_head_kernel<true, 8>, cudaFuncAttributeMaxDynamicSharedMemorySize, CAM_SMEM);
    cudaFuncSetAttribute(camera_head_kernel<false, 8>, cudaFuncAttributeMaxDynamicSharedMemorySize, CAM_SMEM);
    cudaFuncSetAttribute(camera_head_kernel<true, 16>, cudaFuncAttributeMaxDynamicSharedMemorySize, CAM_SMEM);
    cudaFuncSetAttribute(camera_head_kernel<false, 16>, cudaFuncAttributeMaxDynamicSharedMemorySize, CAM_SMEM);
  }
  // every CTA must be resident for the device-wide barrier: a cooperative launch guarantees it (or fails loudly)
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(CAM_THREADS);
  cfg.dynamicSmemBytes = CAM_SMEM;
  cfg.stream = s;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeCooperative;
  at[0].val.cooperative = 1;
  cfg.attrs = at;
  cfg.numAttrs = 1;
  return (int)cudaLaunchKernelEx(&cfg, kern, prog);
}
