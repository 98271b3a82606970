// The part head's two 8x8-window attentions on tensor cores (mma.sync.m16n8k16, fp32 accumulation):
//   OCAB  (iggt/heads/window_sa.py:271-319): 64 queries x 144 overlapping keys x d = 64 per (window, head), relative-position
//         bias, the reference's scrambled query windows (SURVEY F5);
//   HAB   (iggt/heads/window_sa.py:201-227 + heads/block.py:113-130): 64 x 64 x d = 32 per (window, head).
// One CTA of 4 warps per (image, window, head); warp w owns query rows [16 w, 16 w + 16): S = Q K^T in registers (C
// fragments), softmax over the fragment rows (quad shuffles), P re-used as the A operand of P V without leaving registers
// - split into hi + lo 16-bit operands so that the probabilities keep fp32-like precision - and V consumed through
// ldmatrix.trans.  K / V / Q tiles are staged in shared memory with 16-byte rows padded by 16 bytes (bank-conflict-free
// fragment loads); K / V arrive as 16-byte vectors.
#pragma once
#include "ptx.cuh"

namespace iggt {

template <bool BF16>
__device__ __forceinline__ void wa_mma(float (&d)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
  if constexpr (BF16)
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]) : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
  else
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]) : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}
// two 8x8 16-bit matrices, transposed on the way: lanes 0-7 / 8-15 give the row addresses of matrix 0 / 1; thread (g, t)
// receives {M[2t][g], M[2t+1][g]} of each - the B fragment of P V when the rows are keys and the columns head dims
__device__ __forceinline__ void wa_ldsm_x2_trans(uint32_t& r0, uint32_t& r1, const void* row_ptr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x2.trans.shared.b16 {%0, %1}, [%2];" : "=r"(r0), "=r"(r1) : "r"(smem_u32(row_ptr)));
}
template <bool BF16>
__device__ __forceinline__ float wa_unpack_lo(uint32_t u) {
  if constexpr (BF16) return __uint_as_float(u << 16);
  else return __half2float(__ushort_as_half(static_cast<uint16_t>(u & 0xFFFF)));
}
template <bool BF16>
__device__ __forceinline__ float wa_unpack_hi(uint32_t u) {
  if constexpr (BF16) return __uint_as_float(u & 0xFFFF0000u);
  else return __half2float(__ushort_as_half(static_cast<uint16_t>(u >> 16)));
}
// (p0, p1) -> hi pair and lo pair with hi + lo = p to ~2^-22 (fp16) / 2^-16 (bf16)
template <bool BF16>
__device__ __forceinline__ void wa_split2(float p0, float p1, uint32_t& hi, uint32_t& lo) {
  hi = pack16x2<BF16>(p0, p1);
  lo = pack16x2<BF16>(p0 - wa_unpack_lo<BF16>(hi), p1 - wa_unpack_hi<BF16>(hi));
}

// Softmax over the NT n-tiles of a warp's S fragments (rows g and g + 8 of the warp's 16 query rows), then O = P V with
// V in shared memory as [keys][VP 16-bit] (row pitch VP, head dim DT * 8).  Returns O un-normalised and 1 / row sums.
template <bool BF16, int NT, int DT, int VP>
__device__ __forceinline__ void wa_softmax_pv(float (&S)[NT][4], const uint16_t* sV, int lane, float (&O)[DT][4], float& inv0, float& inv1) {
  float m0 = -INFINITY, m1 = -INFINITY;
#pragma unroll
  for (int n = 0; n < NT; ++n) { m0 = fmaxf(m0, fmaxf(S[n][0], S[n][1])); m1 = fmaxf(m1, fmaxf(S[n][2], S[n][3])); }
  m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, 1)); m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, 2));
  m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, 1)); m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, 2));
  float l0 = 0.f, l1 = 0.f;
#pragma unroll
  for (int n = 0; n < NT; ++n) {
    S[n][0] = __expf(S[n][0] - m0); S[n][1] = __expf(S[n][1] - m0);
    S[n][2] = __expf(S[n][2] - m1); S[n][3] = __expf(S[n][3] - m1);
    l0 += S[n][0] + S[n][1]; l1 += S[n][2] + S[n][3];
  }
  l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  inv0 = 1.0f / l0; inv1 = 1.0f / l1;
#pragma unroll
  for (int n = 0; n < DT; ++n)
#pragma unroll
    for (int i = 0; i < 4; ++i) O[n][i] = 0.f;
#pragma unroll
  for (int j = 0; j < NT / 2; ++j) {                       // 16 keys per step: n-tiles 2j, 2j + 1 of S are the A operand
    uint32_t h0, h1, h2, h3, l_0, l_1, l_2, l_3;
    wa_split2<BF16>(S[2 * j][0], S[2 * j][1], h0, l_0);
    wa_split2<BF16>(S[2 * j][2], S[2 * j][3], h1, l_1);
    wa_split2<BF16>(S[2 * j + 1][0], S[2 * j + 1][1], h2, l_2);
    wa_split2<BF16>(S[2 * j + 1][2], S[2 * j + 1][3], h3, l_3);
#pragma unroll
    for (int n = 0; n < DT; ++n) {
      uint32_t b0, b1;
      wa_ldsm_x2_trans(b0, b1, sV + (16 * j + (lane & 15)) * VP + 8 * n);
      wa_mma<BF16>(O[n], h0, h1, h2, h3, b0, b1);
      wa_mma<BF16>(O[n], l_0, l_1, l_2, l_3, b0, b1);
    }
  }
}

// ------------------------------------------------------------------------------------------------ HAB window attention
constexpr int WA_P = 40;                                   // 32 head dims + 8: 80-byte rows
template <bool BF16>
__global__ void __launch_bounds__(128)
window_attention_tc_kernel(const uint16_t* __restrict__ qkv, uint16_t* __restrict__ out, int h, int w) {
  __shared__ __align__(16) uint16_t sQ[64 * WA_P], sK[64 * WA_P], sV[64 * WA_P];
  const int nwx = w / 8, nwy = h / 8;
  const int head = blockIdx.x % 4;
  const int win = (blockIdx.x / 4) % (nwx * nwy);
  const int b = blockIdx.x / (4 * nwx * nwy);
  const int wy = win / nwx, wx = win % nwx;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
  for (int i = tid; i < 64 * 4; i += 128) {                // token x 16-byte chunk of the head's 32 dims
    const int tok = i >> 2, c = i & 3;
    const int64_t pix = (static_cast<int64_t>(b) * h + wy * 8 + (tok >> 3)) * w + wx * 8 + (tok & 7);
    const uint4* p = reinterpret_cast<const uint4*>(qkv + pix * 384 + head * 32 + c * 8);
    *reinterpret_cast<uint4*>(sQ + tok * WA_P + c * 8) = __ldg(p);
    *reinterpret_cast<uint4*>(sK + tok * WA_P + c * 8) = __ldg(p + 16);      // + 128 channels
    *reinterpret_cast<uint4*>(sV + tok * WA_P + c * 8) = __ldg(p + 32);      // + 256 channels
  }
  __syncthreads();
  const int r0 = warp * 16;
  float S[8][4];
#pragma unroll
  for (int n = 0; n < 8; ++n)
#pragma unroll
    for (int i = 0; i < 4; ++i) S[n][i] = 0.f;
#pragma unroll
  for (int s = 0; s < 2; ++s) {                            // d = 32: two k steps
    const uint32_t a0 = *reinterpret_cast<const uint32_t*>(sQ + (r0 + g) * WA_P + 16 * s + 2 * t);
    const uint32_t a1 = *reinterpret_cast<const uint32_t*>(sQ + (r0 + g + 8) * WA_P + 16 * s + 2 * t);
    const uint32_t a2 = *reinterpret_cast<const uint32_t*>(sQ + (r0 + g) * WA_P + 16 * s + 8 + 2 * t);
    const uint32_t a3 = *reinterpret_cast<const uint32_t*>(sQ + (r0 + g + 8) * WA_P + 16 * s + 8 + 2 * t);
#pragma unroll
    for (int n = 0; n < 8; ++n) {
      const uint32_t b0 = *reinterpret_cast<const uint32_t*>(sK + (8 * n + g) * WA_P + 16 * s + 2 * t);
      const uint32_t b1 = *reinterpret_cast<const uint32_t*>(sK + (8 * n + g) * WA_P + 16 * s + 8 + 2 * t);
      wa_mma<BF16>(S[n], a0, a1, a2, a3, b0, b1);
    }
  }
  const float scale = 0.17677669529663687f;                // 32^-0.5
#pragma unroll
  for (int n = 0; n < 8; ++n)
#pragma unroll
    for (int i = 0; i < 4; ++i) S[n][i] *= scale;
  float O[4][4], inv0, inv1;
  wa_softmax_pv<BF16, 8, 4, WA_P>(S, sV, lane, O, inv0, inv1);
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const int tok = r0 + g + 8 * hh;
    const int64_t pix = (static_cast<int64_t>(b) * h + wy * 8 + (tok >> 3)) * w + wx * 8 + (tok & 7);
    const float inv = hh ? inv1 : inv0;
#pragma unroll
    for (int n = 0; n < 4; ++n)
      *reinterpret_cast<uint32_t*>(out + pix * 128 + head * 32 + 8 * n + 2 * t) = pack16x2<BF16>(O[n][2 * hh] * inv, O[n][2 * hh + 1] * inv);
  }
}

// ------------------------------------------------------------------------------------------------ OCAB
constexpr int OA_P = 72;                                   // 64 head dims + 8: 144-byte rows
constexpr int OA_SMEM = (64 + 144 + 144) * OA_P * 2;       // Q, K, V tiles: 50 688 bytes
template <bool BF16>
__global__ void __launch_bounds__(128)
ocab_attention_tc_kernel(const uint16_t* __restrict__ Q, const uint16_t* __restrict__ K, const uint16_t* __restrict__ V,
                         const float* __restrict__ table, const int* __restrict__ rpi, uint16_t* __restrict__ out, int h, int w) {
  extern __shared__ __align__(16) uint16_t oa_sm[];
  uint16_t* sQ = oa_sm;                                    // [64][72]
  uint16_t* sK = sQ + 64 * OA_P;                           // [144][72]
  uint16_t* sV = sK + 144 * OA_P;                          // [144][72]
  const int nwx = w / 8, nwy = h / 8;
  const int head = blockIdx.x % 4;
  const int win = (blockIdx.x / 4) % (nwx * nwy);
  const int b = blockIdx.x / (4 * nwx * nwy);
  const int wy = win / nwx, wx = win % nwx;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
  // scrambled query gather (the reference partitions the (b, c, h, w)-permuted Q with a (b, h, w, c) partition, SURVEY F5)
  for (int i = tid; i < 64 * 64; i += 128) {
    const int tq = i >> 6, d = i & 63;
    int64_t L = (static_cast<int64_t>(win) * 64 + tq) * 256 + head * 64 + d;
    const int x = static_cast<int>(L % w); L /= w;
    const int yi = static_cast<int>(L % 8); L /= 8;
    const int ci = static_cast<int>(L % 8); L /= 8;
    const int yb = static_cast<int>(L % nwy); L /= nwy;
    const int cb = static_cast<int>(L);
    sQ[tq * OA_P + d] = __ldg(Q + ((static_cast<int64_t>(b) * h + yb * 8 + yi) * w + x) * 256 + cb * 8 + ci);
  }
  // 12 x 12 key / value window around the 8 x 8 query window, zeros outside the map: 16-byte vectors
  for (int i = tid; i < 144 * 8; i += 128) {
    const int j = i >> 3, c = i & 7;
    const int yy = wy * 8 - 2 + j / 12, xx = wx * 8 - 2 + j % 12;
    uint4 kv = make_uint4(0u, 0u, 0u, 0u), vv = kv;
    if (yy >= 0 && yy < h && xx >= 0 && xx < w) {
      const int64_t off = ((static_cast<int64_t>(b) * h + yy) * w + xx) * 256 + head * 64 + c * 8;
      kv = __ldg(reinterpret_cast<const uint4*>(K + off));
      vv = __ldg(reinterpret_cast<const uint4*>(V + off));
    }
    *reinterpret_cast<uint4*>(sK + j * OA_P + c * 8) = kv;
    *reinterpret_cast<uint4*>(sV + j * OA_P + c * 8) = vv;
  }
  __syncthreads();
  const int r0 = warp * 16;
  float S[18][4];
#pragma unroll
  for (int n = 0; n < 18; ++n)
#pragma unroll
    for (int i = 0; i < 4; ++i) S[n][i] = 0.f;
#pragma unroll
  for (int s = 0; s < 4; ++s) {                            // d = 64: four k steps
    const uint32_t a0 = *reinterpret_cast<const uint32_t*>(sQ + (r0 + g) * OA_P + 16 * s + 2 * t);
    const uint32_t a1 = *reinterpret_cast<const uint32_t*>(sQ + (r0 + g + 8) * OA_P + 16 * s + 2 * t);
    const uint32_t a2 = *reinterpret_cast<const uint32_t*>(sQ + (r0 + g) * OA_P + 16 * s + 8 + 2 * t);
    const uint32_t a3 = *reinterpret_cast<const uint32_t*>(sQ + (r0 + g + 8) * OA_P + 16 * s + 8 + 2 * t);
#pragma unroll
    for (int n = 0; n < 18; ++n) {
      const uint32_t b0 = *reinterpret_cast<const uint32_t*>(sK + (8 * n + g) * OA_P + 16 * s + 2 * t);
      const uint32_t b1 = *reinterpret_cast<const uint32_t*>(sK + (8 * n + g) * OA_P + 16 * s + 8 + 2 * t);
      wa_mma<BF16>(S[n], a0, a1, a2, a3, b0, b1);
    }
  }
  // scores = (q * 64^-0.5) k^T + table[rpi[t, j]][head]
#pragma unroll
  for (int n = 0; n < 18; ++n)
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int row = r0 + g + 8 * (i >> 1), col = 8 * n + 2 * t + (i & 1);
      S[n][i] = fmaf(S[n][i], 0.125f, __ldg(table + __ldg(rpi + row * 144 + col) * 4 + head));
    }
  float O[8][4], inv0, inv1;
  wa_softmax_pv<BF16, 18, 8, OA_P>(S, sV, lane, O, inv0, inv1);
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const int tok = r0 + g + 8 * hh;
    const int yy = wy * 8 + (tok >> 3), xx = wx * 8 + (tok & 7);
    uint16_t* dst = out + ((static_cast<int64_t>(b) * h + yy) * w + xx) * 256 + head * 64 + 2 * t;
    const float inv = hh ? inv1 : inv0;
#pragma unroll
    for (int n = 0; n < 8; ++n)
      *reinterpret_cast<uint32_t*>(dst + 8 * n) = pack16x2<BF16>(O[n][2 * hh] * inv, O[n][2 * hh + 1] * inv);
  }
}

}  // namespace iggt
