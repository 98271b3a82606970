// Inline-PTX wrappers for the sm_90a features every kernel in this library uses:
// mbarrier, TMA (cp.async.bulk.tensor), wgmma (warpgroup MMA from shared-memory descriptors) and proxy fences.
// Nothing here is a port: the reference (lifuguan/IGGT_official) has no native code on this path
// (SURVEY.md §2.2); these are the building blocks of the Hopper-native kernels.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace iggt {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31; }

__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "elect.sync _|P, 0xffffffff;\n\t"
      "selp.b32 %0, 1, 0, P;\n\t}\n"
      : "=r"(pred));
  return pred != 0;
}

// ---------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
      "selp.b32 %0, 1, 0, P;\n\t}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}

// ---------------------------------------------------------------- fences
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}
// signal a named barrier without waiting: the shared-memory writes before it are visible to the threads that bar.sync
// on it (producer / consumer hand-off between warpgroups)
__device__ __forceinline__ void named_bar_arrive(uint32_t id, uint32_t nthreads) {
  asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// ---------------------------------------------------------------- register reallocation between warpgroups
// Executed by all four warps of a warpgroup: lower / raise the per-thread register limit of the warpgroup (a multiple
// of 8 in [24, 256]); registers one warpgroup gives back can be taken by another of the same CTA.
template <uint32_t N>
__device__ __forceinline__ void reg_dealloc() {
  asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N));
}
template <uint32_t N>
__device__ __forceinline__ void reg_alloc() {
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N));
}

// ---------------------------------------------------------------- TMA
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem, const CUtensorMap* m, uint64_t* bar,
                                            int32_t c0, int32_t c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4}], [%2];" ::"r"(smem_u32(smem)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* smem, const CUtensorMap* m, uint64_t* bar,
                                            int32_t c0, int32_t c1, int32_t c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(smem_u32(smem)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* smem, const CUtensorMap* m, uint64_t* bar,
                                            int32_t c0, int32_t c1, int32_t c2, int32_t c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5, %6}], [%2];" ::"r"(smem_u32(smem)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
// plain (non-tensor) bulk copy global -> shared, completion counted on an mbarrier; 16-byte aligned, size % 16 == 0
__device__ __forceinline__ void tma_bulk_load_1d(void* smem, const void* gptr, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(smem)),
               "l"(reinterpret_cast<uint64_t>(gptr)), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* m, const void* smem, int32_t c0,
                                             int32_t c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(smem_u32(smem)), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void tma_store_3d(const CUtensorMap* m, const void* smem, int32_t c0, int32_t c1, int32_t c2) {
  asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(smem_u32(smem)), "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}
__device__ __forceinline__ void tma_store_4d(const CUtensorMap* m, const void* smem, int32_t c0,
                                             int32_t c1, int32_t c2, int32_t c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::"l"(
          reinterpret_cast<uint64_t>(m)),
      "r"(smem_u32(smem)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
// x[tile] += smem (element type comes from the tensor map: fp32 for the residual stream)
__device__ __forceinline__ void tma_reduce_add_2d(const CUtensorMap* m, const void* smem,
                                                  int32_t c0, int32_t c1) {
  asm volatile(
      "cp.reduce.async.bulk.tensor.2d.global.shared::cta.add.tile.bulk_group [%0, {%2, %3}], [%1];" ::
          "l"(reinterpret_cast<uint64_t>(m)),
      "r"(smem_u32(smem)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_store_commit() {
  asm volatile("cp.async.bulk.commit_group;" ::: "memory");
}
template <int N>
__device__ __forceinline__ void tma_store_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
template <int N>
__device__ __forceinline__ void tma_store_wait_all() {
  asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}

// ---------------------------------------------------------------- wgmma (warpgroup MMA)
// All four warps of a warpgroup issue the same wgmma; the accumulator lives in registers, distributed as:
// thread t of the warpgroup (warp w = t / 32, lane l) holds rows 16 w + l / 4 and 16 w + l / 4 + 8; for every 8-column
// block j its fragment elements [4 j, 4 j + 1] are (row, 8 j + 2 (l % 4) + {0, 1}) and [4 j + 2, 4 j + 3] the same
// columns of row + 8.
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// keeps the compiler from moving accesses of accumulator registers across wgmma_wait
template <int R>
__device__ __forceinline__ void reg_fence(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// accumulator operand lists of the wrappers below: 8 fp32 fragment registers per macro
#define IGGT_D8(o) "+f"(d[o]), "+f"(d[o + 1]), "+f"(d[o + 2]), "+f"(d[o + 3]), "+f"(d[o + 4]), "+f"(d[o + 5]), \
                   "+f"(d[o + 6]), "+f"(d[o + 7])
// D (+)= A[smem desc] * B[smem desc], both operands K-major; d: this thread's accumulator fragment
#define IGGT_WGMMA_SS_32(T)                                                                                     \
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"                                               \
               "wgmma.mma_async.sync.aligned.m64n32k16.f32." T "." T " {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 0, 0;\n\t}\n" \
               : IGGT_D8(0), IGGT_D8(8)                                                                                          \
               : "l"(a_desc), "l"(b_desc), "r"(accumulate))
template <bool BF16>
__device__ __forceinline__ void wgmma_m64n32k16_ss(float (&d)[16], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
  if constexpr (BF16) IGGT_WGMMA_SS_32("bf16");
  else IGGT_WGMMA_SS_32("f16");
}
#define IGGT_WGMMA_SS_64(T)                                                                                     \
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"                                               \
               "wgmma.mma_async.sync.aligned.m64n64k16.f32." T "." T " {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t}\n" \
               : IGGT_D8(0), IGGT_D8(8), IGGT_D8(16), IGGT_D8(24)                                                                                          \
               : "l"(a_desc), "l"(b_desc), "r"(accumulate))
template <bool BF16>
__device__ __forceinline__ void wgmma_m64n64k16_ss(float (&d)[32], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
  if constexpr (BF16) IGGT_WGMMA_SS_64("bf16");
  else IGGT_WGMMA_SS_64("f16");
}
#define IGGT_WGMMA_SS_128(T)                                                                                     \
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"                                               \
               "wgmma.mma_async.sync.aligned.m64n128k16.f32." T "." T " {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t}\n" \
               : IGGT_D8(0), IGGT_D8(8), IGGT_D8(16), IGGT_D8(24), IGGT_D8(32), IGGT_D8(40), IGGT_D8(48), IGGT_D8(56)                                                                                          \
               : "l"(a_desc), "l"(b_desc), "r"(accumulate))
template <bool BF16>
__device__ __forceinline__ void wgmma_m64n128k16_ss(float (&d)[64], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
  if constexpr (BF16) IGGT_WGMMA_SS_128("bf16");
  else IGGT_WGMMA_SS_128("f16");
}
// D (+)= A[registers] * B[smem desc], B MN-major (transposed); a: the mma.sync-style A fragment of k16
#define IGGT_WGMMA_RS_TB_64(T)                                                                                   \
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"                                               \
               "wgmma.mma_async.sync.aligned.m64n64k16.f32." T "." T " {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1, 1;\n\t}\n" \
               : IGGT_D8(0), IGGT_D8(8), IGGT_D8(16), IGGT_D8(24)                                                                                          \
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc), "r"(accumulate))
template <bool BF16>
__device__ __forceinline__ void wgmma_m64n64k16_rs_tb(float (&d)[32], const uint32_t (&a)[4], uint64_t b_desc,
                                                      uint32_t accumulate) {
  if constexpr (BF16) IGGT_WGMMA_RS_TB_64("bf16");
  else IGGT_WGMMA_RS_TB_64("f16");
}

// 8-bit integer form: D (+)= A[smem desc] * B[smem desc] with unsigned bytes, s32 accumulators (exact integer sums);
// both operands K-major (8-bit wgmma has no transposed form), k32 per instruction = 32 bytes of the 128-byte swizzle row,
// so the descriptors step exactly as for the 16-bit k16 forms.  Same fragment layout as above, s32 elements.
template <int R>
__device__ __forceinline__ void reg_fence(uint32_t (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+r"(d[i])::"memory");
}
#define IGGT_R8(o) "+r"(d[o]), "+r"(d[o + 1]), "+r"(d[o + 2]), "+r"(d[o + 3]), "+r"(d[o + 4]), "+r"(d[o + 5]), \
                   "+r"(d[o + 6]), "+r"(d[o + 7])
__device__ __forceinline__ void wgmma_m64n8k32_u8(uint32_t (&d)[4], uint64_t a_desc, uint64_t b_desc) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %6, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n8k32.s32.u8.u8 {%0, %1, %2, %3}, %4, %5, p;\n\t}\n"
               : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3])
               : "l"(a_desc), "l"(b_desc), "r"(1));
}
__device__ __forceinline__ void wgmma_m64n64k32_u8(uint32_t (&d)[32], uint64_t a_desc, uint64_t b_desc) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n64k32.s32.u8.u8 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p;\n\t}\n"
               : IGGT_R8(0), IGGT_R8(8), IGGT_R8(16), IGGT_R8(24)
               : "l"(a_desc), "l"(b_desc), "r"(1));
}
__device__ __forceinline__ void wgmma_m64n128k32_u8(uint32_t (&d)[64], uint64_t a_desc, uint64_t b_desc) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
               "wgmma.mma_async.sync.aligned.m64n128k32.s32.u8.u8 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p;\n\t}\n"
               : IGGT_R8(0), IGGT_R8(8), IGGT_R8(16), IGGT_R8(24), IGGT_R8(32), IGGT_R8(40), IGGT_R8(48), IGGT_R8(56)
               : "l"(a_desc), "l"(b_desc), "r"(1));
}

// ---------------------------------------------------------------- descriptors
// wgmma shared-memory matrix descriptor (sm_90): start>>4 [0,14), LBO>>4 [16,30), SBO>>4 [32,46), layout type [62,64)
// (1 = SWIZZLE_128B).  128-byte swizzle: rows of 128 B (64 x 16-bit), 8-row atoms 1024 B apart (SBO); for a K-major
// operand the k16 steps inside an atom advance the start address by 32 B, for an MN-major operand SBO is the distance
// between groups of 8 k-rows.  Tiles must be 1024-byte aligned (base offset 0).
__device__ __forceinline__ uint64_t make_desc_sw128(uint32_t smem_addr, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);
  d |= static_cast<uint64_t>(1) << 16;                       // LBO (unused for 128B swizzle)
  d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= static_cast<uint64_t>(1) << 62;                       // SWIZZLE_128B
  return d;
}

// ---------------------------------------------------------------- small math helpers
__device__ __forceinline__ uint32_t pack_f16x2(float a, float b) {
  __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}
__device__ __forceinline__ uint32_t pack_bf16x2(float a, float b) {
  __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}
template <bool BF16>
__device__ __forceinline__ uint32_t pack16x2(float a, float b) {
  if constexpr (BF16) return pack_bf16x2(a, b);
  else return pack_f16x2(a, b);
}
// ReLU that keeps a NaN (torch.relu's behaviour; fmaxf would return 0 and hide an overflowed head activation)
__device__ __forceinline__ float relu_nan(float x) {
  float y;
  asm("max.NaN.f32 %0, %1, 0f00000000;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float gelu_erf(float x) {
  return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f));
}
__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// fp32 pairs: two IEEE-rounded fp32 operations (the pair form keeps the callers' arithmetic explicit and in order).
__device__ __forceinline__ float2 ffma2(float2 a, float2 b, float2 c) {
  return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
}
__device__ __forceinline__ float2 fadd2(float2 a, float2 b) {
  return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y));
}
__device__ __forceinline__ float2 fmul2(float2 a, float2 b) {
  return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y));
}
// Exact-erf GELU to ~2e-7 absolute: erf via Abramowitz-Stegun 7.1.26 (|err| <= 1.5e-7), branch-free,
// 2 MUFU + ~12 FMA-pipe instructions (libdevice erff is ~3x longer and serialises the epilogue).
__device__ __forceinline__ float gelu_fast(float x) {
  const float z = fabsf(x) * 0.70710678118654752440f;
  const float t = __fdividef(1.0f, fmaf(0.3275911f, z, 1.0f));
  float poly = fmaf(t, 1.061405429f, -1.453152027f);
  poly = fmaf(poly, t, 1.421413741f);
  poly = fmaf(poly, t, -0.284496736f);
  poly = fmaf(poly, t, 0.254829592f);
  poly *= t;
  const float e = ex2_approx(-z * z * 1.4426950408889634f);
  const float erf_abs = fmaf(-poly, e, 1.0f);
  const float hx = 0.5f * x;
  return fmaf(hx, copysignf(erf_abs, x), hx);
}

// Two GELUs at once on fp32 pairs: the same Abramowitz-Stegun evaluation as gelu_fast, operation for operation
// (every step is an IEEE-rounded fp32 multiply / fma, the two MUFU calls per element are unchanged).
__device__ __forceinline__ float2 gelu_fast2(float2 x) {
  const float2 ax = make_float2(fabsf(x.x), fabsf(x.y));
  const float2 z = fmul2(ax, make_float2(0.70710678118654752440f, 0.70710678118654752440f));
  const float2 den = ffma2(make_float2(0.3275911f, 0.3275911f), z, make_float2(1.0f, 1.0f));
  const float2 t = make_float2(__fdividef(1.0f, den.x), __fdividef(1.0f, den.y));
  float2 poly = ffma2(t, make_float2(1.061405429f, 1.061405429f), make_float2(-1.453152027f, -1.453152027f));
  poly = ffma2(poly, t, make_float2(1.421413741f, 1.421413741f));
  poly = ffma2(poly, t, make_float2(-0.284496736f, -0.284496736f));
  poly = ffma2(poly, t, make_float2(0.254829592f, 0.254829592f));
  poly = fmul2(poly, t);
  const float2 nz = make_float2(-z.x, -z.y);
  const float2 arg = fmul2(fmul2(nz, z), make_float2(1.4426950408889634f, 1.4426950408889634f));
  const float2 e = make_float2(ex2_approx(arg.x), ex2_approx(arg.y));
  const float2 erf_abs = ffma2(make_float2(-poly.x, -poly.y), e, make_float2(1.0f, 1.0f));
  const float2 hx = fmul2(make_float2(0.5f, 0.5f), x);
  return ffma2(hx, make_float2(copysignf(erf_abs.x, x.x), copysignf(erf_abs.y, x.y)), hx);
}


// Exact-erf GELU with ONE MUFU per element: erfc(z) = 2^(z * q(z)) for z = |x| / sqrt(2) in [0, 4.3] (q: degree-6
// least-squares fit of log2(erfc(z)) / z, max error 3e-5 in log2 units), so
//   gelu(x) = 0.5 x + 0.5 |x| (1 - erfc(z)) = hx - na + na * e,   na = -|hx|,  e = erfc(z),  hx = x / 2.
// Absolute error <= 1.6e-6, relative error <= 2.1e-5 wherever the result is an fp16 normal (the result is rounded to
// 16 bit right after, half an fp16 ulp = 2.4e-4).  2 MUFU per pair, against 4 for gelu_fast2 (reciprocal + exponential).
__device__ __forceinline__ float2 gelu_erfc2(float2 x) {
  const float2 hx = fmul2(x, make_float2(0.5f, 0.5f));
  const float2 na = make_float2(__uint_as_float(__float_as_uint(hx.x) | 0x80000000u),
                                __uint_as_float(__float_as_uint(hx.y) | 0x80000000u));
  float2 z = fmul2(na, make_float2(-1.4142135623730951f, -1.4142135623730951f));          // |x| / sqrt(2)
  z.x = fminf(z.x, 4.3f);
  z.y = fminf(z.y, 4.3f);
  float2 q = ffma2(make_float2(-1.5555357094854116e-05f, -1.5555357094854116e-05f), z,
                   make_float2(0.0004183394485153258f, 0.0004183394485153258f));
  q = ffma2(q, z, make_float2(-0.0048510609194636345f, -0.0048510609194636345f));
  q = ffma2(q, z, make_float2(0.03291909396648407f, 0.03291909396648407f));
  q = ffma2(q, z, make_float2(-0.1511300802230835f, -0.1511300802230835f));
  q = ffma2(q, z, make_float2(-0.9178327322006226f, -0.9178327322006226f));
  q = ffma2(q, z, make_float2(-1.6279296875f, -1.6279296875f));
  const float2 pz = fmul2(q, z);
  const float2 e = make_float2(ex2_approx(pz.x), ex2_approx(pz.y));
  const float2 s = ffma2(na, make_float2(-1.0f, -1.0f), hx);                                // hx + |hx|
  return ffma2(na, e, s);
}

}  // namespace iggt
