// Host-side TMA tensor-map construction (cuTensorMapEncodeTiled fetched through the runtime's
// driver entry point so the library has no link-time dependency on libcuda).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

namespace iggt {

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                  const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

inline EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres);
    if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || !p) {
      fprintf(stderr, "[iggt_b200] cuTensorMapEncodeTiled entry point unavailable (%d)\n", (int)e);
      return nullptr;
    }
    fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

enum TmDtype { TM_F16 = 0, TM_BF16 = 1, TM_F32 = 2, TM_U8 = 3 };
// element type of a 16-bit operand (the launchers' dtype, resolved by dispatch_dtype)
constexpr TmDtype tm16(bool bf16) { return bf16 ? TM_BF16 : TM_F16; }

// Generic rank<=4 tiled map. dims[0] is the contiguous dimension; strides_bytes[i] is the pitch of
// dimension i+1 (rank-1 entries). 128-byte swizzle; out-of-bounds elements read as zero.
inline int make_tmap(CUtensorMap* out, TmDtype dt, int rank, const void* base, const uint64_t* dims,
                     const uint64_t* strides_bytes, const uint32_t* box, bool swizzle128 = true) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return -1;
  CUtensorMapDataType cdt = dt == TM_F16    ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16
                            : dt == TM_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16
                            : dt == TM_U8   ? CU_TENSOR_MAP_DATA_TYPE_UINT8
                                            : CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
  cuuint64_t gdim[5];
  cuuint64_t gstr[5];
  cuuint32_t bx[5];
  cuuint32_t estr[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bx[i] = box[i];
    estr[i] = 1;
    if (i + 1 < rank) gstr[i] = strides_bytes[i];
  }
  CUresult r = fn(out, cdt, (cuuint32_t)rank, const_cast<void*>(base), gdim, gstr, bx, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE,
                  swizzle128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    fprintf(stderr, "[iggt_b200] cuTensorMapEncodeTiled failed: %d (rank %d dims %llu %llu box %u %u)\n",
            (int)r, rank, (unsigned long long)dims[0], (unsigned long long)(rank > 1 ? dims[1] : 0),
            box[0], rank > 1 ? box[1] : 0);
    return -2;
  }
  return 0;
}

// Row-major [rows, cols] matrix with row pitch ld (elements); box = {box_cols, box_rows}.
inline int make_tmap_2d(CUtensorMap* out, TmDtype dt, const void* base, uint64_t rows, uint64_t cols,
                        uint64_t ld, uint32_t box_cols, uint32_t box_rows) {
  uint64_t es = dt == TM_F32 ? 4 : dt == TM_U8 ? 1 : 2;
  uint64_t dims[2] = {cols, rows};
  uint64_t str[1] = {ld * es};
  uint32_t box[2] = {box_cols, box_rows};
  return make_tmap(out, dt, 2, base, dims, str, box);
}

}  // namespace iggt
