// Programmatic dependent launch (PDL) helpers.  Every hot kernel does its global-memory-free prologue (mbarrier
// init, tensor-map prefetch), then `griddep_wait()` before it touches global memory, and lets the
// next kernel in the stream begin ITS prologue early with `griddep_launch()`.  With ~730 back-to-back launches per
// forward (each short once the views are sharded over several GPUs) the launch latency and prologues are
// otherwise exposed.  IGGT_PDL=0 falls back to plain stream-ordered launches.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>
#include <initializer_list>
#include <type_traits>
#include <utility>

namespace iggt {

__device__ __forceinline__ void griddep_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void griddep_launch() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// Per-device caches (ADVICE r1: a second device in the same process must get its own cudaFuncSetAttribute opt-in and
// its own SM count).  kMaxDevices bounds the tables; an out-of-range ordinal is simply never cached.
constexpr int kMaxDevices = 64;
inline int current_device() {
  int d = 0;
  cudaGetDevice(&d);
  return d;
}
// first() is true at the first call on each device, and again after reset_current() on that device
struct DeviceOnce {
  bool done[kMaxDevices] = {};
  bool first() {
    const int d = current_device();
    if (d < 0 || d >= kMaxDevices) return true;
    if (done[d]) return false;
    done[d] = true;
    return true;
  }
  void reset_current() {          // configuration failed: try again at the next launch
    const int d = current_device();
    if (d >= 0 && d < kMaxDevices) done[d] = false;
  }
};
// Lets each of `Kernels` use `bytes` of dynamic shared memory on the current device (once per device).  Returns the
// first failing cudaError_t and forgets the attempt, so the next launch tries again instead of failing with a launch
// error that hides the cause.
template <auto... Kernels>
inline cudaError_t opt_in_smem(size_t bytes) {
  static DeviceOnce once;
  if (!once.first()) return cudaSuccess;
  for (const void* k : {reinterpret_cast<const void*>(Kernels)...}) {
    const cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(bytes));
    if (e != cudaSuccess) {
      once.reset_current();
      return e;
    }
  }
  return cudaSuccess;
}
inline int device_sm_count() {
  static int n[kMaxDevices] = {};
  const int d = current_device();
  if (d < 0 || d >= kMaxDevices) return 132;
  if (!n[d]) {
    cudaDeviceGetAttribute(&n[d], cudaDevAttrMultiProcessorCount, d);
    if (n[d] <= 0) n[d] = 132;
  }
  return n[d];
}

// Blocks of a grid-stride launch of `threads`-thread blocks over `work` items: one item per thread, at most 16 blocks
// for each of the H100's 132 SMs.
constexpr int64_t kGridStrideMaxBlocks = 132 * 16;
inline unsigned grid_stride_blocks(int64_t work, int threads = 256) {
  const int64_t g = (work + threads - 1) / threads;
  return static_cast<unsigned>(g < 1 ? 1 : (g > kGridStrideMaxBlocks ? kGridStrideMaxBlocks : g));
}

// Calls f(std::true_type{}) for dtype 1 (bf16) or f(std::false_type{}) for dtype 0 (fp16), so a launcher writes each
// launch once for both element types; any other code returns -3 without calling f.
template <typename F>
inline int dispatch_dtype(int dtype, F&& f) {
  if (dtype == 1) return f(std::true_type{});
  if (dtype == 0) return f(std::false_type{});
  return -3;
}

inline int pdl_enabled() {
  static const int v = [] { const char* e = getenv("IGGT_PDL"); return e ? atoi(e) : 1; }();
  return v;
}

// cluster_x > 1 launches thread-block clusters of that many CTAs along x (grid.x must be a multiple of it).
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl_cluster(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                                      int cluster_x, Args&&... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute at[2];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = pdl_enabled() ? 1 : 0;
  cfg.numAttrs = 1;
  if (cluster_x > 1) {
    at[1].id = cudaLaunchAttributeClusterDimension;
    at[1].val.clusterDim.x = cluster_x;
    at[1].val.clusterDim.y = 1;
    at[1].val.clusterDim.z = 1;
    cfg.numAttrs = 2;
  }
  cfg.attrs = at;
  return cudaLaunchKernelEx(&cfg, kern, std::forward<Args>(args)...);
}

template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                              Args&&... args) {
  return launch_pdl_cluster(kern, grid, block, smem, stream, 1, std::forward<Args>(args)...);
}

}  // namespace iggt
