// Programmatic dependent launch (PDL) helpers.  Every hot kernel does its global-memory-free prologue (mbarrier
// init, tensor-map prefetch), then `griddep_wait()` before it touches global memory, and lets the
// next kernel in the stream begin ITS prologue early with `griddep_launch()`.  With ~730 back-to-back launches per
// forward (each short once the views are sharded over several GPUs) the launch latency and prologues are
// otherwise exposed.  IGGT_PDL=0 falls back to plain stream-ordered launches.
#pragma once
#include <cuda_runtime.h>
#include <stdlib.h>
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
// `static DeviceOnce once; if (once.first()) { ...configure the kernel on the current device... }`
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
