// Library probe entry points.
#include <cuda_runtime.h>
#include "../../include/iggt_b200.h"

extern "C" const char* iggt_version(void) { return "iggt_b200 0.2 (sm_90a)"; }

extern "C" int iggt_device_info(int* sm, int* num_sms) {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return (int)e;
  cudaDeviceProp prop;
  e = cudaGetDeviceProperties(&prop, dev);
  if (e != cudaSuccess) return (int)e;
  if (sm) *sm = prop.major * 10 + prop.minor;
  if (num_sms) *num_sms = prop.multiProcessorCount;
  return 0;
}
