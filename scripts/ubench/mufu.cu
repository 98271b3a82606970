// Micro-benchmark: MUFU.EX2 and FMA-pipe exp2 throughput per SM on this GPU.
#include <cstdio>
#include <cuda_runtime.h>
__device__ __forceinline__ float ex2a(float x) { float y; asm volatile("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float ex2e(float x) {
  x = fmaxf(x, -125.0f);
  const float t = x + 12582912.0f;
  const float f = x - (t - 12582912.0f);
  float p = fmaf(0.05583828315138817f, f, 0.2426394820213318f);
  p = fmaf(p, f, 0.6931367516517639f);
  p = fmaf(p, f, 0.9999245405197144f);
  return __int_as_float(__float_as_int(p) + (__float_as_int(t) << 23));
}
template <int MODE>
__global__ void k(float* out, int iters, float c) {
  float a[16];
  for (int i = 0; i < 16; ++i) a[i] = -0.01f * (threadIdx.x + i);
  float acc = 0.f;
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      float x = fmaf(a[i], c, -0.5f);
      float e;
      if (MODE == 0) e = ex2a(x);
      else if (MODE == 1) e = ex2e(x);
      else e = (i % 4 == 0) ? ex2e(x) : ex2a(x);     // 25% emulated
      acc += e;
      a[i] = x * 0.999f;
    }
  }
  out[blockIdx.x * blockDim.x + threadIdx.x] = acc;
}
int main() {
  int sms; cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
  float* d; cudaMalloc(&d, sms * 1024 * 4);
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  int clk; cudaDeviceGetAttribute(&clk, cudaDevAttrClockRate, 0);
  for (int threads : {128, 256, 512, 1024}) for (int mode = 0; mode < 3; ++mode) {
    const int iters = 4096;
    auto launch = [&]() { if (mode == 0) k<0><<<sms, threads>>>(d, iters, 1.0001f); else if (mode == 1) k<1><<<sms, threads>>>(d, iters, 1.0001f); else k<2><<<sms, threads>>>(d, iters, 1.0001f); };
    launch(); cudaDeviceSynchronize();
    cudaEventRecord(e0); launch(); cudaEventRecord(e1); cudaEventSynchronize(e1);
    float ms; cudaEventElapsedTime(&ms, e0, e1);
    double exps = 1.0 * sms * threads * iters * 16;
    printf("threads %4d mode %d: %.3f ms  %.2f exp/ns/SM (at %.0f MHz nominal: %.2f exp/clk/SM)\n", threads, mode, ms, exps / (ms * 1e6) / sms, clk / 1e3, exps / (ms * 1e-3) / sms / (clk * 1e3));
  }
  return 0;
}
