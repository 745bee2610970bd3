// Issue rates of MUFU.EX2 and F2FP.BF16 (pack) per SM sub-partition on sm_90a.
// nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 scripts/microbench/xu_rate.cu -o /tmp/xu_rate && /tmp/xu_rate
#include <cstdint>
#include <cstdio>
#include <cuda_bf16.h>
#include <cuda_runtime.h>

template <int MODE>  // 0: ex2 only, 1: cvt.rn.bf16x2 only, 2: ex2 + cvt (softmax-like: 2 ex2 per cvt), 3: ffma only
__global__ void __launch_bounds__(1024, 1) k(long long* out, float seed, int iters) {
  float a[8];
  uint32_t acc = 0;
#pragma unroll
  for (int i = 0; i < 8; ++i) a[i] = seed + i * 0.001f + threadIdx.x * 1e-6f;
  __syncthreads();
  const long long t0 = clock64();
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      if (MODE == 0 || MODE == 2) asm volatile("ex2.approx.ftz.f32 %0, %0;" : "+f"(a[i]));
      if (MODE == 3) asm volatile("fma.rn.f32 %0, %0, %0, %0;" : "+f"(a[i]));
    }
    if (MODE == 1 || MODE == 2) {
#pragma unroll
      for (int i = 0; i < 8; i += 2) {
        uint32_t p;
        asm volatile("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(p) : "f"(a[i]), "f"(a[i + 1]));
        acc ^= p;
      }
    }
  }
  const long long t1 = clock64();
  __syncthreads();
  if (threadIdx.x == 0) out[0] = t1 - t0;
  float s = 0;
  for (int i = 0; i < 8; ++i) s += a[i];
  if (s == 123.f || acc == 77) out[1] = 1;
}

int main() {
  long long* d;
  cudaMalloc(&d, 16);
  const int iters = 4000;
  const char* names[] = {"ex2 x8", "cvt.bf16x2 x4", "ex2 x8 + cvt x4", "ffma x8"};
  for (int threads : {128, 256, 512, 1024}) {
    for (int mode = 0; mode < 4; ++mode) {
      long long h = 0;
      if (mode == 0) k<0><<<1, threads>>>(d, 0.3f, iters);
      if (mode == 1) k<1><<<1, threads>>>(d, 0.3f, iters);
      if (mode == 2) k<2><<<1, threads>>>(d, 0.3f, iters);
      if (mode == 3) k<3><<<1, threads>>>(d, 0.3f, iters);
      cudaMemcpy(&h, d, 8, cudaMemcpyDeviceToHost);
      const double warps_per_smsp = threads / 32 / 4.0;
      printf("%-18s warps/SMSP=%.0f  clk per loop iteration per SMSP = %7.2f  (per warp-iteration %.2f)\n", names[mode], warps_per_smsp,
             double(h) / iters, double(h) / iters / warps_per_smsp);
    }
  }
  printf("status: %s\n", cudaGetErrorString(cudaDeviceSynchronize()));
  return 0;
}
