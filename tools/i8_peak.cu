// int8 tensor-pipe peak of this GPU (wgmma.mma_async.m64n256k32.s32.s8.s8), measured the way tools/fp64_peak.cu
// measures the FP64 pipe: no memory traffic at all.  Every CTA keeps ONE operand stage in shared memory (content
// irrelevant) and two warpgroups issue back-to-back wgmmas into register accumulators; this is the denominator of the
// int8 roofline in bench.py.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -o tools/i8_peak tools/i8_peak.cu && tools/i8_peak
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cuda_runtime.h>
#include "../tnc_b200/csrc/sm90.h"

using namespace tncb;

__global__ void __launch_bounds__(256, 1) i8_peak_kernel(int iters, int* sink) {
  extern __shared__ __align__(1024) uint8_t raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(raw) + 1023) & ~(uintptr_t)1023);
  for (int i = threadIdx.x; i < 49152 / 4; i += blockDim.x) reinterpret_cast<uint32_t*>(smem)[i] = 0x01010101u * (uint32_t)(i & 3);
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy smem writes -> visible to the tensor core
  __syncthreads();
  const int wg = threadIdx.x >> 7;
  const uint64_t da = wg_desc<128>(smem + wg * 64 * 128), db = wg_desc<128>(smem + 16384);
  uint32_t acc[128];
#pragma unroll
  for (int i = 0; i < 128; i++) acc[i] = 0u;
  for (int it = 0; it < iters; it++) {
    wg_fence();
#pragma unroll
    for (int k = 0; k < 4; k++) wg_mma_s8_m64n256k32(acc, da + (uint64_t)(2 * k), db + (uint64_t)(2 * k), 1u);
    wg_commit();
    wg_wait<1>();
  }
  wg_wait<0>();
  int s = 0;
#pragma unroll
  for (int i = 0; i < 128; i++) s += (int)acc[i];
  if (s == 0x7fffffff) sink[threadIdx.x] = s;   // keeps the accumulators alive
}

int main() {
  cudaDeviceProp prop;
  cudaGetDeviceProperties(&prop, 0);
  const int sms = prop.multiProcessorCount;
  const int smem = 49152 + 1024;
  cudaFuncSetAttribute(i8_peak_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  int* sink = nullptr;
  cudaMalloc(&sink, 256 * sizeof(int));
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0); cudaEventCreate(&e1);
  printf("%s, %d SMs; wgmma m64n256k32 s8, two warpgroups per SM, operands resident in shared memory\n", prop.name, sms);
  for (int iters : {2000, 20000, 200000}) {
    i8_peak_kernel<<<sms, 256, smem>>>(100, sink);   // warm
    cudaDeviceSynchronize();
    cudaEventRecord(e0);
    i8_peak_kernel<<<sms, 256, smem>>>(iters, sink);
    cudaEventRecord(e1);
    cudaEventSynchronize(e1);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { printf("launch failed: %s\n", cudaGetErrorString(e)); return 1; }
    float ms = 0;
    cudaEventElapsedTime(&ms, e0, e1);
    const double ops = 2.0 * 64.0 * 256.0 * 32.0 * 4.0 * 2.0 * (double)iters * (double)sms;
    printf("iters %8d  %9.3f ms  %8.1f int8 TOP/s\n", iters, ms, ops / (ms * 1e-3) * 1e-12);
  }
  cudaFree(sink);
  return 0;
}
