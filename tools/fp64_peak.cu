// Microbenchmark: FP64 pipe peaks on sm_90a (DFMA vs DMMA mma.sync f64 shapes).
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/fp64_peak tools/fp64_peak.cu
#include <cstdio>
#include <cuda_runtime.h>
#define CK(x) do{cudaError_t e=(x); if(e!=cudaSuccess){printf("CUDA %s @%d\n",cudaGetErrorString(e),__LINE__);return 1;}}while(0)

template<int ILP>
__global__ void k_dfma(double* out, int iters, double s) {
  double acc[ILP];
#pragma unroll
  for (int i=0;i<ILP;i++) acc[i]=threadIdx.x*1e-9+i;
  double a = s, b = 1.0 - s*1e-3;
  for (int it=0; it<iters; ++it) {
#pragma unroll
    for (int i=0;i<ILP;i++) acc[i] = fma(acc[i], b, a);
  }
  double r=0;
#pragma unroll
  for (int i=0;i<ILP;i++) r+=acc[i];
  out[blockIdx.x*blockDim.x+threadIdx.x]=r;
}

template<int ILP>
__global__ void k_dmma884(double* out, int iters, double s) {
  double c[ILP][2];
#pragma unroll
  for (int i=0;i<ILP;i++){c[i][0]=0;c[i][1]=0;}
  double a = s + threadIdx.x*1e-6, b = 1.0 - s*1e-3;
  for (int it=0; it<iters; ++it) {
#pragma unroll
    for (int i=0;i<ILP;i++)
      asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
        : "+d"(c[i][0]), "+d"(c[i][1]) : "d"(a), "d"(b));
  }
  double r=0;
#pragma unroll
  for (int i=0;i<ILP;i++) r+=c[i][0]+c[i][1];
  out[blockIdx.x*blockDim.x+threadIdx.x]=r;
}

template<int ILP>
__global__ void k_dmma1684(double* out, int iters, double s) {
  double c[ILP][4];
#pragma unroll
  for (int i=0;i<ILP;i++){c[i][0]=0;c[i][1]=0;c[i][2]=0;c[i][3]=0;}
  double a0 = s + threadIdx.x*1e-6, a1=a0*0.5, b = 1.0 - s*1e-3;
  for (int it=0; it<iters; ++it) {
#pragma unroll
    for (int i=0;i<ILP;i++)
      asm volatile("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};"
        : "+d"(c[i][0]), "+d"(c[i][1]), "+d"(c[i][2]), "+d"(c[i][3]) : "d"(a0),"d"(a1),"d"(b));
  }
  double r=0;
#pragma unroll
  for (int i=0;i<ILP;i++) r+=c[i][0]+c[i][1]+c[i][2]+c[i][3];
  out[blockIdx.x*blockDim.x+threadIdx.x]=r;
}

template<int ILP>
__global__ void k_dmma1688(double* out, int iters, double s) {
  double c[ILP][4];
#pragma unroll
  for (int i=0;i<ILP;i++){c[i][0]=0;c[i][1]=0;c[i][2]=0;c[i][3]=0;}
  double a0 = s + threadIdx.x*1e-6, a1=a0*0.5, a2=a0*0.25, a3=a0*0.125, b0 = 1.0 - s*1e-3, b1=b0*0.5;
  for (int it=0; it<iters; ++it) {
#pragma unroll
    for (int i=0;i<ILP;i++)
      asm volatile("mma.sync.aligned.m16n8k8.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+d"(c[i][0]), "+d"(c[i][1]), "+d"(c[i][2]), "+d"(c[i][3]) : "d"(a0),"d"(a1),"d"(a2),"d"(a3),"d"(b0),"d"(b1));
  }
  double r=0;
#pragma unroll
  for (int i=0;i<ILP;i++) r+=c[i][0]+c[i][1]+c[i][2]+c[i][3];
  out[blockIdx.x*blockDim.x+threadIdx.x]=r;
}

template<int ILP>
__global__ void k_dmma16816(double* out, int iters, double s) {
  double c[ILP][4];
#pragma unroll
  for (int i=0;i<ILP;i++){c[i][0]=0;c[i][1]=0;c[i][2]=0;c[i][3]=0;}
  double a[8], b[4];
#pragma unroll
  for (int j=0;j<8;j++) a[j]=s+threadIdx.x*1e-6*(j+1);
#pragma unroll
  for (int j=0;j<4;j++) b[j]=1.0-s*1e-3*(j+1);
  for (int it=0; it<iters; ++it) {
#pragma unroll
    for (int i=0;i<ILP;i++)
      asm volatile("mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, {%12,%13,%14,%15}, {%0,%1,%2,%3};"
        : "+d"(c[i][0]), "+d"(c[i][1]), "+d"(c[i][2]), "+d"(c[i][3])
        : "d"(a[0]),"d"(a[1]),"d"(a[2]),"d"(a[3]),"d"(a[4]),"d"(a[5]),"d"(a[6]),"d"(a[7]),"d"(b[0]),"d"(b[1]),"d"(b[2]),"d"(b[3]));
  }
  double r=0;
#pragma unroll
  for (int i=0;i<ILP;i++) r+=c[i][0]+c[i][1]+c[i][2]+c[i][3];
  out[blockIdx.x*blockDim.x+threadIdx.x]=r;
}

template<typename F>
int timeit(const char* name, F launch, double flop_per_launch) {
  cudaEvent_t e0,e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  launch(); launch(); CK(cudaDeviceSynchronize());
  if (cudaGetLastError() != cudaSuccess) { printf("%-28s launch failed (too many registers for this block size)\n", name); return 0; }
  float best=1e30f, tot=0;
  for (int r=0;r<5;r++){ cudaEventRecord(e0); launch(); cudaEventRecord(e1); CK(cudaEventSynchronize(e1)); float ms; cudaEventElapsedTime(&ms,e0,e1); if(ms<best)best=ms; tot+=ms; }
  printf("%-28s best %8.3f ms  %7.2f TFLOP/s   (mean %7.2f TFLOP/s)\n", name, best, flop_per_launch/best*1e-9, flop_per_launch/(tot/5)*1e-9);
  return 0;
}

int main(){
  int dev=0; cudaDeviceProp p; CK(cudaGetDeviceProperties(&p,dev));
  printf("GPU %s SMs %d clock %d kHz\n", p.name, p.multiProcessorCount, p.clockRate);
  int sms=p.multiProcessorCount;
  double* out; CK(cudaMalloc(&out, sizeof(double)*sms*8*1024));
  int iters=20000;
  for (int bps : {1,2,4}) for (int thr : {128,256,512}) {
    if (bps*thr>2048) continue;
    int grid=sms*bps; char nm[64];
    double thr_tot=(double)grid*thr;
    snprintf(nm,64,"dfma ilp8 b%d t%d",bps,thr);
    timeit(nm,[&]{k_dfma<8><<<grid,thr>>>(out,iters,0.5);}, thr_tot*iters*8*2.0);
    double warps=thr_tot/32;
    snprintf(nm,64,"dmma884 ilp8 b%d t%d",bps,thr);
    timeit(nm,[&]{k_dmma884<8><<<grid,thr>>>(out,iters,0.5);}, warps*iters*8*(8*8*4*2.0));
    snprintf(nm,64,"dmma1684 ilp4 b%d t%d",bps,thr);
    timeit(nm,[&]{k_dmma1684<4><<<grid,thr>>>(out,iters,0.5);}, warps*iters*4*(16*8*4*2.0));
    snprintf(nm,64,"dmma1688 ilp4 b%d t%d",bps,thr);
    timeit(nm,[&]{k_dmma1688<4><<<grid,thr>>>(out,iters,0.5);}, warps*iters*4*(16*8*8*2.0));
    snprintf(nm,64,"dmma16816 ilp4 b%d t%d",bps,thr);
    timeit(nm,[&]{k_dmma16816<4><<<grid,thr>>>(out,iters/2,0.5);}, warps*(iters/2)*4*(16*8*16*2.0));
  }
  // sustained: run dmma for ~3 s and report
  {
    int grid=sms*2, thr=256; double warps=(double)grid*thr/32;
    cudaEvent_t e0,e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    cudaEventRecord(e0); int n=0; 
    for (n=0;n<40;n++) k_dmma884<8><<<grid,thr>>>(out,iters*4,0.5);
    cudaEventRecord(e1); cudaEventSynchronize(e1); float ms; cudaEventElapsedTime(&ms,e0,e1);
    printf("sustained dmma884 %d launches %.1f ms  %.2f TFLOP/s\n", n, ms, warps*iters*4.0*8*512.0*n/ms*1e-9);
    cudaEventRecord(e0);
    for (n=0;n<40;n++) k_dfma<8><<<grid,thr>>>(out,iters*4,0.5);
    cudaEventRecord(e1); cudaEventSynchronize(e1); cudaEventElapsedTime(&ms,e0,e1);
    printf("sustained dfma    %d launches %.1f ms  %.2f TFLOP/s\n", n, ms, (double)grid*thr*iters*4.0*8*2.0*n/ms*1e-9);
  }
  return 0;
}
