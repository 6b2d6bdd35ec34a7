// Microbenchmark: issue-bound FP64 throughput of DMMA.8x8x4 (mma.sync.m8n8k4.f64) vs plain DFMA on this GPU.
// nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o fp64_peak tools/fp64_peak.cu
#include <cstdio>
#include <cuda_runtime.h>
__global__ void dmma_loop(double *out, int iters) {
  double c[16][2];
  for (int i = 0; i < 16; i++) { c[i][0] = 0.0; c[i][1] = 0.0; }
  double a = threadIdx.x * 1e-3, b = blockIdx.x * 1e-4 + 1.0;
  for (int it = 0; it < iters; it++) {
#pragma unroll
    for (int i = 0; i < 16; i++)
      asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n" : "+d"(c[i][0]), "+d"(c[i][1]) : "d"(a), "d"(b));
  }
  double s = 0.0;
  for (int i = 0; i < 16; i++) s += c[i][0] + c[i][1];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}
__global__ void dfma_loop(double *out, int iters) {
  double c[32];
  for (int i = 0; i < 32; i++) c[i] = i;
  double a = 1.0 + threadIdx.x * 1e-9, b = blockIdx.x * 1e-9;
  for (int it = 0; it < iters; it++) {
#pragma unroll
    for (int i = 0; i < 32; i++) c[i] = fma(c[i], a, b);
  }
  double s = 0.0;
  for (int i = 0; i < 32; i++) s += c[i];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}
int main() {
  cudaDeviceProp p; cudaGetDeviceProperties(&p, 0);
  const int sms = p.multiProcessorCount;
  double *out; cudaMalloc(&out, sizeof(double) * sms * 8 * 1024);
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  for (int warps = 4; warps <= 32; warps *= 2) {
    const int iters = 20000, blocks = sms * 2, threads = warps * 32 / 2;
    for (int which = 0; which < 2; which++) {
      float best = 1e30f;
      for (int rep = 0; rep < 3; rep++) {
        cudaEventRecord(e0);
        if (which == 0) dmma_loop<<<blocks, threads>>>(out, iters); else dfma_loop<<<blocks, threads>>>(out, iters);
        cudaEventRecord(e1); cudaEventSynchronize(e1);
        float ms; cudaEventElapsedTime(&ms, e0, e1); if (ms < best) best = ms;
      }
      const double flops = which == 0 ? (double)blocks * (threads / 32) * iters * 16 * 512.0 : (double)blocks * threads * iters * 32 * 2.0;
      printf("%s warps/SM=%d  %.2f TF/s\n", which == 0 ? "DMMA.8x8x4" : "DFMA      ", warps, flops / (best * 1e-3) / 1e12);
    }
  }
  return 0;
}
