// Microbenchmark: throughput / latency of the warp-level mma.sync.m16n8k8 TF32 (HMMA.1688.F32.TF32) on sm_90a,
// against packed fp32 FMAs, per SM sub-partition.   nvcc -gencode arch=compute_90a,code=sm_90a -O3 mma_rate.cu
#include <cstdio>
#include <cuda_runtime.h>
__device__ __forceinline__ void mma(float (&d)[4], unsigned a0, unsigned a1, unsigned a2, unsigned a3, unsigned b0, unsigned b1) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]) : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}
template <int CHAINS>
__global__ void k_mma(float* out, long long* cyc, int iters) {
  float d[CHAINS][4];
  for (int c = 0; c < CHAINS; ++c) for (int i = 0; i < 4; ++i) d[c][i] = 0.f;
  unsigned a = threadIdx.x * 0x01010101u + 0x3f800000u, b = a ^ 0x00012300u;
  __syncthreads();
  long long t0 = clock64();
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int c = 0; c < CHAINS; ++c) mma(d[c], a, b, a + c, b + c, a, b);
  }
  long long t1 = clock64();
  float s = 0.f;
  for (int c = 0; c < CHAINS; ++c) for (int i = 0; i < 4; ++i) s += d[c][i];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
  if (threadIdx.x == 0 && blockIdx.x == 0) *cyc = t1 - t0;
}
int main() {
  float* out; long long* cyc; cudaMalloc(&out, 1 << 20); cudaMalloc(&cyc, 8);
  const int iters = 2000;
  for (int warps : {4, 8, 16}) {
    long long h;
#define RUN(C) k_mma<C><<<148, warps * 32>>>(out, cyc, iters); cudaMemcpy(&h, cyc, 8, cudaMemcpyDeviceToHost); \
    printf("warps/SM %2d chains %d: %.1f cycles per MMA per warp, %.1f cycles per MMA per SM sub-partition\n", warps, C, \
           (double)h / iters / C, (double)h / iters / C / (warps / 4.0));
    RUN(1) RUN(2) RUN(4) RUN(8)
  }
  printf("%s\n", cudaGetErrorString(cudaDeviceSynchronize()));
  return 0;
}
