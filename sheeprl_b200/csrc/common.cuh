// Shared helpers for the b200rl CUDA library (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#define B200RL_OK 0
#define B200RL_ERR_ARG 1
#define B200RL_ERR_CUDA 2

extern "C" void b200rl_set_error(const char* fmt, ...);

#define RL_CHECK_ARG(cond, msg)                                            \
  do {                                                                     \
    if (!(cond)) {                                                         \
      b200rl_set_error("%s:%d: bad argument: %s", __FILE__, __LINE__, msg); \
      return B200RL_ERR_ARG;                                               \
    }                                                                      \
  } while (0)

#define RL_CHECK_LAUNCH()                                                                   \
  do {                                                                                      \
    cudaError_t e__ = cudaGetLastError();                                                   \
    if (e__ != cudaSuccess) {                                                               \
      b200rl_set_error("%s:%d: CUDA launch failed: %s", __FILE__, __LINE__, cudaGetErrorString(e__)); \
      return B200RL_ERR_CUDA;                                                               \
    }                                                                                       \
  } while (0)

#define RL_CUDA(call)                                                                       \
  do {                                                                                      \
    cudaError_t e__ = (call);                                                               \
    if (e__ != cudaSuccess) {                                                               \
      b200rl_set_error("%s:%d: %s: %s", __FILE__, __LINE__, #call, cudaGetErrorString(e__)); \
      return B200RL_ERR_CUDA;                                                               \
    }                                                                                       \
  } while (0)

static constexpr float kFp32Eps = 1.1920928955078125e-07f;
static constexpr int kNumSMs = 132;   // H100 SXM

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Block-wide sum; every thread gets the result. `red` must hold >= 32 floats. blockDim.x multiple of 32.
__device__ __forceinline__ float block_sum(float v, float* red) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  v = warp_sum(v);
  __syncthreads();  // protect `red` from a previous use
  if (lane == 0) red[wid] = v;
  __syncthreads();
  const int nw = (blockDim.x + 31) >> 5;
  float r = (lane < nw) ? red[lane] : 0.f;
  r = warp_sum(r);
  return r;
}
__device__ __forceinline__ float block_max(float v, float* red) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  v = warp_max(v);
  __syncthreads();
  if (lane == 0) red[wid] = v;
  __syncthreads();
  const int nw = (blockDim.x + 31) >> 5;
  float r = (lane < nw) ? red[lane] : -INFINITY;
  r = warp_max(r);
  return r;
}

__device__ __forceinline__ float sigmoidf_(float x) { return 1.f / (1.f + expf(-x)); }
__device__ __forceinline__ float siluf_(float x) { return x / (1.f + expf(-x)); }
__device__ __forceinline__ float signf_(float x) { return (x > 0.f) ? 1.f : ((x < 0.f) ? -1.f : 0.f); }
__device__ __forceinline__ float symlogf_(float x) { return signf_(x) * logf(1.f + fabsf(x)); }
__device__ __forceinline__ float symexpf_(float x) { return signf_(x) * (expf(fabsf(x)) - 1.f); }

// one round of Philox4x32-10 (the noise fills key c = {index lo, index hi, stream id, device counter} by the seed)
__device__ __forceinline__ void philox_round(uint32_t (&c)[4], uint32_t k0, uint32_t k1) {
  const uint32_t hi0 = __umulhi(0xD2511F53u, c[0]), lo0 = 0xD2511F53u * c[0];
  const uint32_t hi1 = __umulhi(0xCD9E8D57u, c[2]), lo1 = 0xCD9E8D57u * c[2];
  const uint32_t n0 = hi1 ^ c[1] ^ k0, n1 = lo1, n2 = hi0 ^ c[3] ^ k1, n3 = lo0;
  c[0] = n0; c[1] = n1; c[2] = n2; c[3] = n3;
}

static inline int ceil_div(long long a, long long b) { return (int)((a + b - 1) / b); }

// Deterministic mode (det.cu): the launchers of the float-atomic reductions read det_mode() and, when it is set, write
// per-CTA partials to slots of det_workspace() that det_sum_slots adds in slot order (out += sum).
bool det_mode();
int det_workspace(size_t bytes, cudaStream_t st, void** ws);
int det_sum_slots(const float* part, int slots, long long n, float* out_a, long long na, float* out_b, cudaStream_t st);
int det_sum_slots_d(const double* part, int slots, double* out, cudaStream_t st);
