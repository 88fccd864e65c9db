// Deterministic mode (include/b200rl.h: b200rl_set_deterministic): the process-wide switch, the partials pool and the
// fixed-order reductions shared by the deterministic forms of the kernels that otherwise reduce with float atomics.
//
// Each such kernel, under deterministic mode, writes one partial per CTA (or warp) to a slot chosen by its index, and
// det_sum_slots adds the slots to the output in slot order.  The grid, and so the slot count, depends on the shape
// only, so the sum is bit-reproducible run to run on the same GPU type.
#include <mutex>
#include <vector>

#include "common.cuh"

namespace {

int g_det = 0;

// Partials pool, one per device, grown on demand OUTSIDE stream capture (launches on one stream serialise, so
// consecutive deterministic reductions share it).  A grown pool keeps its older buffers alive: a CUDA graph captured
// before the growth still points at them.
struct DetWs {
  void* buf = nullptr;
  size_t bytes = 0;
  std::vector<void*> retired;
};
DetWs g_ws[16];
std::mutex g_ws_mu;

// out_a[c] (c < na) or out_b[c - na] (c >= na) += sum_z part[z * n + c], z ascending in 32 interleaved chains that are
// then added in chain order.  blockDim = (32, 32): threadIdx.x the column, threadIdx.y the chain.
__global__ void __launch_bounds__(1024)
det_sum_slots_kernel(const float* __restrict__ part, int slots, long long n, float* out_a, long long na, float* out_b) {
  __shared__ float red[32][33];
  const long long c = (long long)blockIdx.x * 32 + threadIdx.x;
  float s = 0.f;
  if (c < n)
    for (int z = threadIdx.y; z < slots; z += 32) s += __ldcg(part + (size_t)z * n + c);
  red[threadIdx.y][threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.y == 0 && c < n) {
    float t = 0.f;
#pragma unroll
    for (int i = 0; i < 32; ++i) t += red[i][threadIdx.x];
    float* o = c < na ? out_a + c : out_b + (c - na);
    *o += t;
  }
}

// *out = sum_z part[z]: one CTA, the same fixed tree for a given slot count
__global__ void __launch_bounds__(256) det_sum_slots_d_kernel(const double* __restrict__ part, int slots, double* out) {
  __shared__ double red[8];
  double s = 0.0;
  for (int z = threadIdx.x; z < slots; z += blockDim.x) s += __ldcg(part + z);
  s = warp_sum_d(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    double r = 0.0;
    for (int i = 0; i < 8; ++i) r += red[i];
    *out = r;
  }
}

}  // namespace

bool det_mode() { return g_det != 0; }

int det_workspace(size_t bytes, cudaStream_t st, void** ws) {
  int dev = 0;
  RL_CUDA(cudaGetDevice(&dev));
  RL_CHECK_ARG(dev < 16, "deterministic workspace: device index out of range");
  std::lock_guard<std::mutex> lk(g_ws_mu);
  DetWs& w = g_ws[dev];
  if (bytes > w.bytes) {
    cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
    RL_CUDA(cudaStreamIsCapturing(st, &cs));
    if (cs != cudaStreamCaptureStatusNone) {
      b200rl_set_error("deterministic workspace must grow outside stream capture: run the step once eagerly first");
      return B200RL_ERR_CUDA;
    }
    const size_t n = bytes + bytes / 2 > ((size_t)16 << 20) ? bytes + bytes / 2 : ((size_t)16 << 20);
    void* p = nullptr;
    RL_CUDA(cudaMalloc(&p, n));
    if (w.buf) w.retired.push_back(w.buf);
    w.buf = p;
    w.bytes = n;
  }
  *ws = w.buf;
  return B200RL_OK;
}

int det_sum_slots(const float* part, int slots, long long n, float* out_a, long long na, float* out_b, cudaStream_t st) {
  if (n <= 0) return B200RL_OK;
  det_sum_slots_kernel<<<(unsigned)((n + 31) / 32), dim3(32, 32), 0, st>>>(part, slots, n, out_a, na, out_b);
  RL_CHECK_LAUNCH();
  return B200RL_OK;
}

int det_sum_slots_d(const double* part, int slots, double* out, cudaStream_t st) {
  det_sum_slots_d_kernel<<<1, 256, 0, st>>>(part, slots, out);
  RL_CHECK_LAUNCH();
  return B200RL_OK;
}

extern "C" int b200rl_set_deterministic(int on) {
  RL_CHECK_ARG(on == 0 || on == 1, "deterministic must be 0 or 1");
  g_det = on;
  return B200RL_OK;
}
extern "C" int b200rl_get_deterministic(void) { return g_det; }

extern "C" int b200rl_deterministic_pool_fill(int byte, cudaStream_t st) {
  RL_CHECK_ARG(byte >= 0 && byte <= 255, "byte must be 0..255");
  int dev = 0;
  RL_CUDA(cudaGetDevice(&dev));
  RL_CHECK_ARG(dev < 16, "deterministic workspace: device index out of range");
  std::lock_guard<std::mutex> lk(g_ws_mu);
  if (g_ws[dev].buf) RL_CUDA(cudaMemsetAsync(g_ws[dev].buf, byte, g_ws[dev].bytes, st));
  return B200RL_OK;
}
