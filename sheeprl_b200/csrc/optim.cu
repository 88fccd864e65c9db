// Optimiser + small utility kernels on the flat parameter groups (pure HBM streaming).
//
// Replaces (reference): fabric.clip_gradients -> torch.nn.utils.clip_grad_norm_ and torch.optim.Adam.step
// (dreamer_v3.py:191-200, :298-304, :318-327; configs/optim/adam.yaml), torch.optim.Adam(weight_decay > 0).step
// (dreamer_v2.py:202-209, :333-337, :349-356; configs/algo/dreamer_v2.yaml), torch.optim.RMSprop.step (a2c/a2c.py:102-105;
// configs/optim/rmsprop.yaml), the per-parameter target-critic EMA
// loop (dreamer_v3.py:674-680), torch.multinomial's Exp(1) noise (Philox4x32-10 here).
// Clip + Adam are one pass: 4 reads + 3 writes of 4 B per parameter = 28 B/param (SURVEY.md §8d).
#include "common.cuh"

namespace {

// DET: the CTA's partial goes to slot blockIdx.x of `out` (det_sum_slots_d adds the slots in order) in place of a double
// atomic into out[0].
template <bool DET>
__global__ void __launch_bounds__(256)
sumsq_kernel(const float* __restrict__ x, long long n, double* __restrict__ out) {
  __shared__ double red[8];
  double s = 0.0;
  const long long stride = (long long)gridDim.x * blockDim.x;
  const long long n4 = n >> 2;
  const float4* x4 = reinterpret_cast<const float4*>(x);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
    const float4 v = x4[i];
    s += (double)v.x * v.x + (double)v.y * v.y + (double)v.z * v.z + (double)v.w * v.w;
  }
  for (long long i = (n4 << 2) + (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
    s += (double)x[i] * x[i];
  s = warp_sum_d(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x < 32) {
    double r = (threadIdx.x < 8) ? red[threadIdx.x] : 0.0;
    r = warp_sum_d(r);
    if (threadIdx.x == 0) {
      if constexpr (DET) out[blockIdx.x] = r;
      else atomicAdd(out, r);
    }
  }
}

// WD: torch's L2 weight decay (torch/optim/adam.py: grad = grad.add(param, alpha=weight_decay)), added to the already
// clipped gradient before the moments.  WD = false is the plain Adam kernel, so weight_decay = 0 stays bit-identical.
template <bool WD>
__global__ void __launch_bounds__(256)
adam_step_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
                 const double* __restrict__ normsq, const int* __restrict__ step_t, float* __restrict__ norm_out,
                 long long n, float max_norm, float lr, float b1, float b2, float eps, float weight_decay, int vec) {
  __shared__ float s_coef, s_step_size, s_bc2_sqrt;
  if (threadIdx.x == 0) {
    const float total = (float)sqrt(*normsq);
    float coef = 1.f;
    if (max_norm > 0.f) coef = fminf(max_norm / (total + 1e-6f), 1.f);
    const int t = *step_t;
    const double bc1 = 1.0 - pow((double)b1, (double)t);
    const double bc2 = 1.0 - pow((double)b2, (double)t);
    s_coef = coef;
    s_step_size = (float)((double)lr / bc1);
    s_bc2_sqrt = (float)sqrt(bc2);
    if (blockIdx.x == 0) norm_out[0] = total;
  }
  __syncthreads();
  const float coef = s_coef, step_size = s_step_size, bc2_sqrt = s_bc2_sqrt;
  const float omb1 = 1.f - b1, omb2 = 1.f - b2;
  const long long stride = (long long)gridDim.x * blockDim.x;
  const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  auto update = [&](float& pi, float gi, float& mi, float& vi) {
    gi *= coef;
    if (WD) gi = gi + weight_decay * pi;
    mi = mi + omb1 * (gi - mi);            // exp_avg.lerp_(grad, 1 - beta1)
    vi = vi * b2 + omb2 * gi * gi;         // exp_avg_sq.mul_(beta2).addcmul_(grad, grad, value=1 - beta2)
    const float denom = sqrtf(vi) / bc2_sqrt + eps;
    pi = pi - step_size * (mi / denom);
  };
  long long done = 0;
  if (vec) {   // 28 B / parameter of HBM traffic as 128-bit accesses (flat groups are 256-byte aligned)
    const long long n4 = n >> 2;
    float4* p4 = reinterpret_cast<float4*>(p);
    const float4* g4 = reinterpret_cast<const float4*>(g);
    float4* m4 = reinterpret_cast<float4*>(m);
    float4* v4 = reinterpret_cast<float4*>(v);
    for (long long i = tid; i < n4; i += stride) {
      float4 pp = p4[i], mm = m4[i], vv = v4[i];
      const float4 gg = g4[i];
      update(pp.x, gg.x, mm.x, vv.x);
      update(pp.y, gg.y, mm.y, vv.y);
      update(pp.z, gg.z, mm.z, vv.z);
      update(pp.w, gg.w, mm.w, vv.w);
      p4[i] = pp;
      m4[i] = mm;
      v4[i] = vv;
    }
    done = n4 << 2;
  }
  for (long long i = done + tid; i < n; i += stride) {
    float pi = p[i], mi = m[i], vi = v[i];
    update(pi, g[i], mi, vi);
    p[i] = pi;
    m[i] = mi;
    v[i] = vi;
  }
}

// One element of clip + torch.optim.RMSprop (single-tensor path, torch/optim/rmsprop.py).  Unlike Adam, eps is added
// AFTER the square root, and the step count does not enter the update.
template <bool CENTERED, bool MOMENTUM>
__device__ __forceinline__ void rmsprop_update(float& p, float g, float& sq, float& buf, float& gavg, float coef,
                                               float lr, float alpha, float eps, float weight_decay, float momentum) {
  g *= coef;
  if (weight_decay != 0.f) g = g + weight_decay * p;               // grad.add(param, alpha=weight_decay)
  sq = sq * alpha + (1.f - alpha) * g * g;                          // square_avg.mul_(alpha).addcmul_(grad, grad, 1-alpha)
  float avg;
  if (CENTERED) {
    gavg = gavg + (1.f - alpha) * (g - gavg);                       // grad_avg.lerp_(grad, 1 - alpha)
    avg = sqrtf(sq - gavg * gavg) + eps;
  } else {
    avg = sqrtf(sq) + eps;
  }
  if (MOMENTUM) {
    buf = buf * momentum + g / avg;                                 // buf.mul_(momentum).addcdiv_(grad, avg)
    p = p - lr * buf;
  } else {
    p = p - lr * (g / avg);
  }
}

// sq = square_avg; buf = momentum_buffer (touched only when MOMENTUM); gavg = grad_avg (only when CENTERED)
template <bool CENTERED, bool MOMENTUM>
__global__ void __launch_bounds__(256)
rmsprop_step_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ sq, float* __restrict__ buf,
                    float* __restrict__ gavg, const double* __restrict__ normsq, float* __restrict__ norm_out,
                    long long n, float max_norm, float lr, float alpha, float eps, float weight_decay, float momentum,
                    int vec) {
  __shared__ float s_coef;
  if (threadIdx.x == 0) {
    const float total = (float)sqrt(*normsq);
    float coef = 1.f;
    if (max_norm > 0.f) coef = fminf(max_norm / (total + 1e-6f), 1.f);
    s_coef = coef;
    if (blockIdx.x == 0) norm_out[0] = total;
  }
  __syncthreads();
  const float coef = s_coef;
  const long long stride = (long long)gridDim.x * blockDim.x;
  const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  long long done = 0;
  if (vec) {   // 128-bit accesses (flat groups are 256-byte aligned)
    const long long n4 = n >> 2;
    float4* p4 = reinterpret_cast<float4*>(p);
    const float4* g4 = reinterpret_cast<const float4*>(g);
    float4* s4 = reinterpret_cast<float4*>(sq);
    float4* b4 = reinterpret_cast<float4*>(buf);
    float4* a4 = reinterpret_cast<float4*>(gavg);
    for (long long i = tid; i < n4; i += stride) {
      float4 pp = p4[i], ss = s4[i];
      const float4 gg = g4[i];
      float4 bb = make_float4(0.f, 0.f, 0.f, 0.f), aa = bb;
      if (MOMENTUM) bb = b4[i];
      if (CENTERED) aa = a4[i];
      rmsprop_update<CENTERED, MOMENTUM>(pp.x, gg.x, ss.x, bb.x, aa.x, coef, lr, alpha, eps, weight_decay, momentum);
      rmsprop_update<CENTERED, MOMENTUM>(pp.y, gg.y, ss.y, bb.y, aa.y, coef, lr, alpha, eps, weight_decay, momentum);
      rmsprop_update<CENTERED, MOMENTUM>(pp.z, gg.z, ss.z, bb.z, aa.z, coef, lr, alpha, eps, weight_decay, momentum);
      rmsprop_update<CENTERED, MOMENTUM>(pp.w, gg.w, ss.w, bb.w, aa.w, coef, lr, alpha, eps, weight_decay, momentum);
      p4[i] = pp;
      s4[i] = ss;
      if (MOMENTUM) b4[i] = bb;
      if (CENTERED) a4[i] = aa;
    }
    done = n4 << 2;
  }
  for (long long i = done + tid; i < n; i += stride) {
    float pi = p[i], si = sq[i];
    float bi = MOMENTUM ? buf[i] : 0.f, ai = CENTERED ? gavg[i] : 0.f;
    rmsprop_update<CENTERED, MOMENTUM>(pi, g[i], si, bi, ai, coef, lr, alpha, eps, weight_decay, momentum);
    p[i] = pi;
    sq[i] = si;
    if (MOMENTUM) buf[i] = bi;
    if (CENTERED) gavg[i] = ai;
  }
}

__global__ void ema_kernel(float* __restrict__ tgt, const float* __restrict__ src, long long n, float tau, int vec) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  long long done = 0;
  if (vec) {
    const long long n4 = n >> 2;
    float4* t4 = reinterpret_cast<float4*>(tgt);
    const float4* s4 = reinterpret_cast<const float4*>(src);
    for (long long i = tid; i < n4; i += stride) {
      float4 t = t4[i];
      const float4 s = s4[i];
      t.x = t.x * (1.f - tau) + tau * s.x;
      t.y = t.y * (1.f - tau) + tau * s.y;
      t.z = t.z * (1.f - tau) + tau * s.z;
      t.w = t.w * (1.f - tau) + tau * s.w;
      t4[i] = t;
    }
    done = n4 << 2;
  }
  for (long long i = done + tid; i < n; i += stride) tgt[i] = tgt[i] * (1.f - tau) + tau * src[i];
}

__global__ void fill_exponential_kernel(float* __restrict__ out, long long n, uint32_t seed_lo, uint32_t seed_hi,
                                        uint32_t stream, const int* __restrict__ counter) {
  const uint32_t ctr = counter ? (uint32_t)(*counter) : 0u;  // device-side call counter (CUDA-graph safe)
  const long long stride = (long long)gridDim.x * blockDim.x;
  const long long n4 = (n + 3) >> 2;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
    uint32_t c[4] = {(uint32_t)i, (uint32_t)(i >> 32), stream, ctr};
    uint32_t k0 = seed_lo, k1 = seed_hi;
#pragma unroll
    for (int r = 0; r < 10; ++r) {
      philox_round(c, k0, k1);
      k0 += 0x9E3779B9u;
      k1 += 0xBB67AE85u;
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const long long idx = i * 4 + j;
      if (idx < n) {
        const float u = ((float)(c[j] >> 8) + 1.0f) * (1.0f / 16777216.0f);  // (0, 1]
        out[idx] = fmaxf(-logf(u), 1e-20f);                                   // Exp(1), strictly positive
      }
    }
  }
}

__global__ void fill_normal_kernel(float* __restrict__ out, long long n, uint32_t seed_lo, uint32_t seed_hi,
                                   uint32_t stream, const int* __restrict__ counter) {
  const uint32_t ctr = counter ? (uint32_t)(*counter) : 0u;
  const long long stride = (long long)gridDim.x * blockDim.x;
  const long long n4 = (n + 3) >> 2;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
    uint32_t c[4] = {(uint32_t)i, (uint32_t)(i >> 32), stream, ctr};
    uint32_t k0 = seed_lo, k1 = seed_hi;
#pragma unroll
    for (int r = 0; r < 10; ++r) {
      philox_round(c, k0, k1);
      k0 += 0x9E3779B9u;
      k1 += 0xBB67AE85u;
    }
#pragma unroll
    for (int j = 0; j < 4; j += 2) {                                         // Box-Muller on two uniforms
      const float u1 = ((float)(c[j] >> 8) + 1.0f) * (1.0f / 16777216.0f);   // (0, 1]
      const float u2 = (float)(c[j + 1] >> 8) * (1.0f / 16777216.0f);        // [0, 1)
      const float r = sqrtf(-2.f * logf(u1));
      float sn, cs;
      sincospif(2.f * u2, &sn, &cs);
      const long long idx = i * 4 + j;
      if (idx < n) out[idx] = r * cs;
      if (idx + 1 < n) out[idx + 1] = r * sn;
    }
  }
}

__global__ void copy2d_kernel(const float* __restrict__ src, float* __restrict__ dst, long long M, int C,
                              long long lds, long long ldd) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= M * C) return;
  const long long m = idx / C;
  const int c = (int)(idx - m * C);
  dst[m * ldd + c] = src[m * lds + c];
}

__global__ void axpy_kernel(const float* __restrict__ x, float* __restrict__ y, long long n, float alpha) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) y[i] = fmaf(alpha, x[i], y[i]);
}
__global__ void affine_kernel(const float* __restrict__ x, float* __restrict__ y, long long n, float alpha, float beta) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) y[i] = alpha * x[i] + beta;
}
// y[m, c] = symlog(x[m, c]) for a [M, C] block with row strides (vector observations squashed on the way into the
// MLP encoder, dreamer_v3/agent.py:150; the same tensor is the MLP decoder's regression target, distribution.py:180)
__global__ void symlog2d_kernel(const float* __restrict__ x, float* __restrict__ y, long long M, int C, long long ldx,
                                long long ldy) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M * C) return;
  const long long m = i / C;
  const int c = (int)(i - m * C);
  y[m * ldy + c] = symlogf_(x[m * ldx + c]);
}
__global__ void tanh_fwd_kernel(const float* __restrict__ x, float* __restrict__ y, long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) y[i] = tanhf(x[i]);
}
__global__ void tanh_bwd_kernel(const float* __restrict__ y, const float* __restrict__ dy, float* __restrict__ dx,
                                long long n, int accumulate) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    const float r = dy[i] * (1.f - y[i] * y[i]);
    dx[i] = accumulate ? dx[i] + r : r;
  }
}
__global__ void increment_kernel(int* p) { *p += 1; }

int stream_grid(long long n) {
  long long b = (n + 255) / 256;
  const long long cap = (long long)kNumSMs * 8;
  return (int)(b > cap ? cap : (b < 1 ? 1 : b));
}

}  // namespace

extern "C" int b200rl_sumsq(const float* x, long long n, double* out, cudaStream_t st) {
  RL_CHECK_ARG(x && out, "null pointer");
  RL_CHECK_ARG((reinterpret_cast<uintptr_t>(x) & 15) == 0, "x must be 16-byte aligned");
  RL_CUDA(cudaMemsetAsync(out, 0, sizeof(double), st));
  if (n <= 0) return B200RL_OK;
  const int grid = stream_grid(n / 4 + 1);
  if (det_mode()) {
    void* ws = nullptr;
    if (int rc = det_workspace(sizeof(double) * grid, st, &ws)) return rc;
    sumsq_kernel<true><<<grid, 256, 0, st>>>(x, n, static_cast<double*>(ws));
    RL_CHECK_LAUNCH();
    return det_sum_slots_d(static_cast<const double*>(ws), grid, out, st);
  }
  sumsq_kernel<false><<<grid, 256, 0, st>>>(x, n, out);
  RL_CHECK_LAUNCH();
  return B200RL_OK;
}

extern "C" int b200rl_adam_step_wd(float* p, const float* g, float* m, float* v, const double* normsq,
                                   const int* step_t, float* norm_out, long long n, float max_norm, float lr, float b1,
                                   float b2, float eps, float weight_decay, cudaStream_t st) {
  RL_CHECK_ARG(p && g && m && v && normsq && step_t && norm_out, "null pointer");
  RL_CHECK_ARG(weight_decay >= 0.f, "weight_decay must be >= 0");
  if (n <= 0) return B200RL_OK;
  const int vec = ((reinterpret_cast<uintptr_t>(p) | reinterpret_cast<uintptr_t>(g) | reinterpret_cast<uintptr_t>(m) |
                    reinterpret_cast<uintptr_t>(v)) & 15) == 0;
  auto k = weight_decay != 0.f ? adam_step_kernel<true> : adam_step_kernel<false>;
  k<<<stream_grid(vec ? (n + 3) / 4 : n), 256, 0, st>>>(p, g, m, v, normsq, step_t, norm_out, n, max_norm, lr, b1, b2, eps,
                                                        weight_decay, vec);
  RL_CHECK_LAUNCH();
  return B200RL_OK;
}

extern "C" int b200rl_adam_step(float* p, const float* g, float* m, float* v, const double* normsq, const int* step_t,
                                float* norm_out, long long n, float max_norm, float lr, float b1, float b2, float eps,
                                cudaStream_t st) {
  return b200rl_adam_step_wd(p, g, m, v, normsq, step_t, norm_out, n, max_norm, lr, b1, b2, eps, 0.f, st);
}

extern "C" int b200rl_rmsprop_step(float* p, const float* g, float* square_avg, float* momentum_buf, float* grad_avg,
                                   const double* normsq, float* norm_out, long long n, float max_norm, float lr,
                                   float alpha, float eps, float weight_decay, float momentum, cudaStream_t st) {
  RL_CHECK_ARG(p && g && square_avg && normsq && norm_out, "null pointer");
  RL_CHECK_ARG(momentum <= 0.f || momentum_buf, "momentum > 0 needs the momentum buffer");
  if (n <= 0) return B200RL_OK;
  const int vec = ((reinterpret_cast<uintptr_t>(p) | reinterpret_cast<uintptr_t>(g) |
                    reinterpret_cast<uintptr_t>(square_avg) |
                    reinterpret_cast<uintptr_t>(momentum > 0.f ? momentum_buf : nullptr) |
                    reinterpret_cast<uintptr_t>(grad_avg)) & 15) == 0;
  const int grid = stream_grid(vec ? (n + 3) / 4 : n);
  const bool centered = grad_avg != nullptr, mom = momentum > 0.f;
  auto k = centered ? (mom ? rmsprop_step_kernel<true, true> : rmsprop_step_kernel<true, false>)
                    : (mom ? rmsprop_step_kernel<false, true> : rmsprop_step_kernel<false, false>);
  k<<<grid, 256, 0, st>>>(p, g, square_avg, momentum_buf, grad_avg, normsq, norm_out, n, max_norm, lr, alpha, eps,
                          weight_decay, momentum, vec);
  RL_CHECK_LAUNCH();
  return B200RL_OK;
}

extern "C" int b200rl_ema(float* target, const float* src, long long n, float tau, cudaStream_t st) {
  RL_CHECK_ARG(target && src, "null pointer");
  if (n <= 0) return B200RL_OK;
  const int vec = ((reinterpret_cast<uintptr_t>(target) | reinterpret_cast<uintptr_t>(src)) & 15) == 0;
  ema_kernel<<<stream_grid(vec ? (n + 3) / 4 : n), 256, 0, st>>>(target, src, n, tau, vec);
  RL_CHECK_LAUNCH();
  return B200RL_OK;
}

extern "C" int b200rl_fill_exponential(float* out, long long n, unsigned long long seed, unsigned int stream_id,
                                       const int* counter_dev, cudaStream_t st) {
  RL_CHECK_ARG(out, "null pointer");
  if (n <= 0) return B200RL_OK;
  fill_exponential_kernel<<<stream_grid((n + 3) / 4), 256, 0, st>>>(out, n, (uint32_t)seed, (uint32_t)(seed >> 32),
                                                                   stream_id, counter_dev);
  RL_CHECK_LAUNCH();
  return B200RL_OK;
}

extern "C" int b200rl_fill_normal(float* out, long long n, unsigned long long seed, unsigned int stream_id,
                                  const int* counter_dev, cudaStream_t st) {
  RL_CHECK_ARG(out, "null pointer");
  if (n <= 0) return B200RL_OK;
  fill_normal_kernel<<<stream_grid((n + 3) / 4), 256, 0, st>>>(out, n, (uint32_t)seed, (uint32_t)(seed >> 32), stream_id,
                                                              counter_dev);
  RL_CHECK_LAUNCH();
  return B200RL_OK;
}

extern "C" int b200rl_zero(float* x, long long n, cudaStream_t st) {
  RL_CHECK_ARG(x, "null pointer");
  if (n > 0) RL_CUDA(cudaMemsetAsync(x, 0, sizeof(float) * (size_t)n, st));
  return B200RL_OK;
}

extern "C" int b200rl_copy2d(const float* src, float* dst, long long M, int C, long long lds, long long ldd,
                             cudaStream_t st) {
  RL_CHECK_ARG(src && dst, "null pointer");
  if (M * C <= 0) return B200RL_OK;
  if (lds == C && ldd == C) {
    RL_CUDA(cudaMemcpyAsync(dst, src, sizeof(float) * (size_t)(M * C), cudaMemcpyDeviceToDevice, st));
    return B200RL_OK;
  }
  copy2d_kernel<<<ceil_div(M * C, 256), 256, 0, st>>>(src, dst, M, C, lds, ldd);
  RL_CHECK_LAUNCH();
  return B200RL_OK;
}

extern "C" int b200rl_axpy(const float* x, float* y, long long n, float alpha, cudaStream_t st) {
  RL_CHECK_ARG(x && y, "null pointer");
  if (n <= 0) return B200RL_OK;
  axpy_kernel<<<ceil_div(n, 256), 256, 0, st>>>(x, y, n, alpha);
  RL_CHECK_LAUNCH();
  return B200RL_OK;
}

extern "C" int b200rl_affine(const float* x, float* y, long long n, float alpha, float beta, cudaStream_t st) {
  RL_CHECK_ARG(x && y, "null pointer");
  if (n <= 0) return B200RL_OK;
  affine_kernel<<<ceil_div(n, 256), 256, 0, st>>>(x, y, n, alpha, beta);
  RL_CHECK_LAUNCH();
  return B200RL_OK;
}

extern "C" int b200rl_symlog(const float* x, float* y, long long M, int C, long long ldx, long long ldy, cudaStream_t st) {
  RL_CHECK_ARG(x && y, "null pointer");
  RL_CHECK_ARG(C > 0 && ldx >= C && ldy >= C, "bad C / ld");
  if (M <= 0) return B200RL_OK;
  symlog2d_kernel<<<ceil_div(M * C, 256), 256, 0, st>>>(x, y, M, C, ldx, ldy);
  RL_CHECK_LAUNCH();
  return B200RL_OK;
}

extern "C" int b200rl_tanh_fwd(const float* x, float* y, long long n, cudaStream_t st) {
  RL_CHECK_ARG(x && y, "null pointer");
  if (n <= 0) return B200RL_OK;
  tanh_fwd_kernel<<<ceil_div(n, 256), 256, 0, st>>>(x, y, n);
  RL_CHECK_LAUNCH();
  return B200RL_OK;
}

extern "C" int b200rl_tanh_bwd(const float* y, const float* dy, float* dx, long long n, int accumulate,
                               cudaStream_t st) {
  RL_CHECK_ARG(y && dy && dx, "null pointer");
  if (n <= 0) return B200RL_OK;
  tanh_bwd_kernel<<<ceil_div(n, 256), 256, 0, st>>>(y, dy, dx, n, accumulate);
  RL_CHECK_LAUNCH();
  return B200RL_OK;
}

extern "C" int b200rl_increment(int* p, cudaStream_t st) {
  RL_CHECK_ARG(p, "null pointer");
  increment_kernel<<<1, 1, 0, st>>>(p);
  RL_CHECK_LAUNCH();
  return B200RL_OK;
}
