// Loss kernels: forward value + seed gradient fused (HBM-bound, one pass over the logits).
//
// Replaces (reference): MSEDistribution.log_prob (sheeprl/utils/distribution.py:212-221),
// TwoHotEncodingDistribution.log_prob/.mean (distribution.py:224-276) with symlog/symexp
// (utils/utils.py:148-153), Bernoulli(logits).log_prob (continue head, dreamer_v3.py:167, loss.py:77),
// compute_lambda_values + discount cumprod (dreamer_v3/utils.py:66-77, dreamer_v3.py:244-260),
// Moments (dreamer_v3/utils.py:40-63, torch.quantile 'linear'), the discrete policy loss
// (dreamer_v3.py:272-297) -- and the autograd backward of each.
#include "common.cuh"

namespace {

// torch.linspace(low, high, nb)[i] in fp32 (symmetric fill, as ATen's CPU/CUDA kernels do)
__device__ __forceinline__ float bin_value(int i, int nb, float low, float high) {
  const float step = (high - low) / (float)(nb - 1);
  return (i < nb / 2) ? (low + step * (float)i) : (high - step * (float)(nb - 1 - i));
}

__global__ void __launch_bounds__(256)
mse_loss_grad_kernel(const float* pred, const float* __restrict__ target, float* __restrict__ loss_row, float* grad,
                     int P, float scale) {
  __shared__ float red[32];
  const long long m = blockIdx.x;
  const float* p = pred + m * P;
  const float* t = target + m * P;
  float* g = grad + m * P;
  float s = 0.f;
  for (int i = threadIdx.x; i < P; i += blockDim.x) {
    const float d = p[i] - t[i];
    s = fmaf(d, d, s);
    g[i] = 2.f * scale * d;  // grad may alias pred: element i is read before it is written by the same thread
  }
  s = block_sum(s, red);
  if (threadIdx.x == 0) loss_row[m] = s;
}

// One warp per row.
__global__ void __launch_bounds__(256)
twohot_loss_grad_kernel(const float* __restrict__ logits, const float* __restrict__ x, const float* __restrict__ weight,
                        float* __restrict__ loss_row, float* __restrict__ dlogits, long long M, int nb, long long ldl,
                        long long ldd, float low, float high, float scale, int accumulate) {
  const int lane = threadIdx.x & 31;
  const long long m = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (m >= M) return;
  const float* l = logits + m * ldl;
  const float xs = symlogf_(x[m]);
  int cnt = 0;
  float mx = -INFINITY;
  for (int c = lane; c < nb; c += 32) {
    cnt += (bin_value(c, nb, low, high) <= xs) ? 1 : 0;
    mx = fmaxf(mx, l[c]);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
  mx = warp_max(mx);
  float se = 0.f;
  for (int c = lane; c < nb; c += 32) se += expf(l[c] - mx);
  const float lse = mx + logf(warp_sum(se));
  int below = cnt - 1, above = below + 1;
  above = min(above, nb - 1);
  below = max(below, 0);
  float w_lo, w_hi;
  if (below == above) { w_lo = 0.5f; w_hi = 0.5f; }   // dist 1 / (1+1) each, both scattered onto the same bin
  else {
    const float d_lo = fabsf(bin_value(below, nb, low, high) - xs);
    const float d_hi = fabsf(bin_value(above, nb, low, high) - xs);
    const float tot = d_lo + d_hi;
    w_lo = d_hi / tot;
    w_hi = d_lo / tot;
  }
  const float wr = scale * (weight ? weight[m] : 1.f);
  float* d = dlogits + m * ldd;
  for (int c = lane; c < nb; c += 32) {
    float tgt = 0.f;
    if (c == below) tgt += w_lo;
    if (c == above) tgt += w_hi;
    const float g = (expf(l[c] - lse) - tgt) * wr;
    d[c] = accumulate ? d[c] + g : g;
  }
  if (lane == 0) {
    const float lr = -(w_lo * (l[below] - lse) + w_hi * (l[above] - lse));
    loss_row[m] = accumulate ? loss_row[m] + lr : lr;
  }
}

__global__ void bce_loss_grad_kernel(const float* __restrict__ logit, const float* __restrict__ target,
                                     float* __restrict__ loss_row, float* __restrict__ dlogit, long long M,
                                     float loss_scale, float scale) {
  const long long m = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= M) return;
  const float l = logit[m], y = target[m];
  // binary_cross_entropy_with_logits: (1-y)*l + log1p(exp(-|l|)) + max(-l, 0)
  const float v = (1.f - y) * l + fmaxf(-l, 0.f) + log1pf(expf(-fabsf(l)));
  loss_row[m] = loss_scale * v;
  dlogit[m] = loss_scale * scale * (sigmoidf_(l) - y);
}

__global__ void __launch_bounds__(256)
twohot_mean_kernel(const float* __restrict__ logits, float* __restrict__ out, long long M, int nb, long long ldl,
                   float low, float high) {
  const int lane = threadIdx.x & 31;
  const long long m = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (m >= M) return;
  const float* l = logits + m * ldl;
  float mx = -INFINITY;
  for (int c = lane; c < nb; c += 32) mx = fmaxf(mx, l[c]);
  mx = warp_max(mx);
  float se = 0.f, sb = 0.f;
  for (int c = lane; c < nb; c += 32) se += expf(l[c] - mx);
  se = warp_sum(se);
  for (int c = lane; c < nb; c += 32) sb = fmaf(expf(l[c] - mx) / se, bin_value(c, nb, low, high), sb);
  sb = warp_sum(sb);
  if (lane == 0) out[m] = symexpf_(sb);
}

// thread per column n: reverse scan over H (lambda returns) + forward cumprod (discount)
__global__ void lambda_returns_kernel(const float* __restrict__ rew, const float* __restrict__ val,
                                      const float* __restrict__ cont_logit, const float* __restrict__ true_cont,
                                      float* __restrict__ lam, float* __restrict__ discount, int H, int N, float gamma,
                                      float lmbda) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  float nxt = val[(long long)H * N + n];
  for (int t = H - 1; t >= 0; --t) {
    const long long i = (long long)(t + 1) * N + n;
    const float c = ((sigmoidf_(cont_logit[i]) > 0.5f) ? 1.f : 0.f) * gamma;
    const float interm = rew[i] + c * val[i] * (1.f - lmbda);
    nxt = interm + c * lmbda * nxt;
    lam[(long long)t * N + n] = nxt;
  }
  float prod = 1.f;
  for (int t = 0; t <= H; ++t) {
    const long long i = (long long)t * N + n;
    const float c = (t == 0) ? true_cont[n] : ((sigmoidf_(cont_logit[i]) > 0.5f) ? 1.f : 0.f);
    prod *= c * gamma;
    discount[i] = prod / gamma;
  }
}

__device__ __forceinline__ unsigned int float_key(float f) {
  const unsigned int u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);  // monotone: larger float -> larger key
}
__device__ __forceinline__ float key_float(unsigned int k) {
  const unsigned int u = (k & 0x80000000u) ? (k & 0x7fffffffu) : ~k;
  return __uint_as_float(u);
}

// exact k-th smallest (0-based) of x[0..n) by MSB radix select; single block; hist: 256 ints of smem
__device__ float select_kth(const float* __restrict__ x, long long n, long long k, unsigned int* hist,
                            unsigned int* bcast) {
  unsigned int prefix = 0, mask = 0;
  for (int shift = 24; shift >= 0; shift -= 8) {
    for (int i = threadIdx.x; i < 256; i += blockDim.x) hist[i] = 0;
    __syncthreads();
    for (long long i = threadIdx.x; i < n; i += blockDim.x) {
      const unsigned int key = float_key(x[i]);
      if ((key & mask) == prefix) atomicAdd(&hist[(key >> shift) & 0xffu], 1u);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      long long kk = k;
      unsigned int b = 0;
      for (; b < 256; ++b) {
        if (kk < (long long)hist[b]) break;
        kk -= hist[b];
      }
      bcast[0] = b;
      bcast[1] = (unsigned int)kk;
    }
    __syncthreads();
    prefix |= bcast[0] << shift;
    mask |= 0xffu << shift;
    k = bcast[1];
    __syncthreads();
  }
  return key_float(prefix);
}

// torch.quantile 'linear' of NaN-free x: the fp32 rank q (n - 1), the order statistics at its floor and ceil, ATen's
// lerp.  At an integral rank both are the same element, so the result is that element (an infinite one gives NaN, as
// ATen's lerp(a, a, 0) does) and never a zero weight times the next order statistic.
__device__ float quantile_linear(const float* x, long long n, float q, unsigned int* hist, unsigned int* bcast) {
  const float rank = q * (float)(n - 1);
  const float lo = floorf(rank);
  const long long ilo = (long long)lo;
  const long long ihi = (long long)ceilf(rank);
  const float w = rank - lo;
  const float a = select_kth(x, n, ilo, hist, bcast);
  const float b = (ihi == ilo) ? a : select_kth(x, n, ihi, hist, bcast);
  return (w < 0.5f) ? (a + w * (b - a)) : (b - (b - a) * (1.f - w));  // ATen lerp
}

__global__ void __launch_bounds__(1024)
moments_update_kernel(const float* __restrict__ x, long long n, float* __restrict__ state, float* __restrict__ out,
                      float decay, float one_minus_decay, float inv_max, float p_low, float p_high) {
  __shared__ unsigned int hist[256];
  __shared__ unsigned int bcast[2];
  int nan_seen = 0;
  for (long long i = threadIdx.x; i < n; i += blockDim.x) nan_seen |= isnan(x[i]) ? 1 : 0;
  // torch.quantile returns NaN for both quantiles when x holds a NaN
  const bool any_nan = __syncthreads_or(nan_seen) != 0;
  const float lo = any_nan ? NAN : quantile_linear(x, n, p_low, hist, bcast);
  const float hi = any_nan ? NAN : quantile_linear(x, n, p_high, hist, bcast);
  if (threadIdx.x == 0) {
    const float l = decay * state[0] + one_minus_decay * lo;
    const float h = decay * state[1] + one_minus_decay * hi;
    state[0] = l;
    state[1] = h;
    out[0] = l;
    const float d = h - l;
    out[1] = isnan(d) ? d : fmaxf(inv_max, d);  // torch.max propagates NaN; fmaxf would drop it
  }
}

constexpr int MAX_HEADS = 16;
struct HeadDims { int n; int dim[MAX_HEADS]; };

// One warp per row; loops over the action heads.
__global__ void __launch_bounds__(256)
actor_loss_grad_kernel(const float* __restrict__ raw, const float* __restrict__ actions, const float* __restrict__ lam,
                       const float* __restrict__ val, const float* __restrict__ discount,
                       const float* __restrict__ moments, float* __restrict__ rows, float* __restrict__ draw,
                       long long M, int A, HeadDims heads, float unimix, float ent_coef, float scale) {
  const int lane = threadIdx.x & 31;
  const long long m = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (m >= M) return;
  const float off = moments[0], inv = moments[1];
  const float adv = (lam[m] - off) / inv - (val[m] - off) / inv;
  const float disc = discount[m];
  float obj = 0.f, ent_tot = 0.f;
  int o = 0;
  for (int hd = 0; hd < heads.n; ++hd) {
    const int K = heads.dim[hd];
    const float* x = raw + m * A + o;
    const float* av = actions + m * A + o;
    float* dr = draw + m * A + o;
    const float invK = 1.f / (float)K;
    float mx = -INFINITY, amax = -INFINITY;
    int aidx = 0x7fffffff;
    for (int c = lane; c < K; c += 32) {
      mx = fmaxf(mx, x[c]);
      if (av[c] > amax) { amax = av[c]; aidx = c; }
    }
    mx = warp_max(mx);
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) {
      const float ob = __shfl_xor_sync(0xffffffffu, amax, s);
      const int oi = __shfl_xor_sync(0xffffffffu, aidx, s);
      if (ob > amax || (ob == amax && oi < aidx)) { amax = ob; aidx = oi; }
    }
    float se = 0.f;
    for (int c = lane; c < K; c += 32) se += expf(x[c] - mx);
    se = warp_sum(se);
    // unimix log-probs and their logsumexp
    float lmx = -INFINITY;
    for (int c = lane; c < K; c += 32) {
      float l = x[c];
      if (unimix > 0.f) { const float pm = (1.f - unimix) * (expf(x[c] - mx) / se) + unimix * invK;
                          l = logf(fminf(fmaxf(pm, kFp32Eps), 1.f - kFp32Eps)); }
      lmx = fmaxf(lmx, l);
    }
    lmx = warp_max(lmx);
    float ls = 0.f;
    for (int c = lane; c < K; c += 32) {
      float l = x[c];
      if (unimix > 0.f) { const float pm = (1.f - unimix) * (expf(x[c] - mx) / se) + unimix * invK;
                          l = logf(fminf(fmaxf(pm, kFp32Eps), 1.f - kFp32Eps)); }
      ls += expf(l - lmx);
    }
    const float lse = lmx + logf(warp_sum(ls));
    float ent = 0.f, logp = 0.f;
    for (int c = lane; c < K; c += 32) {
      float l = x[c];
      if (unimix > 0.f) { const float pm = (1.f - unimix) * (expf(x[c] - mx) / se) + unimix * invK;
                          l = logf(fminf(fmaxf(pm, kFp32Eps), 1.f - kFp32Eps)); }
      const float lg = l - lse;
      ent = fmaf(-expf(lg), lg, ent);
      if (c == aidx) logp = lg;
    }
    ent = warp_sum(ent);
    logp = warp_sum(logp);
    obj = fmaf(logp, adv, obj);
    ent_tot += ent;
    // gradient wrt the unimix log-probs, then through unimix + softmax to the raw logits
    const float gs = -scale * disc;
    float sds = 0.f;
    for (int c = lane; c < K; c += 32) {
      const float s = expf(x[c] - mx) / se;
      float pm = 0.f, l = x[c];
      if (unimix > 0.f) { pm = (1.f - unimix) * s + unimix * invK; l = logf(fminf(fmaxf(pm, kFp32Eps), 1.f - kFp32Eps)); }
      const float lg = l - lse, p = expf(lg);
      const float gg = gs * (adv * (((c == aidx) ? 1.f : 0.f) - p) + ent_coef * (-p * (lg + ent)));
      if (unimix > 0.f) {
        const bool inside = pm >= kFp32Eps && pm <= 1.f - kFp32Eps;
        sds = fmaf(s, inside ? gg * (1.f - unimix) / pm : 0.f, sds);
      }
    }
    sds = warp_sum(sds);
    for (int c = lane; c < K; c += 32) {
      const float s = expf(x[c] - mx) / se;
      float pm = 0.f, l = x[c];
      if (unimix > 0.f) { pm = (1.f - unimix) * s + unimix * invK; l = logf(fminf(fmaxf(pm, kFp32Eps), 1.f - kFp32Eps)); }
      const float lg = l - lse, p = expf(lg);
      float gg = gs * (adv * (((c == aidx) ? 1.f : 0.f) - p) + ent_coef * (-p * (lg + ent)));
      if (unimix > 0.f) {
        const bool inside = pm >= kFp32Eps && pm <= 1.f - kFp32Eps;
        gg = s * ((inside ? gg * (1.f - unimix) / pm : 0.f) - sds);
      }
      dr[c] = gg;
    }
    o += K;
  }
  if (lane == 0) rows[m] = disc * (obj + ent_coef * ent_tot);
}

// out[c] = scale * sum_m X[m*ld + c]; one block per column (deterministic)
__global__ void __launch_bounds__(1024)
sum_rows_kernel(const float* __restrict__ X, float* __restrict__ out, long long M, long long ldx, float scale) {
  __shared__ float red[32];
  const int c = blockIdx.x;
  float s = 0.f;
  for (long long m = threadIdx.x; m < M; m += blockDim.x) s += X[m * ldx + c];
  s = block_sum(s, red);
  if (threadIdx.x == 0) out[c] = scale * s;
}

__global__ void __launch_bounds__(1024)
weighted_mean_kernel(const float* __restrict__ x, const float* __restrict__ w, float* __restrict__ out, long long n,
                     float scale) {
  __shared__ float red[32];
  float s = 0.f;
  for (long long i = threadIdx.x; i < n; i += blockDim.x) s = fmaf(x[i], w[i], s);
  s = block_sum(s, red);
  if (threadIdx.x == 0) out[0] = scale * s;
}

}  // namespace

extern "C" int b200rl_mse_loss_grad(const float* pred, const float* target, float* loss_row, float* grad, long long M,
                                    int P, float scale, cudaStream_t st) {
  RL_CHECK_ARG(pred && target && loss_row && grad, "null pointer");
  if (M <= 0) return B200RL_OK;
  mse_loss_grad_kernel<<<(unsigned)M, 256, 0, st>>>(pred, target, loss_row, grad, P, scale);
  RL_CHECK_LAUNCH();
  return B200RL_OK;
}

extern "C" int b200rl_twohot_loss_grad(const float* logits, const float* x, const float* weight, float* loss_row,
                                       float* dlogits, long long M, int nb, long long ldl, long long ldd, float low,
                                       float high, float scale, int accumulate, cudaStream_t st) {
  RL_CHECK_ARG(logits && x && loss_row && dlogits, "null pointer");
  RL_CHECK_ARG(nb >= 2, "need at least two bins");
  if (M <= 0) return B200RL_OK;
  twohot_loss_grad_kernel<<<ceil_div(M, 8), 256, 0, st>>>(logits, x, weight, loss_row, dlogits, M, nb, ldl, ldd, low,
                                                          high, scale, accumulate);
  RL_CHECK_LAUNCH();
  return B200RL_OK;
}

extern "C" int b200rl_bce_loss_grad(const float* logit, const float* target, float* loss_row, float* dlogit,
                                    long long M, float loss_scale, float scale, cudaStream_t st) {
  RL_CHECK_ARG(logit && target && loss_row && dlogit, "null pointer");
  if (M <= 0) return B200RL_OK;
  bce_loss_grad_kernel<<<ceil_div(M, 256), 256, 0, st>>>(logit, target, loss_row, dlogit, M, loss_scale, scale);
  RL_CHECK_LAUNCH();
  return B200RL_OK;
}

extern "C" int b200rl_twohot_mean(const float* logits, float* out, long long M, int nb, long long ldl, float low,
                                  float high, cudaStream_t st) {
  RL_CHECK_ARG(logits && out, "null pointer");
  if (M <= 0) return B200RL_OK;
  twohot_mean_kernel<<<ceil_div(M, 8), 256, 0, st>>>(logits, out, M, nb, ldl, low, high);
  RL_CHECK_LAUNCH();
  return B200RL_OK;
}

extern "C" int b200rl_lambda_returns(const float* rew, const float* val, const float* cont_logit,
                                     const float* true_cont, float* lam, float* discount, int H, int N, float gamma,
                                     float lmbda, cudaStream_t st) {
  RL_CHECK_ARG(rew && val && cont_logit && true_cont && lam && discount, "null pointer");
  if (N <= 0 || H <= 0) return B200RL_OK;
  lambda_returns_kernel<<<ceil_div(N, 128), 128, 0, st>>>(rew, val, cont_logit, true_cont, lam, discount, H, N, gamma,
                                                          lmbda);
  RL_CHECK_LAUNCH();
  return B200RL_OK;
}

extern "C" int b200rl_moments_update(const float* x, long long n, float* state, float* out, float decay, float max_,
                                     float p_low, float p_high, cudaStream_t st) {
  RL_CHECK_ARG(x && state && out, "null pointer");
  RL_CHECK_ARG(n >= 1, "empty input");
  moments_update_kernel<<<1, 1024, 0, st>>>(x, n, state, out, decay, (float)(1.0 - (double)decay), 1.f / max_, p_low,
                                            p_high);
  RL_CHECK_LAUNCH();
  return B200RL_OK;
}

extern "C" int b200rl_actor_loss_grad(const float* raw, const float* actions, const float* lam, const float* val,
                                      const float* discount, const float* moments, float* rows, float* draw,
                                      long long M, const int* head_dims, int n_heads, float unimix, float ent_coef,
                                      float scale, cudaStream_t st) {
  RL_CHECK_ARG(raw && actions && lam && val && discount && moments && rows && draw && head_dims, "null pointer");
  RL_CHECK_ARG(n_heads >= 1 && n_heads <= MAX_HEADS, "unsupported number of action heads");
  HeadDims hd;
  hd.n = n_heads;
  int A = 0;
  for (int i = 0; i < n_heads; ++i) { hd.dim[i] = head_dims[i]; A += head_dims[i]; }
  if (M <= 0) return B200RL_OK;
  actor_loss_grad_kernel<<<ceil_div(M, 8), 256, 0, st>>>(raw, actions, lam, val, discount, moments, rows, draw, M, A, hd,
                                                         unimix, ent_coef, scale);
  RL_CHECK_LAUNCH();
  return B200RL_OK;
}

extern "C" int b200rl_sum_rows(const float* X, float* out, long long M, int C, long long ldx, float scale,
                               cudaStream_t st) {
  RL_CHECK_ARG(X && out, "null pointer");
  if (C <= 0) return B200RL_OK;
  sum_rows_kernel<<<C, 1024, 0, st>>>(X, out, M, ldx, scale);
  RL_CHECK_LAUNCH();
  return B200RL_OK;
}

extern "C" int b200rl_weighted_mean(const float* x, const float* w, float* out, long long n, float scale,
                                    cudaStream_t st) {
  RL_CHECK_ARG(x && w && out, "null pointer");
  weighted_mean_kernel<<<1, 1024, 0, st>>>(x, w, out, n, scale);
  RL_CHECK_LAUNCH();
  return B200RL_OK;
}
