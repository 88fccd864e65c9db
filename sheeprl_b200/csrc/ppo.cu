// PPO update: the pieces around the dense products (csrc/mlp.cu) — patch gather / scatter for the NatureCNN
// convolutions and the fused PPO objective.
//
// Replaces (reference): NatureCNN's Conv2d(k8,s4) / (k4,s2) / (k3,s1) forward + backward
// (sheeprl/models/models.py:288-328, cnn_forward utils/model.py:165-223), PPOAgent.forward's distribution glue
// (OneHotCategorical / Independent(Normal) log_prob + entropy, sheeprl/algos/ppo/agent.py:179-239),
// normalize_tensor (utils/utils.py:121-130) and policy_loss / value_loss / entropy_loss (ppo/loss.py:6-75) with
// their autograd backward.
//
// Convolutions are channel-last: rows of the patch matrix are output pixels (b, oy, ox), columns are (ky, kx, c), so
// a conv is patch-gather -> product with the [Cout, k, k, Cin] weight (stored in that layout in the flat parameter
// group) -> [B*Ho*Wo, Cout], which is already the next layer's channel-last input.  A PPO minibatch is 64..256
// images: ~6 GFLOP per update, i.e. launch-latency territory, hence the emphasis on few, fused launches.
#include "common.cuh"

namespace {

// `tanh_normal` (ppo/agent.py:194-206, 257-268): stored actions are tanh-squashed; x = safeatanh(a) with the clamp
// 1 - finfo(float32).resolution (utils/utils.py:304-313) and the reference's log-prob term 2*(log 2 - a - softplus(-2a)).
constexpr float kSafeLim = 0.999999f;
__device__ __forceinline__ float safe_atanh(float y) { return atanhf(fminf(fmaxf(y, -kSafeLim), kSafeLim)); }
__device__ __forceinline__ float tanh_logp_term(float ta) {
  const float v = -2.f * ta;
  const float sp = v > 20.f ? v : log1pf(expf(v));          // torch softplus (threshold 20)
  return 2.f * (0.6931471805599453f - ta - sp);
}

// col[(b,oy,ox), (ky,kx,c)] = x[b, oy*s+ky, ox*s+kx, c]      (no padding: NatureCNN uses none)
__global__ void im2col_kernel(const float* __restrict__ x, float* __restrict__ col, int B, int H, int W, int C, int k,
                              int s, int Ho, int Wo) {
  // 32-bit index arithmetic (host guarantees < 2^31 elements): 64-bit div/mod would dominate this copy kernel
  const unsigned total = (unsigned)B * Ho * Wo * k * k * C;
  const unsigned stride = gridDim.x * blockDim.x;
  const unsigned kkc = k * k * C, kc = k * C;
  for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) {
    const unsigned row = i / kkc, col_j = i - row * kkc;
    const unsigned ky = col_j / kc, r = col_j - ky * kc;        // r = kx*C + c : contiguous run in x
    const unsigned t = row / Wo, ox = row - t * Wo;
    const unsigned b = t / Ho, oy = t - b * Ho;
    col[i] = __ldg(x + (((size_t)b * H + oy * s + ky) * W + ox * s) * C + r);
  }
}

// dx[b,y,x,c] = mask * sum over (ky,kx) with (y-ky) % s == 0, (x-kx) % s == 0 of dcol[(b,(y-ky)/s,(x-kx)/s), (ky,kx,c)]
// mask = (act[b,y,x,c] > 0) when `act` (the ReLU output that fed this conv) is given.
__global__ void col2im_kernel(const float* __restrict__ dcol, const float* __restrict__ act, float* __restrict__ dx,
                              int B, int H, int W, int C, int k, int s, int Ho, int Wo) {
  const unsigned total = (unsigned)B * H * W * C;
  const unsigned stride = gridDim.x * blockDim.x;
  const unsigned kkc = k * k * C;
  for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) {
    unsigned t = i / C;
    const int c = (int)(i - t * C);
    const unsigned t2 = t / W;
    const int xx = (int)(t - t2 * W);
    const unsigned b = t2 / H;
    const int yy = (int)(t2 - b * H);
    float acc = 0.f;
    if (!act || act[i] > 0.f) {
      for (int ky = yy % s; ky < k && ky <= yy; ky += s) {
        const int oy = (yy - ky) / s;
        if (oy >= Ho) continue;
        for (int kx = xx % s; kx < k && kx <= xx; kx += s) {
          const int ox = (xx - kx) / s;
          if (ox >= Wo) continue;
          acc += __ldg(dcol + ((size_t)(b * Ho + oy) * Wo + ox) * kkc + (ky * k + kx) * C + c);
        }
      }
    }
    dx[i] = acc;
  }
}

struct PpoLossArgs {
  const float* head;        // discrete: logits [B, sumA]; continuous: [mean | log_std] [B, 2A]
  const float* actions;     // discrete: one-hot [B, sumA]; continuous: [B, A]
  const float* old_logp; const float* adv; const float* values; const float* old_values; const float* returns;
  float* dhead; float* dvalues; float* losses;   // losses[3] = policy, value, entropy
  const float* mask;        // ppo_loss_masked only: rows with mask != 0 enter the objective
  int B, n_heads; int head_dims[8];
  int is_continuous, clip_vloss, normalize_adv;   // is_continuous: 0 discrete, 1 Normal, 2 tanh-squashed Normal
  float clip_coef, vf_coef, ent_coef;
};

// One CTA: B is a minibatch (<= a few thousand rows).  MASKED (ppo_recurrent.py:77-101): only rows with
// mask != 0 count; the means are over their number n, advantages are normalised over them when n > 1, and the other
// rows get zero gradients.
template <bool MASKED>
__global__ void __launch_bounds__(256) ppo_loss_kernel(const PpoLossArgs a) {
  __shared__ float red[32];
  const int B = a.B;
  float n_rows = (float)B;
  if (MASKED) {
    float n = 0.f;
    for (int b = threadIdx.x; b < B; b += blockDim.x) n += (a.mask[b] != 0.f) ? 1.f : 0.f;
    n_rows = block_sum(n, red);
  }
  const float invB = MASKED ? (n_rows > 0.f ? 1.f / n_rows : 0.f) : 1.f / (float)B;
  const bool normalize = a.normalize_adv && (!MASKED || n_rows > 1.f);
  // ---- advantage normalisation (utils/utils.py:121-130): (x - mean) / (std_unbiased + 1e-8)
  float mean = 0.f, inv_std = 1.f;
  if (normalize) {
    float s = 0.f;
    for (int b = threadIdx.x; b < B; b += blockDim.x)
      if (!MASKED || a.mask[b] != 0.f) s += a.adv[b];
    mean = block_sum(s, red) * invB;
    float v = 0.f;
    for (int b = threadIdx.x; b < B; b += blockDim.x)
      if (!MASKED || a.mask[b] != 0.f) { const float d = a.adv[b] - mean; v += d * d; }
    v = block_sum(v, red) / (n_rows - 1.f);
    inv_std = 1.f / (sqrtf(v) + 1e-8f);
  }
  int width = 0;
  for (int h = 0; h < a.n_heads; ++h) width += a.head_dims[h];
  if (a.is_continuous) width *= 2;
  float s_pg = 0.f, s_v = 0.f, s_e = 0.f;
  for (int b = threadIdx.x; b < B; b += blockDim.x) {
    const float* hd = a.head + (long long)b * width;
    float* dh = a.dhead + (long long)b * width;
    if (MASKED && a.mask[b] == 0.f) {
      for (int j = 0; j < width; ++j) dh[j] = 0.f;
      a.dvalues[b] = 0.f;
      continue;
    }
    float lp = 0.f, ent = 0.f;
    // ---- pass 1: log-prob of the taken action and entropy (ppo/agent.py:179-239)
    if (a.is_continuous) {
      const int A = width / 2;
      float corr = 0.f;
      for (int j = 0; j < A; ++j) {
        float x = a.actions[(long long)b * A + j];
        if (a.is_continuous == 2) { corr += tanh_logp_term(x); x = safe_atanh(x); }
        const float mu = hd[j], ls = hd[A + j], sd = expf(ls), d = x - mu;
        lp += -(d * d) / (2.f * sd * sd) - ls - 0.9189385332046727f;
        ent += 0.5f + 0.9189385332046727f + ls;
      }
      lp -= corr;
    } else {
      int off = 0;
      for (int h = 0; h < a.n_heads; ++h) {
        const int n = a.head_dims[h];
        float m = -INFINITY;
        for (int j = 0; j < n; ++j) m = fmaxf(m, hd[off + j]);
        float z = 0.f;
        for (int j = 0; j < n; ++j) z += expf(hd[off + j] - m);
        const float lse = m + logf(z);
        float hh = 0.f;
        for (int j = 0; j < n; ++j) {
          const float lpj = hd[off + j] - lse;
          lp += lpj * a.actions[(long long)b * width + off + j];
          hh -= expf(lpj) * lpj;
        }
        ent += hh;
        off += n;
      }
    }
    // ---- objective (ppo/loss.py) and d/dlp, d/dent, d/dvalue
    const float adv = (a.adv[b] - mean) * inv_std;
    const float ratio = expf(lp - a.old_logp[b]);
    const float pg1 = adv * ratio;
    const float pg2 = adv * fminf(fmaxf(ratio, 1.f - a.clip_coef), 1.f + a.clip_coef);
    s_pg += -fminf(pg1, pg2);
    const float dlp = (pg1 <= pg2) ? -pg1 * invB : 0.f;             // d(-min)/dlp = -adv*ratio on the unclipped branch
    const float val = a.values[b], ret = a.returns[b];
    float dval;
    if (a.clip_vloss) {
      const float old = a.old_values[b];
      const float dv = val - old;
      const float vc = old + fminf(fmaxf(dv, -a.clip_coef), a.clip_coef);
      const float u = (val - ret) * (val - ret), c = (vc - ret) * (vc - ret);
      s_v += 0.5f * fmaxf(u, c);
      const float inside = (dv >= -a.clip_coef && dv <= a.clip_coef) ? 1.f : 0.f;
      const float gu = (val - ret), gc = (vc - ret) * inside;
      dval = (u > c) ? gu : ((u < c) ? gc : 0.5f * (gu + gc));        // torch.max splits ties evenly
    } else {
      s_v += (val - ret) * (val - ret);
      dval = 2.f * (val - ret);
    }
    a.dvalues[b] = a.vf_coef * dval * invB;
    s_e += -ent;
    const float dent = -a.ent_coef * invB;
    // ---- pass 2: gradient w.r.t. the head outputs
    if (a.is_continuous) {
      const int A = width / 2;
      for (int j = 0; j < A; ++j) {
        float x = a.actions[(long long)b * A + j];
        if (a.is_continuous == 2) x = safe_atanh(x);             // the squash term does not depend on the head
        const float mu = hd[j], ls = hd[A + j], sd = expf(ls), d = x - mu;
        dh[j] = dlp * d / (sd * sd);
        dh[A + j] = dlp * (d * d / (sd * sd) - 1.f) + dent;
      }
    } else {
      int off = 0;
      for (int h = 0; h < a.n_heads; ++h) {
        const int n = a.head_dims[h];
        float m = -INFINITY;
        for (int j = 0; j < n; ++j) m = fmaxf(m, hd[off + j]);
        float z = 0.f;
        for (int j = 0; j < n; ++j) z += expf(hd[off + j] - m);
        const float lse = m + logf(z);
        float hh = 0.f, asum = 0.f;
        for (int j = 0; j < n; ++j) {
          const float lpj = hd[off + j] - lse;
          hh -= expf(lpj) * lpj;
          asum += a.actions[(long long)b * width + off + j];
        }
        for (int j = 0; j < n; ++j) {
          const float lpj = hd[off + j] - lse, pj = expf(lpj);
          dh[off + j] = dlp * (a.actions[(long long)b * width + off + j] - pj * asum) - dent * pj * (lpj + hh);
        }
        off += n;
      }
    }
  }
  s_pg = block_sum(s_pg, red);
  s_v = block_sum(s_v, red);
  s_e = block_sum(s_e, red);
  if (threadIdx.x == 0) {
    a.losses[0] = s_pg * invB;
    a.losses[1] = s_v * invB;
    a.losses[2] = s_e * invB;
  }
}

// PPOPlayer.forward (ppo/agent.py:269-293): sample an action per head (OneHotCategorical: arg-max of p / q with
// q ~ Exp(1), identical to torch.multinomial; Normal: mean + std * eps) or take the mode / mean when greedy, and
// its log-probability.  Thread per row.
__global__ void ppo_act_kernel(const float* __restrict__ head, const float* __restrict__ noise, float* __restrict__ actions,
                               float* __restrict__ logp, int B, int n_heads, PpoLossArgs dims, int is_continuous,
                               int greedy) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  int width = 0;
  for (int h = 0; h < n_heads; ++h) width += dims.head_dims[h];
  float lp = 0.f;
  if (is_continuous) {
    const int A = width;
    const float* hd = head + (long long)b * 2 * A;
    // is_continuous: 1 Normal; 2 tanh_normal as PPOPlayer.forward returns it (safetanh of the sample, corrected
    // log-prob, agent.py:257-268); 3 tanh_normal as PPOPlayer.get_actions returns it (safeatanh of the sample / mean,
    // agent.py:306-311 — the reference's behaviour, kept as is)
    for (int j = 0; j < A; ++j) {
      const float mu = hd[j], ls = hd[A + j], sd = expf(ls);
      const float e = (greedy || !noise) ? 0.f : noise[(long long)b * A + j];
      float a = mu + sd * e;
      const float d = a - mu;
      lp += -(d * d) / (2.f * sd * sd) - ls - 0.9189385332046727f;
      if (is_continuous == 2) {
        a = fminf(fmaxf(tanhf(a), -kSafeLim), kSafeLim);
        lp -= tanh_logp_term(a);
      } else if (is_continuous == 3) {
        a = safe_atanh(a);
      }
      actions[(long long)b * A + j] = a;
    }
  } else {
    const float* hd = head + (long long)b * width;
    int off = 0;
    for (int h = 0; h < n_heads; ++h) {
      const int n = dims.head_dims[h];
      float m = -INFINITY;
      for (int j = 0; j < n; ++j) m = fmaxf(m, hd[off + j]);
      float z = 0.f;
      for (int j = 0; j < n; ++j) z += expf(hd[off + j] - m);
      const float lse = m + logf(z);
      float best = -INFINITY;
      int arg = 0;
      for (int j = 0; j < n; ++j) {
        float p = expf(hd[off + j] - lse);
        if (!greedy && noise) p = p / noise[(long long)b * width + off + j];
        if (p > best) { best = p; arg = j; }
      }
      for (int j = 0; j < n; ++j) actions[(long long)b * width + off + j] = (j == arg) ? 1.f : 0.f;
      lp += hd[off + arg] - lse;
      off += n;
    }
  }
  logp[b] = lp;
}

}  // namespace

extern "C" int b200rl_im2col(const float* x, float* col, int B, int H, int W, int C, int k, int stride, cudaStream_t st) {
  RL_CHECK_ARG(x && col, "null pointer");
  RL_CHECK_ARG(B > 0 && H >= k && W >= k && C > 0 && k > 0 && stride > 0, "bad dims");
  const int Ho = (H - k) / stride + 1, Wo = (W - k) / stride + 1;
  const long long total = (long long)B * Ho * Wo * k * k * C;
  RL_CHECK_ARG(total < 2147483647LL, "patch matrix too large for 32-bit indexing: split the minibatch");
  long long blocks = (total + 255) / 256;
  if (blocks > (long long)kNumSMs * 16) blocks = (long long)kNumSMs * 16;
  im2col_kernel<<<(unsigned)blocks, 256, 0, st>>>(x, col, B, H, W, C, k, stride, Ho, Wo);
  RL_CHECK_LAUNCH();
  return B200RL_OK;
}

extern "C" int b200rl_col2im(const float* dcol, const float* act, float* dx, int B, int H, int W, int C, int k, int stride,
                             cudaStream_t st) {
  RL_CHECK_ARG(dcol && dx, "null pointer");
  RL_CHECK_ARG(B > 0 && H >= k && W >= k && C > 0 && k > 0 && stride > 0, "bad dims");
  const int Ho = (H - k) / stride + 1, Wo = (W - k) / stride + 1;
  const long long total = (long long)B * H * W * C;
  RL_CHECK_ARG(total < 2147483647LL && (long long)B * Ho * Wo * k * k * C < 2147483647LL, "image too large for 32-bit indexing");
  long long blocks = (total + 255) / 256;
  if (blocks > (long long)kNumSMs * 16) blocks = (long long)kNumSMs * 16;
  col2im_kernel<<<(unsigned)blocks, 256, 0, st>>>(dcol, act, dx, B, H, W, C, k, stride, Ho, Wo);
  RL_CHECK_LAUNCH();
  return B200RL_OK;
}

extern "C" int b200rl_ppo_loss(const float* head, const float* actions, const float* old_logp, const float* adv,
                               const float* values, const float* old_values, const float* returns, float* dhead,
                               float* dvalues, float* losses, int B, const int* head_dims, int n_heads, int is_continuous,
                               int clip_vloss, int normalize_adv, float clip_coef, float vf_coef, float ent_coef,
                               cudaStream_t st) {
  RL_CHECK_ARG(head && actions && old_logp && adv && values && old_values && returns && dhead && dvalues && losses,
               "null pointer");
  RL_CHECK_ARG(B > 0 && n_heads > 0 && n_heads <= 8 && head_dims, "bad dims (at most 8 action heads)");
  RL_CHECK_ARG(!normalize_adv || B > 1, "advantage normalisation needs at least two rows");
  RL_CHECK_ARG(is_continuous >= 0 && is_continuous <= 2, "is_continuous: 0 discrete, 1 normal, 2 tanh_normal");
  PpoLossArgs a{};
  a.head = head; a.actions = actions; a.old_logp = old_logp; a.adv = adv; a.values = values;
  a.old_values = old_values; a.returns = returns; a.dhead = dhead; a.dvalues = dvalues; a.losses = losses;
  a.B = B; a.n_heads = n_heads;
  for (int i = 0; i < n_heads; ++i) a.head_dims[i] = head_dims[i];
  a.is_continuous = is_continuous; a.clip_vloss = clip_vloss; a.normalize_adv = normalize_adv;
  a.clip_coef = clip_coef; a.vf_coef = vf_coef; a.ent_coef = ent_coef;
  ppo_loss_kernel<false><<<1, 256, 0, st>>>(a);
  RL_CHECK_LAUNCH();
  return B200RL_OK;
}

extern "C" int b200rl_ppo_loss_masked(const float* head, const float* actions, const float* old_logp, const float* adv,
                                      const float* values, const float* old_values, const float* returns,
                                      const float* mask, float* dhead, float* dvalues, float* losses, int B,
                                      const int* head_dims, int n_heads, int is_continuous, int clip_vloss,
                                      int normalize_adv, float clip_coef, float vf_coef, float ent_coef,
                                      cudaStream_t st) {
  RL_CHECK_ARG(head && actions && old_logp && adv && values && old_values && returns && mask && dhead && dvalues &&
               losses, "null pointer");
  RL_CHECK_ARG(B > 0 && n_heads > 0 && n_heads <= 8 && head_dims, "bad dims (at most 8 action heads)");
  RL_CHECK_ARG(is_continuous >= 0 && is_continuous <= 2, "is_continuous: 0 discrete, 1 normal, 2 tanh_normal");
  PpoLossArgs a{};
  a.head = head; a.actions = actions; a.old_logp = old_logp; a.adv = adv; a.values = values;
  a.old_values = old_values; a.returns = returns; a.dhead = dhead; a.dvalues = dvalues; a.losses = losses;
  a.mask = mask; a.B = B; a.n_heads = n_heads;
  for (int i = 0; i < n_heads; ++i) a.head_dims[i] = head_dims[i];
  a.is_continuous = is_continuous; a.clip_vloss = clip_vloss; a.normalize_adv = normalize_adv;
  a.clip_coef = clip_coef; a.vf_coef = vf_coef; a.ent_coef = ent_coef;
  ppo_loss_kernel<true><<<1, 256, 0, st>>>(a);
  RL_CHECK_LAUNCH();
  return B200RL_OK;
}

extern "C" int b200rl_ppo_act(const float* head, const float* noise, float* actions, float* logp, int B,
                              const int* head_dims, int n_heads, int is_continuous, int greedy, cudaStream_t st) {
  RL_CHECK_ARG(head && actions && logp && head_dims, "null pointer");
  RL_CHECK_ARG(B > 0 && n_heads > 0 && n_heads <= 8, "bad dims (at most 8 action heads)");
  RL_CHECK_ARG(is_continuous >= 0 && is_continuous <= 3, "is_continuous: 0 discrete, 1 normal, 2 / 3 tanh_normal");
  PpoLossArgs d{};
  for (int i = 0; i < n_heads; ++i) d.head_dims[i] = head_dims[i];
  ppo_act_kernel<<<ceil_div(B, 128), 128, 0, st>>>(head, noise, actions, logp, B, n_heads, d, is_continuous, greedy);
  RL_CHECK_LAUNCH();
  return B200RL_OK;
}
