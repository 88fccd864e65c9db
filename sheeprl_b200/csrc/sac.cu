// SAC update: the element-wise stages between the Linear layers (csrc/mlp.cu), one launch each.
//
// Replaces (reference): SACActor._get_actions_and_log_probs sheeprl/algos/sac/agent.py:110-142 (+ its autograd
// backward), SACAgent.get_next_target_q_values agent.py:254-262, critic_loss / policy_loss / entropy_loss
// sheeprl/algos/sac/loss.py:9-29 and the `.mean()` / `torch.min` glue of train() sheeprl/algos/sac/sac.py:45-73; DroQ's
// policy loss over the mean of its critics (sheeprl/algos/droq/droq.py:147-150).
// The temperature is read from the device-resident log_alpha (the reference does `.exp().item()`: a host sync per
// use), so a whole update can sit in one CUDA graph.  B <= a few thousand rows: single-CTA reductions.
#include "common.cuh"

namespace {

constexpr float kLogStdMax = 2.f, kLogStdMin = -5.f;          // agent.py:15-16
constexpr float kHalfLog2Pi = 0.9189385332046727f;            // log(sqrt(2*pi))

// head[b, 0:A] = mean, head[b, A:2A] = log_std.  x_t = mean + std*eps; y = tanh(x_t); a = y*scale + bias;
// logp = sum_j N(x_t; mean, std).log_prob - log(scale*(1 - y^2) + 1e-6)
__global__ void sac_sample_fwd_kernel(const float* __restrict__ head, const float* __restrict__ eps,
                                      const float* __restrict__ scale, const float* __restrict__ abias,
                                      float* __restrict__ action, long long ld_action, float* __restrict__ logp,
                                      float* __restrict__ tanh_out, int B, int A) {
  const int b = blockIdx.x * blockDim.y + threadIdx.y;
  if (b >= B) return;
  float lp = 0.f;
  for (int j = threadIdx.x; j < A; j += 32) {
    const float mean = head[(long long)b * 2 * A + j];
    const float ls = fminf(fmaxf(head[(long long)b * 2 * A + A + j], kLogStdMin), kLogStdMax);
    const float std = expf(ls);
    const float e = eps[(long long)b * A + j];
    const float xt = mean + std * e;
    const float y = tanhf(xt);
    const float d = xt - mean;
    lp += -(d * d) / (2.f * std * std) - logf(std) - kHalfLog2Pi - logf(scale[j] * (1.f - y * y) + 1e-6f);
    action[(long long)b * ld_action + j] = y * scale[j] + abias[j];
    if (tanh_out) tanh_out[(long long)b * A + j] = y;
  }
  lp = warp_sum(lp);
  if (threadIdx.x == 0) logp[b] = lp;
}

// dhead from d(action) (sum over the critics' input gradients) and d(logp) = *dlogp_scalar (same for every row).
__global__ void sac_sample_bwd_kernel(const float* __restrict__ head, const float* __restrict__ eps,
                                      const float* __restrict__ tanh_y, const float* __restrict__ scale,
                                      const float* __restrict__ dact, long long stride_net, int nets,
                                      const float* __restrict__ log_alpha, float inv_B, float* __restrict__ dhead,
                                      int B, int A) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)B * A) return;
  const int b = (int)(i / A), j = (int)(i - (long long)b * A);
  const float dlogp = expf(log_alpha[0]) * inv_B;               // d actor_loss / d logp[b]   (loss.py:9-11)
  const float raw_ls = head[(long long)b * 2 * A + A + j];
  const float ls = fminf(fmaxf(raw_ls, kLogStdMin), kLogStdMax);
  const float std = expf(ls);
  const float e = eps[i], y = tanh_y[i], s = scale[j];
  float da = 0.f;
  for (int n = 0; n < nets; ++n) da += dact[n * stride_net + i];
  const float one_m_y2 = 1.f - y * y;
  // d/dx_t: through the action and through the -log(scale*(1-y^2)+1e-6) term of logp.  The Normal log-density term
  // is -(eps^2)/2 - log std once x_t = mean + std*eps is substituted: no x_t / mean dependence.
  const float dxt = da * s * one_m_y2 + dlogp * (2.f * s * y * one_m_y2) / (s * one_m_y2 + 1e-6f);
  const float dstd = dxt * e - dlogp / std;
  const bool pass = raw_ls >= kLogStdMin && raw_ls <= kLogStdMax;   // torch.clamp passes the gradient on [min, max]
  dhead[(long long)b * 2 * A + j] = dxt;
  dhead[(long long)b * 2 * A + A + j] = pass ? dstd * std : 0.f;
}

// y = r + (1 - d) * gamma * (min_n q_target[n] - alpha * logp')          (agent.py:254-262)
__global__ void sac_target_kernel(const float* __restrict__ qt, long long stride_net, int nets,
                                  const float* __restrict__ logp, const float* __restrict__ rewards,
                                  const float* __restrict__ terminated, const float* __restrict__ log_alpha, float gamma,
                                  float* __restrict__ y, int B) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  float m = qt[b];
  for (int n = 1; n < nets; ++n) m = fminf(m, qt[n * stride_net + b]);
  const float alpha = expf(log_alpha[0]);
  y[b] = rewards[b] + (1.f - terminated[b]) * gamma * (m - alpha * logp[b]);
}

// qf_loss = sum_n mean_b (q[n,b] - y[b])^2 ; dq[n,b] = 2 (q - y) / B                 (loss.py:14-20)
__global__ void __launch_bounds__(256)
sac_critic_loss_kernel(const float* __restrict__ q, long long stride_net, int nets, const float* __restrict__ y,
                       float* __restrict__ dq, float* __restrict__ loss_out, int B) {
  __shared__ float red[32];
  float acc = 0.f;
  const float invB = 1.f / (float)B;
  for (int n = 0; n < nets; ++n)
    for (int b = threadIdx.x; b < B; b += blockDim.x) {
      const float d = q[n * stride_net + b] - y[b];
      acc += d * d;
      dq[n * stride_net + b] = 2.f * d * invB;
    }
  acc = block_sum(acc, red);
  if (threadIdx.x == 0) loss_out[0] = acc * invB;
}

// actor_loss = mean(alpha*logp - Q) with Q = min_n q[n] (SAC) or mean_n q[n] (DroQ, droq.py:147-150).
// min: dq[n,b] = -1/B at the arg-min critic (first on ties, as torch.min); mean: dq[n,b] = -1/(nets*B) for every critic.
// alpha_loss = mean(-log_alpha * (logp + target_entropy)) ; d/dlog_alpha = -mean(logp + target_entropy)
template <bool kMeanOverCritics>
__global__ void __launch_bounds__(256)
sac_actor_loss_kernel(const float* __restrict__ q, long long stride_net, int nets, const float* __restrict__ logp,
                      const float* __restrict__ log_alpha, float target_entropy, float* __restrict__ dq,
                      float* __restrict__ actor_loss, float* __restrict__ alpha_loss, float* __restrict__ dlog_alpha,
                      int B) {
  __shared__ float red[32];
  const float la = log_alpha[0], alpha = expf(la), invB = 1.f / (float)B;
  float s_actor = 0.f, s_ent = 0.f;
  for (int b = threadIdx.x; b < B; b += blockDim.x) {
    float m = q[b];
    if (kMeanOverCritics) {
      const float inv_nets = 1.f / (float)nets;
      for (int n = 1; n < nets; ++n) m += q[n * stride_net + b];
      m *= inv_nets;
      for (int n = 0; n < nets; ++n) dq[n * stride_net + b] = -invB * inv_nets;
    } else {
      int arg = 0;
      for (int n = 1; n < nets; ++n) {
        const float v = q[n * stride_net + b];
        if (v < m) { m = v; arg = n; }
      }
      for (int n = 0; n < nets; ++n) dq[n * stride_net + b] = (n == arg) ? -invB : 0.f;
    }
    s_actor += alpha * logp[b] - m;
    s_ent += logp[b] + target_entropy;
  }
  s_actor = block_sum(s_actor, red);
  s_ent = block_sum(s_ent, red);
  if (threadIdx.x == 0) {
    actor_loss[0] = s_actor * invB;
    alpha_loss[0] = -la * s_ent * invB;
    dlog_alpha[0] = -s_ent * invB;
  }
}

}  // namespace

extern "C" int b200rl_sac_sample_fwd(const float* head, const float* eps, const float* scale, const float* abias,
                                     float* action, long long ld_action, float* logp, float* tanh_out, int B, int A,
                                     cudaStream_t st) {
  RL_CHECK_ARG(head && eps && scale && abias && action && logp, "null pointer");
  RL_CHECK_ARG(B > 0 && A > 0 && ld_action >= A, "bad dims");
  dim3 block(32, 8);
  sac_sample_fwd_kernel<<<ceil_div(B, 8), block, 0, st>>>(head, eps, scale, abias, action, ld_action, logp, tanh_out, B, A);
  RL_CHECK_LAUNCH();
  return B200RL_OK;
}

extern "C" int b200rl_sac_sample_bwd(const float* head, const float* eps, const float* tanh_y, const float* scale,
                                     const float* dact, long long stride_net, int nets, const float* log_alpha,
                                     float* dhead, int B, int A, cudaStream_t st) {
  RL_CHECK_ARG(head && eps && tanh_y && scale && dact && log_alpha && dhead, "null pointer");
  RL_CHECK_ARG(B > 0 && A > 0 && nets > 0, "bad dims");
  sac_sample_bwd_kernel<<<ceil_div((long long)B * A, 256), 256, 0, st>>>(head, eps, tanh_y, scale, dact, stride_net, nets,
                                                                        log_alpha, 1.f / (float)B, dhead, B, A);
  RL_CHECK_LAUNCH();
  return B200RL_OK;
}

extern "C" int b200rl_sac_target(const float* q_target, long long stride_net, int nets, const float* logp,
                                 const float* rewards, const float* terminated, const float* log_alpha, float gamma,
                                 float* y, int B, cudaStream_t st) {
  RL_CHECK_ARG(q_target && logp && rewards && terminated && log_alpha && y, "null pointer");
  RL_CHECK_ARG(B > 0 && nets > 0, "bad dims");
  sac_target_kernel<<<ceil_div(B, 256), 256, 0, st>>>(q_target, stride_net, nets, logp, rewards, terminated, log_alpha,
                                                      gamma, y, B);
  RL_CHECK_LAUNCH();
  return B200RL_OK;
}

extern "C" int b200rl_sac_critic_loss(const float* q, long long stride_net, int nets, const float* y, float* dq,
                                      float* loss_out, int B, cudaStream_t st) {
  RL_CHECK_ARG(q && y && dq && loss_out, "null pointer");
  RL_CHECK_ARG(B > 0 && nets > 0, "bad dims");
  sac_critic_loss_kernel<<<1, 256, 0, st>>>(q, stride_net, nets, y, dq, loss_out, B);
  RL_CHECK_LAUNCH();
  return B200RL_OK;
}

template <bool kMeanOverCritics>
static int actor_loss_launch(const float* q, long long stride_net, int nets, const float* logp, const float* log_alpha,
                             float target_entropy, float* dq, float* actor_loss, float* alpha_loss, float* dlog_alpha,
                             int B, cudaStream_t st) {
  RL_CHECK_ARG(q && logp && log_alpha && dq && actor_loss && alpha_loss && dlog_alpha, "null pointer");
  RL_CHECK_ARG(B > 0 && nets > 0, "bad dims");
  sac_actor_loss_kernel<kMeanOverCritics><<<1, 256, 0, st>>>(q, stride_net, nets, logp, log_alpha, target_entropy, dq,
                                                             actor_loss, alpha_loss, dlog_alpha, B);
  RL_CHECK_LAUNCH();
  return B200RL_OK;
}

extern "C" int b200rl_sac_actor_loss(const float* q, long long stride_net, int nets, const float* logp,
                                     const float* log_alpha, float target_entropy, float* dq, float* actor_loss,
                                     float* alpha_loss, float* dlog_alpha, int B, cudaStream_t st) {
  return actor_loss_launch<false>(q, stride_net, nets, logp, log_alpha, target_entropy, dq, actor_loss, alpha_loss,
                                  dlog_alpha, B, st);
}

extern "C" int b200rl_droq_actor_loss(const float* q, long long stride_net, int nets, const float* logp,
                                      const float* log_alpha, float target_entropy, float* dq, float* actor_loss,
                                      float* alpha_loss, float* dlog_alpha, int B, cudaStream_t st) {
  return actor_loss_launch<true>(q, stride_net, nets, logp, log_alpha, target_entropy, dq, actor_loss, alpha_loss,
                                 dlog_alpha, B, st);
}
