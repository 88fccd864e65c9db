// RSSM element-wise / small-reduction kernels: GRU gate, is_first masking, unimix + categorical
// straight-through sampling, categorical KL with free nats.  32-way class groups map onto the 32 lanes
// of a warp, so softmax / log-sum-exp / KL / arg-max reductions are pure warp shuffles.
//
// Replaces (reference): LayerNormGRUCell gate math (sheeprl/models/models.py:399-403), RSSM.dynamic masking
// (agent.py:425-430), RSSM._uniform_mix (agent.py:437-449), compute_stochastic_state
// (dreamer_v2/utils.py:44-61) incl. torch's OneHotCategoricalStraightThrough / Categorical semantics,
// the KL-balancing part of reconstruction_loss (dreamer_v3/loss.py:61-75), and their backward.
#include "common.cuh"

namespace {

__global__ void gru_gate_fwd_kernel(const float* __restrict__ G, const float* __restrict__ Hin, float* __restrict__ Hout,
                                    long long M, int R, long long ldg, long long ldhi, long long ldho) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= M * R) return;
  const long long m = idx / R;
  const int j = (int)(idx - m * R);
  const float* g = G + m * ldg;
  const float r = sigmoidf_(g[j]);
  const float c = tanhf(r * g[R + j]);
  const float u = sigmoidf_(g[2 * R + j] - 1.f);
  const float h = Hin[m * ldhi + j];
  Hout[m * ldho + j] = u * c + (1.f - u) * h;
}

__global__ void gru_gate_bwd_kernel(const float* __restrict__ G, const float* __restrict__ Hin,
                                    const float* __restrict__ dH, float* __restrict__ dG, float* __restrict__ dHin,
                                    long long M, int R, long long ldg, long long ldhi, long long lddh,
                                    long long lddg, long long lddhi) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= M * R) return;
  const long long m = idx / R;
  const int j = (int)(idx - m * R);
  const float* g = G + m * ldg;
  const float gc = g[R + j];
  const float r = sigmoidf_(g[j]);
  const float c = tanhf(r * gc);
  const float u = sigmoidf_(g[2 * R + j] - 1.f);
  const float h = Hin[m * ldhi + j];
  const float dh = dH[m * lddh + j];
  const float du = dh * (c - h);
  const float drc = dh * u * (1.f - c * c);
  float* dg = dG + m * lddg;
  dg[j] = drc * gc * r * (1.f - r);
  dg[R + j] = drc * r;
  dg[2 * R + j] = du * u * (1.f - u);
  dHin[m * lddhi + j] = dh * (1.f - u);
}

// out[m,c] = (1-f[m]) * prev[m,c] + f[m] * init[c]   (init == nullptr: plain row masking)
__global__ void mask_mix_kernel(const float* __restrict__ prev, const float* __restrict__ init,
                                const float* __restrict__ first, float* __restrict__ out, long long M, int C,
                                long long ldp, long long ldo) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= M * C) return;
  const long long m = idx / C;
  const int c = (int)(idx - m * C);
  const float f = first[m];
  float v = (1.f - f) * prev[m * ldp + c];
  if (init) v += f * init[c];
  out[m * ldo + c] = v;
}

// dPrev[m,c] = (1-f[m]) * dIn[m,c];  dInit[c] += sum_m f[m]*dIn[m,c]   (one thread per column, M small)
__global__ void mask_bwd_kernel(const float* __restrict__ dIn, const float* __restrict__ first,
                                float* __restrict__ dPrev, float* __restrict__ dInit, int M, int C, long long ldi,
                                long long ldp) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  float s = 0.f;
  for (int m = 0; m < M; ++m) {
    const float f = first[m];
    const float d = dIn[m * ldi + c];
    dPrev[m * ldp + c] = (1.f - f) * d;
    s = fmaf(f, d, s);
  }
  if (dInit) dInit[c] += s;
}

struct GroupStats {
  float raw_max, raw_sum;  // softmax of raw logits: s = exp(x-raw_max)/raw_sum
  float lse;               // logsumexp of the unimix log-probs (torch Categorical normalisation)
};

__device__ __forceinline__ float unimix_logprob(float s, float unimix, float invK, float& pm) {
  pm = (1.f - unimix) * s + unimix * invK;
  return logf(fminf(fmaxf(pm, kFp32Eps), 1.f - kFp32Eps));
}

// One warp per (row, group).  Computes everything the forward/backward need about one categorical.
__device__ __forceinline__ GroupStats group_stats(const float* x, int K, float unimix, int lane) {
  GroupStats st;
  float mx = -INFINITY;
  for (int c = lane; c < K; c += 32) mx = fmaxf(mx, x[c]);
  mx = warp_max(mx);
  float sm = 0.f;
  for (int c = lane; c < K; c += 32) sm += expf(x[c] - mx);
  sm = warp_sum(sm);
  st.raw_max = mx;
  st.raw_sum = sm;
  const float invK = 1.f / (float)K;
  // logsumexp over l_c (max-shifted like torch.logsumexp)
  float lmx = -INFINITY;
  for (int c = lane; c < K; c += 32) {
    float l = x[c];
    if (unimix > 0.f) { float pm; l = unimix_logprob(expf(x[c] - mx) / sm, unimix, invK, pm); }
    lmx = fmaxf(lmx, l);
  }
  lmx = warp_max(lmx);
  float ls = 0.f;
  for (int c = lane; c < K; c += 32) {
    float l = x[c];
    if (unimix > 0.f) { float pm; l = unimix_logprob(expf(x[c] - mx) / sm, unimix, invK, pm); }
    ls += expf(l - lmx);
  }
  ls = warp_sum(ls);
  st.lse = lmx + logf(ls);
  return st;
}

__global__ void __launch_bounds__(256)
cat_sample_kernel(const float* __restrict__ raw, const float* __restrict__ noise, float* __restrict__ onehot,
                  float* __restrict__ mix_out, long long M, int groups, int K, long long ldr, long long ldn,
                  long long ldo, long long ldm, float unimix) {
  const int lane = threadIdx.x & 31;
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (warp >= M * groups) return;
  const long long m = warp / groups;
  const int g = (int)(warp - m * groups);
  const float* x = raw + m * ldr + (long long)g * K;
  const GroupStats st = group_stats(x, K, unimix, lane);
  const float invK = 1.f / (float)K;
  // normalised log-probs lg = l - lse; probs = softmax(lg) (max-shifted); ratio = probs / q
  float lgmax = -INFINITY;
  for (int c = lane; c < K; c += 32) {
    float l = x[c];
    if (unimix > 0.f) { float pm; l = unimix_logprob(expf(x[c] - st.raw_max) / st.raw_sum, unimix, invK, pm); }
    if (mix_out) mix_out[m * ldm + (long long)g * K + c] = l;
    lgmax = fmaxf(lgmax, l - st.lse);
  }
  lgmax = warp_max(lgmax);
  float psum = 0.f;
  for (int c = lane; c < K; c += 32) {
    float l = x[c];
    if (unimix > 0.f) { float pm; l = unimix_logprob(expf(x[c] - st.raw_max) / st.raw_sum, unimix, invK, pm); }
    psum += expf(l - st.lse - lgmax);
  }
  psum = warp_sum(psum);
  if (!onehot) return;
  float best = -INFINITY;
  int besti = 0x7fffffff;
  for (int c = lane; c < K; c += 32) {
    float l = x[c];
    if (unimix > 0.f) { float pm; l = unimix_logprob(expf(x[c] - st.raw_max) / st.raw_sum, unimix, invK, pm); }
    float p = expf(l - st.lse - lgmax) / psum;
    if (noise) p = p / noise[m * ldn + (long long)g * K + c];
    if (p > best) { best = p; besti = c; }  // strict > keeps the first maximum within a lane
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ob = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, besti, o);
    if (ob > best || (ob == best && oi < besti)) { best = ob; besti = oi; }
  }
  for (int c = lane; c < K; c += 32) onehot[m * ldo + (long long)g * K + c] = (c == besti) ? 1.f : 0.f;
}

// K <= 32: one class per lane, every quantity computed once and kept in a register.  Same expressions and the same
// butterfly reductions as cat_sample_kernel, so samples and log-probs are bit-identical to the general path.
__device__ __forceinline__ void cat_sample_lane(float xv, bool on, int K, int lane, float unimix,
                                                const float* __restrict__ noise_row, float* __restrict__ onehot_row,
                                                float* __restrict__ mix_row) {
  const float mx = warp_max(xv);
  const float sm = warp_sum(on ? expf(xv - mx) : 0.f);
  const float invK = 1.f / (float)K;
  float l = xv;
  if (unimix > 0.f && on) { float pm; l = unimix_logprob(expf(xv - mx) / sm, unimix, invK, pm); }
  const float lmx = warp_max(on ? l : -INFINITY);
  const float ls = warp_sum(on ? expf(l - lmx) : 0.f);
  const float lse = lmx + logf(ls);
  if (mix_row && on) mix_row[lane] = l;
  const float lgmax = warp_max(on ? l - lse : -INFINITY);
  const float e = on ? expf(l - lse - lgmax) : 0.f;
  const float psum = warp_sum(e);
  if (!onehot_row) return;
  float best = -INFINITY;
  int besti = 0x7fffffff;
  if (on) {
    float p = e / psum;
    if (noise_row) p = p / noise_row[lane];
    if (p > best) { best = p; besti = lane; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ob = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, besti, o);
    if (ob > best || (ob == best && oi < besti)) { best = ob; besti = oi; }
  }
  if (on) onehot_row[lane] = (lane == besti) ? 1.f : 0.f;
}

__global__ void __launch_bounds__(256)
cat_sample_small_kernel(const float* __restrict__ raw, const float* __restrict__ noise, float* __restrict__ onehot,
                        float* __restrict__ mix_out, long long M, int groups, int K, long long ldr, long long ldn,
                        long long ldo, long long ldm, float unimix) {
  const int lane = threadIdx.x & 31;
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (warp >= M * groups) return;
  const long long m = warp / groups;
  const int g = (int)(warp - m * groups);
  const bool on = lane < K;
  const float xv = on ? raw[m * ldr + (long long)g * K + lane] : -INFINITY;
  cat_sample_lane(xv, on, K, lane, unimix, noise ? noise + m * ldn + (long long)g * K : nullptr,
                  onehot ? onehot + m * ldo + (long long)g * K : nullptr, mix_out ? mix_out + m * ldm + (long long)g * K : nullptr);
}

// Policy head + sample in one launch (Actor.mlp_heads[i] then OneHotCategoricalStraightThrough.rsample, agent.py:793-818):
// one warp per row computes the A <= 32 logits of a [A, Kin] Linear (+ bias) on its row (Kin % 4 == 0, Kin <= 1024: the
// row stays in registers), writes them (`raw`, kept for the policy gradient) and draws the sample like cat_sample.
__global__ void __launch_bounds__(256)
head_sample_kernel(const float* __restrict__ X, const float* __restrict__ W, const float* __restrict__ bias,
                   const float* __restrict__ noise, float* __restrict__ raw, float* __restrict__ onehot, long long M, int Kin,
                   int A, long long ldx, long long ldw, long long ldr, long long ldn, long long ldo, float unimix) {
  const int lane = threadIdx.x & 31;
  const long long m = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (m >= M) return;
  const int k4 = Kin >> 2;
  float4 x[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int c = lane + 32 * i;
    x[i] = c < k4 ? reinterpret_cast<const float4*>(X + m * ldx)[c] : make_float4(0.f, 0.f, 0.f, 0.f);
  }
  float mine = -INFINITY;
  for (int a = 0; a < A; ++a) {
    const float4* w = reinterpret_cast<const float4*>(W + (long long)a * ldw);
    float acc = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int c = lane + 32 * i;
      if (c < k4) {
        const float4 t = __ldg(w + c);
        acc = fmaf(x[i].x, t.x, acc); acc = fmaf(x[i].y, t.y, acc); acc = fmaf(x[i].z, t.z, acc); acc = fmaf(x[i].w, t.w, acc);
      }
    }
    acc = warp_sum(acc);
    if (lane == a) mine = acc + (bias ? bias[a] : 0.f);
  }
  const bool on = lane < A;
  if (on) raw[m * ldr + lane] = mine;
  cat_sample_lane(mine, on, A, lane, unimix, noise ? noise + m * ldn : nullptr, onehot + m * ldo, nullptr);
}

// MineDojo functional actions whose argument head is masked (sheeprl/envs/minedojo.py ACTION_MAP; agent.py:905-924)
constexpr int kMinedojoCraft = 15, kMinedojoEquip = 16, kMinedojoPlace = 17, kMinedojoDestroy = 18;

// One K-way head of one row on one warp, with an optional class mask (nonzero = allowed): unimix over ALL K classes,
// then the disallowed log-probs become -inf (they are skipped), then torch's Categorical normalisation and the
// exponential race of cat_sample_kernel (noise == nullptr: the mode).  The loops, expressions and butterfly
// reductions are cat_sample_kernel's, so with every class allowed the one-hot is bit-identical to it (and to
// cat_sample_small_kernel, which is bit-identical to it).  A mask that allows no class is ignored: the head falls back
// to its unmasked distribution.  Returns the drawn class on every lane.
__device__ __forceinline__ int masked_head_sample(const float* __restrict__ x, int K, const float* __restrict__ mask,
                                                  const float* __restrict__ noise, float* __restrict__ onehot,
                                                  float unimix, int lane) {
  bool any = false;
  if (mask) {
    for (int c = lane; c < K; c += 32) any = any || mask[c] != 0.f;
    any = __any_sync(0xffffffffu, any);
  }
  const float* mk = any ? mask : nullptr;
  float mx = -INFINITY;
  for (int c = lane; c < K; c += 32) mx = fmaxf(mx, x[c]);
  mx = warp_max(mx);
  float sm = 0.f;
  for (int c = lane; c < K; c += 32) sm += expf(x[c] - mx);
  sm = warp_sum(sm);
  const float invK = 1.f / (float)K;
  float lmx = -INFINITY;
  for (int c = lane; c < K; c += 32) {
    if (mk && mk[c] == 0.f) continue;
    float l = x[c];
    if (unimix > 0.f) { float pm; l = unimix_logprob(expf(x[c] - mx) / sm, unimix, invK, pm); }
    lmx = fmaxf(lmx, l);
  }
  lmx = warp_max(lmx);
  float ls = 0.f;
  for (int c = lane; c < K; c += 32) {
    if (mk && mk[c] == 0.f) continue;
    float l = x[c];
    if (unimix > 0.f) { float pm; l = unimix_logprob(expf(x[c] - mx) / sm, unimix, invK, pm); }
    ls += expf(l - lmx);
  }
  ls = warp_sum(ls);
  const float lse = lmx + logf(ls);
  float lgmax = -INFINITY;
  for (int c = lane; c < K; c += 32) {
    if (mk && mk[c] == 0.f) continue;
    float l = x[c];
    if (unimix > 0.f) { float pm; l = unimix_logprob(expf(x[c] - mx) / sm, unimix, invK, pm); }
    lgmax = fmaxf(lgmax, l - lse);
  }
  lgmax = warp_max(lgmax);
  float psum = 0.f;
  for (int c = lane; c < K; c += 32) {
    if (mk && mk[c] == 0.f) continue;
    float l = x[c];
    if (unimix > 0.f) { float pm; l = unimix_logprob(expf(x[c] - mx) / sm, unimix, invK, pm); }
    psum += expf(l - lse - lgmax);
  }
  psum = warp_sum(psum);
  float best = -INFINITY;
  int besti = 0x7fffffff;
  for (int c = lane; c < K; c += 32) {
    if (mk && mk[c] == 0.f) continue;
    float l = x[c];
    if (unimix > 0.f) { float pm; l = unimix_logprob(expf(x[c] - mx) / sm, unimix, invK, pm); }
    float p = expf(l - lse - lgmax) / psum;
    if (noise) p = p / noise[c];
    if (p > best) { best = p; besti = c; }  // strict > keeps the first maximum within a lane
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ob = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, besti, o);
    if (ob > best || (ob == best && oi < besti)) { best = ob; besti = oi; }
  }
  for (int c = lane; c < K; c += 32) onehot[c] = (c == besti) ? 1.f : 0.f;
  return besti;
}

// MinedojoActor.forward with action masks (agent.py:898-932): one warp per row draws the functional action (head 0,
// masked by mask_action_type), then the craft / smelt item (head 1, masked by mask_craft_smelt where head 0 drew
// craft) and the item (head 2, masked by mask_equip_place after equip / place, by mask_destroy after destroy).  The
// three heads are consecutive column blocks of one row in raw, noise and onehot.  No atomics: every row's result
// depends on its own inputs only.
__global__ void __launch_bounds__(256)
minedojo_sample_kernel(const float* __restrict__ raw, const float* __restrict__ noise, float* __restrict__ onehot,
                       const float* __restrict__ m_type, const float* __restrict__ m_craft,
                       const float* __restrict__ m_equip, const float* __restrict__ m_destroy, long long M, int K0,
                       int K1, int K2, long long ldr, long long ldn, long long ldo, long long ld_type,
                       long long ld_craft, long long ld_equip, long long ld_destroy, float unimix) {
  const int lane = threadIdx.x & 31;
  const long long m = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (m >= M) return;
  const float* x = raw + m * ldr;
  const float* q = noise ? noise + m * ldn : nullptr;
  float* o = onehot + m * ldo;
  const int a0 = masked_head_sample(x, K0, m_type ? m_type + m * ld_type : nullptr, q, o, unimix, lane);
  const float* mk1 = (a0 == kMinedojoCraft && m_craft) ? m_craft + m * ld_craft : nullptr;
  masked_head_sample(x + K0, K1, mk1, q ? q + K0 : nullptr, o + K0, unimix, lane);
  const float* mk2 = nullptr;
  if ((a0 == kMinedojoEquip || a0 == kMinedojoPlace) && m_equip) mk2 = m_equip + m * ld_equip;
  else if (a0 == kMinedojoDestroy && m_destroy) mk2 = m_destroy + m * ld_destroy;
  masked_head_sample(x + K0 + K1, K2, mk2, q ? q + K0 + K1 : nullptr, o + K0 + K1, unimix, lane);
}

__global__ void __launch_bounds__(256)
cat_sample_bwd_kernel(const float* __restrict__ raw, const float* __restrict__ dz, const float* __restrict__ dmix,
                      float* __restrict__ draw, long long M, int groups, int K, long long ldr, long long lddz,
                      long long lddm, long long lddr, float unimix) {
  const int lane = threadIdx.x & 31;
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (warp >= M * groups) return;
  const long long m = warp / groups;
  const int g = (int)(warp - m * groups);
  const long long go = (long long)g * K;
  const float* x = raw + m * ldr + go;
  const GroupStats st = group_stats(x, K, unimix, lane);
  const float invK = 1.f / (float)K;
  // pass 1: sum_c p_c * dz_c  (p = exp(l - lse): softmax of the normalised log-probs)
  float pdz = 0.f;
  if (dz) {
    for (int c = lane; c < K; c += 32) {
      float l = x[c];
      if (unimix > 0.f) { float pm; l = unimix_logprob(expf(x[c] - st.raw_max) / st.raw_sum, unimix, invK, pm); }
      pdz = fmaf(expf(l - st.lse), dz[m * lddz + go + c], pdz);
    }
    pdz = warp_sum(pdz);
  }
  // pass 2: g_c = dmix_c + p_c (dz_c - pdz); ds_c = g_c (1-u)/pm_c; sds = sum s_c ds_c
  float sds = 0.f;
  for (int c = lane; c < K; c += 32) {
    const float s = expf(x[c] - st.raw_max) / st.raw_sum;
    float pm = 0.f, l = x[c];
    if (unimix > 0.f) l = unimix_logprob(s, unimix, invK, pm);
    float gg = dmix ? dmix[m * lddm + go + c] : 0.f;
    if (dz) gg += expf(l - st.lse) * (dz[m * lddz + go + c] - pdz);
    if (unimix > 0.f) {
      const bool inside = pm >= kFp32Eps && pm <= 1.f - kFp32Eps;
      const float ds = inside ? gg * (1.f - unimix) / pm : 0.f;
      sds = fmaf(s, ds, sds);
    }
  }
  sds = warp_sum(sds);
  for (int c = lane; c < K; c += 32) {
    const float s = expf(x[c] - st.raw_max) / st.raw_sum;
    float pm = 0.f, l = x[c];
    if (unimix > 0.f) l = unimix_logprob(s, unimix, invK, pm);
    float gg = dmix ? dmix[m * lddm + go + c] : 0.f;
    if (dz) gg += expf(l - st.lse) * (dz[m * lddz + go + c] - pdz);
    if (unimix > 0.f) {
      const bool inside = pm >= kFp32Eps && pm <= 1.f - kFp32Eps;
      const float ds = inside ? gg * (1.f - unimix) / pm : 0.f;
      gg = s * (ds - sds);
    }
    draw[m * lddr + go + c] = gg;
  }
}

// One block (8 warps) per row; warps loop over the groups.  Inputs are unimix log-probs.
__global__ void __launch_bounds__(256)
kl_loss_grad_kernel(const float* __restrict__ post, const float* __restrict__ prior, float* __restrict__ d_post,
                    float* __restrict__ d_prior, float* __restrict__ rows, int groups, int K, long long ldp,
                    long long ldq, long long lddp, long long lddq, float kl_dyn, float kl_rep, float free_nats,
                    float coef /* scale * regularizer */) {
  __shared__ float red[32];
  const long long m = blockIdx.x;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const float* lp0 = post + m * ldp;
  const float* lq0 = prior + m * ldq;
  float kl = 0.f, hp = 0.f, hq = 0.f;
  for (int g = wid; g < groups; g += nw) {
    const float* a = lp0 + (long long)g * K;
    const float* b = lq0 + (long long)g * K;
    float ma = -INFINITY, mb = -INFINITY;
    for (int c = lane; c < K; c += 32) { ma = fmaxf(ma, a[c]); mb = fmaxf(mb, b[c]); }
    ma = warp_max(ma); mb = warp_max(mb);
    float sa = 0.f, sb = 0.f;
    for (int c = lane; c < K; c += 32) { sa += expf(a[c] - ma); sb += expf(b[c] - mb); }
    const float lsea = ma + logf(warp_sum(sa)), lseb = mb + logf(warp_sum(sb));
    float t = 0.f, ea = 0.f, eb = 0.f;
    for (int c = lane; c < K; c += 32) {
      const float lpa = a[c] - lsea, lqb = b[c] - lseb;
      const float pa = expf(lpa), pb = expf(lqb);
      t = fmaf(pa, lpa - lqb, t);
      ea = fmaf(-pa, lpa, ea);
      eb = fmaf(-pb, lqb, eb);
    }
    kl += t; hp += ea; hq += eb;  // per-lane partials; reduced below
  }
  kl = block_sum(kl, red);
  hp = block_sum(hp, red);
  hq = block_sum(hq, red);
  if (threadIdx.x == 0) {
    rows[m * 4 + 0] = kl;
    rows[m * 4 + 1] = (kl_dyn + kl_rep) * fmaxf(kl, free_nats);
    rows[m * 4 + 2] = hp;
    rows[m * 4 + 3] = hq;
  }
  const float live = (kl > free_nats) ? coef : 0.f;
  for (int g = wid; g < groups; g += nw) {
    const float* a = lp0 + (long long)g * K;
    const float* b = lq0 + (long long)g * K;
    float ma = -INFINITY, mb = -INFINITY;
    for (int c = lane; c < K; c += 32) { ma = fmaxf(ma, a[c]); mb = fmaxf(mb, b[c]); }
    ma = warp_max(ma); mb = warp_max(mb);
    float sa = 0.f, sb = 0.f;
    for (int c = lane; c < K; c += 32) { sa += expf(a[c] - ma); sb += expf(b[c] - mb); }
    const float lsea = ma + logf(warp_sum(sa)), lseb = mb + logf(warp_sum(sb));
    float t = 0.f;
    for (int c = lane; c < K; c += 32) {
      const float lpa = a[c] - lsea, lqb = b[c] - lseb;
      t = fmaf(expf(lpa), lpa - lqb, t);
    }
    const float klg = warp_sum(t);
    for (int c = lane; c < K; c += 32) {
      const float lpa = a[c] - lsea, lqb = b[c] - lseb;
      const float pa = expf(lpa), pb = expf(lqb);
      d_prior[m * lddq + (long long)g * K + c] = kl_dyn * live * (pb - pa);
      d_post[m * lddp + (long long)g * K + c] = kl_rep * live * pa * ((lpa - lqb) - klg);
    }
  }
}


// out[m, :] = sum_g WT[g*K + idx(m,g), :] + sum_a act[m,a] * WT[S*K + a, :]   with idx = the hot class of group g.
// z is a concatenation of S one-hot groups (a straight-through categorical sample), so Linear([z, a]) is a gather-sum
// of S+A rows of the transposed weight instead of a K = S*K + A product (agent.py:328-341 RecurrentModel.mlp input).
// One CTA per row; WT [S*K + A, N] row-major (transposed copy of the Linear weight, L2 resident).
// With `gamma`: the row continues through LayerNorm(eps) + SiLU (RecurrentModel.mlp's miniblock) before it is written
// (launched with N / 4 threads, one float4 of the row each); `pre` optionally keeps the Linear output for a backward.
__global__ void __launch_bounds__(256)
onehot_linear_kernel(const float* __restrict__ z, const float* __restrict__ act, const float* __restrict__ WT,
                     float* __restrict__ out, int S, int K, int A, int N, long long ldz, long long lda, long long ldo,
                     const float* __restrict__ gamma, const float* __restrict__ beta, float eps, float* __restrict__ pre,
                     long long ldpre) {
  __shared__ int idx[64];
  __shared__ float av[32];
  __shared__ float red[8];
  const long long m = blockIdx.x;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int g = warp; g < S; g += (int)(blockDim.x >> 5)) {  // hot index of each group by ballot
    int found = 0;
    for (int c0 = 0; c0 < K; c0 += 32) {
      const int c = c0 + lane;
      const unsigned b = __ballot_sync(0xffffffffu, c < K && z[m * ldz + (long long)g * K + c] != 0.f);
      if (b) { found = c0 + __ffs(b) - 1; break; }
    }
    if (lane == 0) idx[g] = found;
  }
  if (threadIdx.x < A) av[threadIdx.x] = act[m * lda + threadIdx.x];
  __syncthreads();
  if (gamma == nullptr) {
    for (int n = threadIdx.x; n < N; n += blockDim.x) {
      float acc = 0.f;
#pragma unroll 8
      for (int g = 0; g < S; ++g) acc += __ldg(WT + ((long long)g * K + idx[g]) * N + n);   // independent L2 loads in flight
      for (int a = 0; a < A; ++a) acc = fmaf(av[a], __ldg(WT + ((long long)S * K + a) * N + n), acc);
      out[m * ldo + n] = acc;
    }
    return;
  }
  // LayerNorm path: one float4 of the row per thread (blockDim.x == N / 4): 128-bit gathers, the row never leaves registers
  const int t = threadIdx.x, nw = (blockDim.x + 31) >> 5;
  const float4* W4 = reinterpret_cast<const float4*>(WT);
  const int n4 = N >> 2;
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 8
  for (int g = 0; g < S; ++g) {
    const float4 w = __ldg(W4 + ((long long)g * K + idx[g]) * n4 + t);
    acc.x += w.x; acc.y += w.y; acc.z += w.z; acc.w += w.w;
  }
  for (int a = 0; a < A; ++a) {
    const float4 w = __ldg(W4 + ((long long)S * K + a) * n4 + t);
    acc.x = fmaf(av[a], w.x, acc.x); acc.y = fmaf(av[a], w.y, acc.y); acc.z = fmaf(av[a], w.z, acc.z); acc.w = fmaf(av[a], w.w, acc.w);
  }
  if (pre) *reinterpret_cast<float4*>(pre + m * ldpre + 4 * t) = acc;
  auto block_sum = [&](float x) {
    x = warp_sum(x);
    __syncthreads();
    if (lane == 0) red[warp] = x;
    __syncthreads();
    float r = 0.f;
    for (int w = 0; w < nw; ++w) r += red[w];
    return r;
  };
  const float mu = block_sum((acc.x + acc.y) + (acc.z + acc.w)) / (float)N;
  const float dx = acc.x - mu, dy = acc.y - mu, dz = acc.z - mu, dw = acc.w - mu;
  const float rstd = rsqrtf(block_sum((dx * dx + dy * dy) + (dz * dz + dw * dw)) / (float)N + eps);
  const float4 gm = reinterpret_cast<const float4*>(gamma)[t], bt = reinterpret_cast<const float4*>(beta)[t];
  float4 y;
  y.x = dx * rstd * gm.x + bt.x; y.y = dy * rstd * gm.y + bt.y; y.z = dz * rstd * gm.z + bt.z; y.w = dw * rstd * gm.w + bt.w;
  y.x = y.x / (1.f + expf(-y.x)); y.y = y.y / (1.f + expf(-y.y)); y.z = y.z / (1.f + expf(-y.z)); y.w = y.w / (1.f + expf(-y.w));
  *reinterpret_cast<float4*>(out + m * ldo + 4 * t) = y;
}

}  // namespace

extern "C" int b200rl_gru_gate_fwd(const float* G, const float* Hin, float* Hout, long long M, int R, long long ldg,
                                   long long ldhi, long long ldho, cudaStream_t st) {
  RL_CHECK_ARG(G && Hin && Hout, "null pointer");
  if (M * R <= 0) return B200RL_OK;
  gru_gate_fwd_kernel<<<ceil_div(M * R, 256), 256, 0, st>>>(G, Hin, Hout, M, R, ldg, ldhi, ldho);
  RL_CHECK_LAUNCH();
  return B200RL_OK;
}

extern "C" int b200rl_gru_gate_bwd(const float* G, const float* Hin, const float* dH, float* dG, float* dHin,
                                   long long M, int R, long long ldg, long long ldhi, long long lddh, long long lddg,
                                   long long lddhi, cudaStream_t st) {
  RL_CHECK_ARG(G && Hin && dH && dG && dHin, "null pointer");
  if (M * R <= 0) return B200RL_OK;
  gru_gate_bwd_kernel<<<ceil_div(M * R, 256), 256, 0, st>>>(G, Hin, dH, dG, dHin, M, R, ldg, ldhi, lddh, lddg, lddhi);
  RL_CHECK_LAUNCH();
  return B200RL_OK;
}

extern "C" int b200rl_mask_mix(const float* prev, const float* init, const float* first, float* out, long long M,
                               int C, long long ldp, long long ldo, cudaStream_t st) {
  RL_CHECK_ARG(prev && first && out, "null pointer");
  if (M * C <= 0) return B200RL_OK;
  mask_mix_kernel<<<ceil_div(M * C, 256), 256, 0, st>>>(prev, init, first, out, M, C, ldp, ldo);
  RL_CHECK_LAUNCH();
  return B200RL_OK;
}

extern "C" int b200rl_mask_bwd(const float* dIn, const float* first, float* dPrev, float* dInit, int M, int C,
                               long long ldi, long long ldp, cudaStream_t st) {
  RL_CHECK_ARG(dIn && first && dPrev, "null pointer");
  if (M <= 0 || C <= 0) return B200RL_OK;
  mask_bwd_kernel<<<ceil_div(C, 128), 128, 0, st>>>(dIn, first, dPrev, dInit, M, C, ldi, ldp);
  RL_CHECK_LAUNCH();
  return B200RL_OK;
}

extern "C" int b200rl_cat_sample(const float* raw, const float* noise, float* onehot, float* mix_out, long long M,
                                 int groups, int K, long long ldr, long long ldn, long long ldo, long long ldm,
                                 float unimix, cudaStream_t st) {
  RL_CHECK_ARG(raw, "null pointer");
  RL_CHECK_ARG(groups > 0 && K > 0, "bad groups / classes");
  if (M <= 0) return B200RL_OK;
  const long long warps = M * groups;
  if (K <= 32)
    cat_sample_small_kernel<<<ceil_div(warps, 8), 256, 0, st>>>(raw, noise, onehot, mix_out, M, groups, K, ldr, ldn, ldo,
                                                                ldm, unimix);
  else
    cat_sample_kernel<<<ceil_div(warps, 8), 256, 0, st>>>(raw, noise, onehot, mix_out, M, groups, K, ldr, ldn, ldo, ldm,
                                                          unimix);
  RL_CHECK_LAUNCH();
  return B200RL_OK;
}

extern "C" int b200rl_head_sample_supported(const float* X, const float* W, int Kin, int A, long long ldx, long long ldw) {
  return A > 0 && A <= 32 && Kin > 0 && Kin <= 1024 && Kin % 4 == 0 && ldx % 4 == 0 && ldw % 4 == 0 &&
         ((reinterpret_cast<uintptr_t>(X) | reinterpret_cast<uintptr_t>(W)) & 15) == 0;
}

extern "C" int b200rl_head_sample(const float* X, const float* W, const float* bias, const float* noise, float* raw,
                                  float* onehot, long long M, int Kin, int A, long long ldx, long long ldw, long long ldr,
                                  long long ldn, long long ldo, float unimix, cudaStream_t st) {
  RL_CHECK_ARG(X && W && raw && onehot, "null pointer");
  RL_CHECK_ARG(b200rl_head_sample_supported(X, W, Kin, A, ldx, ldw),
               "head_sample: A <= 32, Kin <= 1024, 16-byte aligned rows");
  if (M <= 0) return B200RL_OK;
  head_sample_kernel<<<ceil_div(M * 32, 256), 256, 0, st>>>(X, W, bias, noise, raw, onehot, M, Kin, A, ldx, ldw, ldr, ldn, ldo,
                                                            unimix);
  RL_CHECK_LAUNCH();
  return B200RL_OK;
}

extern "C" int b200rl_minedojo_sample_supported(int K0, int K1, int K2) {
  return K0 > 0 && K0 <= 2048 && K1 > 0 && K1 <= 2048 && K2 > 0 && K2 <= 2048;
}

extern "C" int b200rl_minedojo_sample(const float* raw, const float* noise, float* onehot, const float* mask_action_type,
                                      const float* mask_craft_smelt, const float* mask_equip_place,
                                      const float* mask_destroy, long long M, int K0, int K1, int K2, long long ldr,
                                      long long ldn, long long ldo, long long ld_action_type, long long ld_craft_smelt,
                                      long long ld_equip_place, long long ld_destroy, float unimix, cudaStream_t st) {
  RL_CHECK_ARG(raw && onehot, "null pointer");
  RL_CHECK_ARG(b200rl_minedojo_sample_supported(K0, K1, K2), "minedojo_sample: every head has 1 to 2048 classes");
  if (M <= 0) return B200RL_OK;
  minedojo_sample_kernel<<<ceil_div(M * 32, 256), 256, 0, st>>>(
      raw, noise, onehot, mask_action_type, mask_craft_smelt, mask_equip_place, mask_destroy, M, K0, K1, K2, ldr, ldn, ldo,
      ld_action_type, ld_craft_smelt, ld_equip_place, ld_destroy, unimix);
  RL_CHECK_LAUNCH();
  return B200RL_OK;
}

extern "C" int b200rl_cat_sample_bwd(const float* raw, const float* dz, const float* dmix, float* draw, long long M,
                                     int groups, int K, long long ldr, long long lddz, long long lddm,
                                     long long lddr, float unimix, cudaStream_t st) {
  RL_CHECK_ARG(raw && draw, "null pointer");
  RL_CHECK_ARG(groups > 0 && K > 0, "bad groups / classes");
  if (M <= 0) return B200RL_OK;
  const long long warps = M * groups;
  cat_sample_bwd_kernel<<<ceil_div(warps, 8), 256, 0, st>>>(raw, dz, dmix, draw, M, groups, K, ldr, lddz, lddm, lddr,
                                                            unimix);
  RL_CHECK_LAUNCH();
  return B200RL_OK;
}

extern "C" int b200rl_kl_loss_grad(const float* post_mix, const float* prior_mix, float* d_post, float* d_prior,
                                   float* rows, long long M, int groups, int K, long long ldp, long long ldq,
                                   long long lddp, long long lddq, float kl_dyn, float kl_rep, float free_nats,
                                   float regularizer, float scale, cudaStream_t st) {
  RL_CHECK_ARG(post_mix && prior_mix && d_post && d_prior && rows, "null pointer");
  if (M <= 0) return B200RL_OK;
  kl_loss_grad_kernel<<<(unsigned)M, 256, 0, st>>>(post_mix, prior_mix, d_post, d_prior, rows, groups, K, ldp, ldq,
                                                   lddp, lddq, kl_dyn, kl_rep, free_nats, scale * regularizer);
  RL_CHECK_LAUNCH();
  return B200RL_OK;
}

extern "C" int b200rl_onehot_linear_supported(int S, int K, int A, int N) {
  return S > 0 && S <= 64 && K > 0 && A >= 0 && A <= 32 && N > 0;
}

extern "C" int b200rl_onehot_linear_ln_supported(const float* WT, const float* gamma, const float* beta, const float* out,
                                                 const float* pre, int N, long long ldo, long long ldpre) {
  return N >= 128 && N <= 1024 && N % 128 == 0 && ldo % 4 == 0 && ldpre % 4 == 0 &&
         ((reinterpret_cast<uintptr_t>(WT) | reinterpret_cast<uintptr_t>(gamma) | reinterpret_cast<uintptr_t>(beta) |
           reinterpret_cast<uintptr_t>(out) | reinterpret_cast<uintptr_t>(pre)) & 15) == 0;
}

extern "C" int b200rl_onehot_linear(const float* z, const float* act, const float* WT, float* out, long long M, int S,
                                    int K, int A, int N, long long ldz, long long lda, long long ldo, cudaStream_t st) {
  RL_CHECK_ARG(z && (act || A == 0) && WT && out, "null pointer");   // act is read only for A > 0 action columns
  RL_CHECK_ARG(b200rl_onehot_linear_supported(S, K, A, N), "bad dims (S <= 64 groups, A <= 32)");
  if (M <= 0) return B200RL_OK;
  onehot_linear_kernel<<<(unsigned)M, 256, 0, st>>>(z, act, WT, out, S, K, A, N, ldz, lda, ldo, nullptr, nullptr, 0.f, nullptr, 0);
  RL_CHECK_LAUNCH();
  return B200RL_OK;
}

extern "C" int b200rl_onehot_linear_ln(const float* z, const float* act, const float* WT, const float* gamma,
                                       const float* beta, float eps, float* pre, long long ldpre, float* out, long long M,
                                       int S, int K, int A, int N, long long ldz, long long lda, long long ldo,
                                       cudaStream_t st) {
  RL_CHECK_ARG(z && (act || A == 0) && WT && out && gamma && beta, "null pointer");
  RL_CHECK_ARG(b200rl_onehot_linear_supported(S, K, A, N), "bad dims (S <= 64 groups, A <= 32)");
  RL_CHECK_ARG(b200rl_onehot_linear_ln_supported(WT, gamma, beta, out, pre, N, ldo, ldpre),
               "onehot_linear_ln: N a multiple of 128 up to 1024, 16-byte aligned rows");
  if (M <= 0) return B200RL_OK;
  onehot_linear_kernel<<<(unsigned)M, N / 4, 0, st>>>(z, act, WT, out, S, K, A, N, ldz, lda, ldo, gamma, beta, eps, pre, ldpre);
  RL_CHECK_LAUNCH();
  return B200RL_OK;
}
