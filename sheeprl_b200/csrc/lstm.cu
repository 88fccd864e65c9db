// Single-layer LSTM over padded sequences, forward and backward-through-time, each in ONE launch.
//
// Replaces (reference): RecurrentModel.forward's pack_padded_sequence -> nn.LSTM -> pad_packed_sequence
// (sheeprl/algos/ppo_recurrent/agent.py:67-80; cuDNN LSTM on a GPU) and its autograd backward.
//
// torch semantics: gates in the order i, f, g, o; c' = f*c + i*g; h' = o*tanh(c').  The input projection
// xw = x W_ih^T + b_ih + b_hh of all T*B rows is one dense product done beforehand (csrc/mlp.cu), and the weight /
// bias / input gradients are dense products over d_gates afterwards; what is left here is the recurrence.
//
// Layout: time-major, row (t, b) of every [T, B, *] tensor is at (t*B + b).  Sequence b is valid for steps
// t < lengths[b] (a prefix, lengths in [1, T]); at padded steps `out` is 0 (what pad_packed_sequence returns) and the
// state does not advance, so (hT, cT) is the state after step lengths[b]-1.
//
// Sequences are independent, so each CTA owns SB of them and keeps their h / c (forward) or dh / dc (backward) in
// shared memory for all T steps: no cross-CTA hand-off and no atomics.  The recurrent product h W_hh^T is a plain
// fp32 FMA loop in a fixed order (at H = 64 it is 64 KB of weights per step, latency-bound), so results are
// bit-reproducible run to run.  W_hh is read through L1 / L2 every step, which works for every hidden size.
#include "common.cuh"

namespace {

constexpr int kLstmThreads = 256;

__device__ __forceinline__ float lstm_act(int j, int H, float x) {
  return (j >= 2 * H && j < 3 * H) ? tanhf(x) : sigmoidf_(x);       // g uses tanh, i / f / o the sigmoid
}

template <int SB>
__global__ void __launch_bounds__(kLstmThreads) lstm_seq_fwd_kernel(
    const float* __restrict__ xw, const float* __restrict__ W, const float* __restrict__ h0,
    const float* __restrict__ c0, const int* __restrict__ lengths, float* __restrict__ out,
    float* __restrict__ gates, float* __restrict__ cs, float* __restrict__ hT, float* __restrict__ cT, int T, int B,
    int H) {
  extern __shared__ float sm[];
  float* h_s = sm;                       // [SB][H]
  float* c_s = h_s + SB * H;             // [SB][H]
  float* g_s = c_s + SB * H;             // [SB][4H] activated gates of the current step
  const int b0 = blockIdx.x * SB;
  const int G = 4 * H;
  int len[SB];
#pragma unroll
  for (int s = 0; s < SB; ++s) len[s] = (b0 + s < B) ? lengths[b0 + s] : 0;
  for (int e = threadIdx.x; e < SB * H; e += blockDim.x) {
    const int s = e / H, i = e - s * H, b = b0 + s;
    h_s[e] = (b < B) ? h0[(long long)b * H + i] : 0.f;
    c_s[e] = (b < B) ? c0[(long long)b * H + i] : 0.f;
  }
  __syncthreads();
  for (int t = 0; t < T; ++t) {
    // ---- gates = act(xw[t] + h W_hh^T): one gate row per thread, SB sequences per weight read
    for (int j = threadIdx.x; j < G; j += blockDim.x) {
      float acc[SB];
#pragma unroll
      for (int s = 0; s < SB; ++s) acc[s] = (t < len[s]) ? xw[((long long)t * B + b0 + s) * G + j] : 0.f;
      const float* w = W + (long long)j * H;
#pragma unroll 4
      for (int k = 0; k < H; ++k) {
        const float wk = __ldg(w + k);
#pragma unroll
        for (int s = 0; s < SB; ++s) acc[s] = fmaf(wk, h_s[s * H + k], acc[s]);
      }
#pragma unroll
      for (int s = 0; s < SB; ++s) g_s[s * G + j] = lstm_act(j, H, acc[s]);
    }
    __syncthreads();
    // ---- cell update for the valid sequences; padded steps write zeros and keep the state
    for (int e = threadIdx.x; e < SB * H; e += blockDim.x) {
      const int s = e / H, i = e - s * H, b = b0 + s;
      if (b >= B) continue;
      const long long row = (long long)t * B + b;
      const float* g = g_s + s * G;
      if (t < len[s]) {
        const float c = g[H + i] * c_s[e] + g[i] * g[2 * H + i];
        const float h = g[3 * H + i] * tanhf(c);
        c_s[e] = c;
        h_s[e] = h;
        out[row * H + i] = h;
        if (cs) cs[row * H + i] = c;
        if (gates) {
#pragma unroll
          for (int q = 0; q < 4; ++q) gates[row * G + q * H + i] = g[q * H + i];
        }
      } else {
        out[row * H + i] = 0.f;
        if (cs) cs[row * H + i] = 0.f;
        if (gates) {
#pragma unroll
          for (int q = 0; q < 4; ++q) gates[row * G + q * H + i] = 0.f;
        }
      }
    }
    __syncthreads();
  }
  for (int e = threadIdx.x; e < SB * H; e += blockDim.x) {
    const int s = e / H, i = e - s * H, b = b0 + s;
    if (b >= B) continue;
    if (hT) hT[(long long)b * H + i] = h_s[e];
    if (cT) cT[(long long)b * H + i] = c_s[e];
  }
}

// d_gates[t] = d(loss)/d(pre-activation gates at t); the state gradient dh_{t-1} = d_gates[t] W_hh and
// dc_{t-1} = dc_t * f_t are carried on chip.  h0 / c0 get no gradient (they come from the rollout data).
template <int SB>
__global__ void __launch_bounds__(kLstmThreads) lstm_seq_bwd_kernel(
    const float* __restrict__ d_out, const float* __restrict__ W, const float* __restrict__ gates,
    const float* __restrict__ cs, const float* __restrict__ c0, const int* __restrict__ lengths,
    float* __restrict__ d_gates, int T, int B, int H) {
  extern __shared__ float sm[];
  float* dh_s = sm;                      // [SB][H] carried dh from step t+1
  float* dc_s = dh_s + SB * H;           // [SB][H] carried dc from step t+1
  float* dg_s = dc_s + SB * H;           // [SB][4H]
  const int b0 = blockIdx.x * SB;
  const int G = 4 * H;
  int len[SB];
#pragma unroll
  for (int s = 0; s < SB; ++s) len[s] = (b0 + s < B) ? lengths[b0 + s] : 0;
  for (int e = threadIdx.x; e < SB * H; e += blockDim.x) dh_s[e] = dc_s[e] = 0.f;
  __syncthreads();
  for (int t = T - 1; t >= 0; --t) {
    for (int e = threadIdx.x; e < SB * H; e += blockDim.x) {
      const int s = e / H, i = e - s * H, b = b0 + s;
      float* dg = dg_s + s * G;
      if (b < B && t < len[s]) {
        const long long row = (long long)t * B + b;
        const float* g = gates + row * G;
        const float ig = g[i], fg = g[H + i], gg = g[2 * H + i], og = g[3 * H + i];
        const float c = cs[row * H + i];
        const float cp = (t > 0) ? cs[(row - B) * H + i] : c0[(long long)b * H + i];
        const float tc = tanhf(c);
        const float dh = d_out[row * H + i] + dh_s[e];
        const float dc = dc_s[e] + dh * og * (1.f - tc * tc);
        dg[i] = dc * gg * ig * (1.f - ig);
        dg[H + i] = dc * cp * fg * (1.f - fg);
        dg[2 * H + i] = dc * ig * (1.f - gg * gg);
        dg[3 * H + i] = dh * tc * og * (1.f - og);
        dc_s[e] = dc * fg;
      } else {
        dg[i] = dg[H + i] = dg[2 * H + i] = dg[3 * H + i] = 0.f;
      }
      if (b < B) {
        const long long row = (long long)t * B + b;
#pragma unroll
        for (int q = 0; q < 4; ++q) d_gates[row * G + q * H + i] = dg[q * H + i];
      }
    }
    __syncthreads();
    if (t > 0) {
      // dh_{t-1}[k] = sum_j d_gates[t][j] W_hh[j][k]: one column k per thread (coalesced rows of W_hh)
      for (int k = threadIdx.x; k < H; k += blockDim.x) {
        float acc[SB];
#pragma unroll
        for (int s = 0; s < SB; ++s) acc[s] = 0.f;
#pragma unroll 4
        for (int j = 0; j < G; ++j) {
          const float wjk = __ldg(W + (long long)j * H + k);
#pragma unroll
          for (int s = 0; s < SB; ++s) acc[s] = fmaf(dg_s[s * G + j], wjk, acc[s]);
        }
#pragma unroll
        for (int s = 0; s < SB; ++s) dh_s[s * H + k] = acc[s];
      }
    }
    __syncthreads();
  }
}

// Sequences per CTA: as many as keep >= one wave of CTAs on the SMs, at most 8, and within 160 KB of shared memory.
int pick_sb(int B, int H) {
  int sb = 1;
  while (sb < 8 && (long long)B > (long long)kNumSMs * sb * 2 && (long long)(2 * sb) * 6 * H * 4 <= 160 * 1024) sb *= 2;
  return sb;
}

template <typename K>
int launch_cfg(K kernel, size_t smem) {
  if (smem > 48 * 1024) RL_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  return B200RL_OK;
}

}  // namespace

extern "C" int b200rl_lstm_seq_fwd(const float* xw, const float* W_hh, const float* h0, const float* c0,
                                   const int* lengths, float* out, float* gates, float* cs, float* hT, float* cT, int T,
                                   int B, int H, cudaStream_t st) {
  RL_CHECK_ARG(xw && W_hh && h0 && c0 && lengths && out, "null pointer");
  RL_CHECK_ARG(T > 0 && B > 0 && H > 0, "bad dims");
  RL_CHECK_ARG((gates == nullptr) == (cs == nullptr), "gates and cs are saved together (both or neither)");
  const int sb = pick_sb(B, H);
  const size_t smem = (size_t)sb * 6 * H * sizeof(float);
  RL_CHECK_ARG(smem <= 227 * 1024, "hidden size too large for the on-chip state");
  const int grid = ceil_div(B, sb);
#define RL_LSTM_FWD(SB_)                                                                                   \
  case SB_: {                                                                                             \
    int rc = launch_cfg(lstm_seq_fwd_kernel<SB_>, smem);                                                  \
    if (rc) return rc;                                                                                    \
    lstm_seq_fwd_kernel<SB_><<<grid, kLstmThreads, smem, st>>>(xw, W_hh, h0, c0, lengths, out, gates, cs, hT, cT, T, \
                                                               B, H);                                    \
    break;                                                                                                \
  }
  switch (sb) { RL_LSTM_FWD(1) RL_LSTM_FWD(2) RL_LSTM_FWD(4) RL_LSTM_FWD(8) default: break; }
#undef RL_LSTM_FWD
  RL_CHECK_LAUNCH();
  return B200RL_OK;
}

extern "C" int b200rl_lstm_seq_bwd(const float* d_out, const float* W_hh, const float* gates, const float* cs,
                                   const float* c0, const int* lengths, float* d_gates, int T, int B, int H,
                                   cudaStream_t st) {
  RL_CHECK_ARG(d_out && W_hh && gates && cs && c0 && lengths && d_gates, "null pointer");
  RL_CHECK_ARG(T > 0 && B > 0 && H > 0, "bad dims");
  const int sb = pick_sb(B, H);
  const size_t smem = (size_t)sb * 6 * H * sizeof(float);
  RL_CHECK_ARG(smem <= 227 * 1024, "hidden size too large for the on-chip state");
  const int grid = ceil_div(B, sb);
#define RL_LSTM_BWD(SB_)                                                                                   \
  case SB_: {                                                                                             \
    int rc = launch_cfg(lstm_seq_bwd_kernel<SB_>, smem);                                                  \
    if (rc) return rc;                                                                                    \
    lstm_seq_bwd_kernel<SB_><<<grid, kLstmThreads, smem, st>>>(d_out, W_hh, gates, cs, c0, lengths, d_gates, T, B, H); \
    break;                                                                                                \
  }
  switch (sb) { RL_LSTM_BWD(1) RL_LSTM_BWD(2) RL_LSTM_BWD(4) RL_LSTM_BWD(8) default: break; }
#undef RL_LSTM_BWD
  RL_CHECK_LAUNCH();
  return B200RL_OK;
}
