// DroQ critics: the miniblock `Dropout -> LayerNorm -> ReLU` that follows each hidden Linear, for all n critics of a
// batched stack in one launch, and the dropout keep masks of a whole train() call in one launch.
//
// Replaces (reference): DROQCritic sheeprl/algos/droq/agent.py:19-47 (MLP of miniblocks, sheeprl/utils/model.py:34-88:
// layer -> nn.Dropout(p) -> nn.LayerNorm(H, eps) -> nn.ReLU) in train mode, forward and autograd backward.  Torch's
// dropout is x * mask * (1/(1-p)) with mask ~ Bernoulli(1-p); here the mask is bit-packed, one 32-bit word per 32
// columns of a row, so a [n, B, H] activation's mask is [n, B, ceil(H/32)] words; bits past column H are padding and
// never read.  Row layouts [n, B, H] are contiguous; gamma / beta (and dgamma / dbeta) of critic i sit at
// i * stride_param, the constant inter-critic stride of the flat parameter group.
#include "common.cuh"

namespace {

constexpr int kMaxCols = 1024;   // 32 columns per lane: the widest row the kernels hold in registers

__device__ __forceinline__ bool keep_bit(const uint32_t* __restrict__ mrow, int k, int lane) {
  return (mrow[k] >> lane) & 1u;
}

// keep bit i of the fill = (Philox word >= thr): P(keep) = 1 - thr / 2^32.  Word w takes Philox counters 8w .. 8w+7.
__global__ void dropout_mask_kernel(uint32_t* __restrict__ mask, long long n_words, uint32_t thr, uint32_t seed_lo,
                                    uint32_t seed_hi, uint32_t stream, const int* __restrict__ counter) {
  const uint32_t ctr = counter ? (uint32_t)(*counter) : 0u;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long w = (long long)blockIdx.x * blockDim.x + threadIdx.x; w < n_words; w += stride) {
    uint32_t bits = 0u;
#pragma unroll 1
    for (int q = 0; q < 8; ++q) {
      const long long i = w * 8 + q;
      uint32_t c[4] = {(uint32_t)i, (uint32_t)(i >> 32), stream, ctr};
      uint32_t k0 = seed_lo, k1 = seed_hi;
#pragma unroll
      for (int r = 0; r < 10; ++r) {
        philox_round(c, k0, k1);
        k0 += 0x9E3779B9u;
        k1 += 0xBB67AE85u;
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) bits |= (c[j] >= thr ? 1u : 0u) << (q * 4 + j);
    }
    mask[w] = bits;
  }
}

// One warp per row; lane l holds columns l + 32k, k < CPL (CPL = ceil(H/32) rounded up to a power of two), so the mask
// word of column l + 32k is word k of the row.  y = relu(LN(x) * gamma + beta), x = z * keep / (1-p); stats = (mean, rstd).
template <int CPL>
__global__ void __launch_bounds__(256)
dln_fwd_kernel(const float* __restrict__ z, const uint32_t* __restrict__ mask, float scale,
               const float* __restrict__ gamma, const float* __restrict__ beta, long long sp, float eps,
               float* __restrict__ y, float* __restrict__ stats, int B, int H) {
  const int lane = threadIdx.x & 31, net = blockIdx.y;
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= B) return;
  const long long r = (long long)net * B + row;
  const float* zr = z + r * H;
  const uint32_t* mr = mask ? mask + r * ((H + 31) >> 5) : nullptr;
  const float* g = gamma + net * sp;
  const float* bt = beta + net * sp;
  float x[CPL];
  float s = 0.f;
#pragma unroll
  for (int k = 0; k < CPL; ++k) {
    const int c = lane + 32 * k;
    float v = 0.f;
    if (c < H) {
      v = zr[c];
      if (mr) v = keep_bit(mr, k, lane) ? v * scale : 0.f;
    }
    x[k] = v;
    s += v;
  }
  const float mean = warp_sum(s) / (float)H;
  float s2 = 0.f;
#pragma unroll
  for (int k = 0; k < CPL; ++k) {
    const float d = x[k] - mean;
    if (lane + 32 * k < H) s2 += d * d;
  }
  const float rstd = 1.f / sqrtf(warp_sum(s2) / (float)H + eps);
  float* yr = y + r * H;
#pragma unroll
  for (int k = 0; k < CPL; ++k) {
    const int c = lane + 32 * k;
    if (c < H) yr[c] = fmaxf((x[k] - mean) * rstd * g[c] + bt[c], 0.f);
  }
  if (lane == 0) {
    stats[2 * r] = mean;
    stats[2 * r + 1] = rstd;
  }
}

// dReLU (y > 0), LayerNorm backward (xhat recomputed from z, the mask and the saved stats), then the mask scale:
// dz = keep/(1-p) * rstd * (dxhat - mean(dxhat) - xhat * mean(dxhat * xhat)), dxhat = gamma * dy * [y > 0].
// With dgamma (and dbeta) the grid is one CTA per critic: warp w takes rows w, w + WARPS, ... and keeps per-lane column
// partials of sum(g * xhat) and sum(g); the warps then add theirs in warp order, so both are bit-identical run to run.
template <int CPL, int WARPS>
__global__ void __launch_bounds__(WARPS * 32)
dln_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ y, const float* __restrict__ z,
               const uint32_t* __restrict__ mask, float scale, const float* __restrict__ stats,
               const float* __restrict__ gamma, long long sp, float* __restrict__ dz, float* __restrict__ dgamma,
               float* __restrict__ dbeta, int B, int H) {
  __shared__ float acc[2][kMaxCols];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, net = blockIdx.y;
  const int W = (H + 31) >> 5;
  const float* gm = gamma + net * sp;
  const float invH = 1.f / (float)H;
  float ag[CPL], ab[CPL];
#pragma unroll
  for (int k = 0; k < CPL; ++k) ag[k] = ab[k] = 0.f;
  for (int row = blockIdx.x * WARPS + warp; row < B; row += gridDim.x * WARPS) {
    const long long r = (long long)net * B + row;
    const float mean = stats[2 * r], rstd = stats[2 * r + 1];
    const uint32_t* mr = mask ? mask + r * W : nullptr;
    float g[CPL], xh[CPL];
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int k = 0; k < CPL; ++k) {
      const int c = lane + 32 * k;
      g[k] = xh[k] = 0.f;
      if (c < H) {
        float x = z[r * H + c];
        if (mr) x = keep_bit(mr, k, lane) ? x * scale : 0.f;
        xh[k] = (x - mean) * rstd;
        g[k] = y[r * H + c] > 0.f ? dy[r * H + c] : 0.f;
        const float dxh = g[k] * gm[c];
        s1 += dxh;
        s2 += dxh * xh[k];
        ag[k] += g[k] * xh[k];
        ab[k] += g[k];
      }
    }
    s1 = warp_sum(s1) * invH;
    s2 = warp_sum(s2) * invH;
#pragma unroll
    for (int k = 0; k < CPL; ++k) {
      const int c = lane + 32 * k;
      if (c < H) {
        float d = rstd * (g[k] * gm[c] - s1 - xh[k] * s2);
        if (mr) d = keep_bit(mr, k, lane) ? d * scale : 0.f;
        dz[r * H + c] = d;
      }
    }
  }
  if (dgamma == nullptr) return;                     // uniform over the CTA: no barrier is skipped by some threads only
  for (int w = 0; w < WARPS; ++w) {
    if (warp == w) {
#pragma unroll
      for (int k = 0; k < CPL; ++k) {
        const int c = lane + 32 * k;
        if (c < H) {
          acc[0][c] = (w == 0 ? 0.f : acc[0][c]) + ag[k];
          acc[1][c] = (w == 0 ? 0.f : acc[1][c]) + ab[k];
        }
      }
    }
    __syncthreads();
  }
  for (int c = threadIdx.x; c < H; c += blockDim.x) {
    dgamma[net * sp + c] = acc[0][c];
    dbeta[net * sp + c] = acc[1][c];
  }
}

template <int CPL>
void dln_fwd_launch(const float* z, const uint32_t* mask, float scale, const float* gamma, const float* beta,
                    long long sp, float eps, float* y, float* stats, int nets, int B, int H, cudaStream_t st) {
  dln_fwd_kernel<CPL><<<dim3(ceil_div(B, 8), nets), 256, 0, st>>>(z, mask, scale, gamma, beta, sp, eps, y, stats, B, H);
}

template <int CPL, int WARPS>
void dln_bwd_launch(const float* dy, const float* y, const float* z, const uint32_t* mask, float scale,
                    const float* stats, const float* gamma, long long sp, float* dz, float* dgamma, float* dbeta,
                    int nets, int B, int H, cudaStream_t st) {
  const int ctas = dgamma ? 1 : ceil_div(B, WARPS);
  dln_bwd_kernel<CPL, WARPS><<<dim3(ctas, nets), WARPS * 32, 0, st>>>(dy, y, z, mask, scale, stats, gamma, sp, dz,
                                                                      dgamma, dbeta, B, H);
}

// columns per lane: the smallest power of two >= ceil(H / 32)
int cols_per_lane(int H) {
  int c = 1;
  while (32 * c < H) c <<= 1;
  return c;
}

}  // namespace

extern "C" int b200rl_dropout_mask(unsigned int* mask, long long n_words, float p, unsigned long long seed,
                                   unsigned int stream_id, const int* counter_dev, cudaStream_t st) {
  RL_CHECK_ARG(mask, "null pointer");
  RL_CHECK_ARG(n_words > 0, "bad dims");
  RL_CHECK_ARG(p >= 0.f && p < 1.f, "dropout probability outside [0, 1)");
  const double t = (double)p * 4294967296.0;
  const uint32_t thr = t >= 4294967295.0 ? 0xFFFFFFFFu : (uint32_t)llrint(t);
  const long long grid = n_words < 256LL * 4 * kNumSMs ? (n_words + 255) / 256 : 4LL * kNumSMs;
  dropout_mask_kernel<<<(int)grid, 256, 0, st>>>(mask, n_words, thr, (uint32_t)seed, (uint32_t)(seed >> 32), stream_id,
                                                 counter_dev);
  RL_CHECK_LAUNCH();
  return B200RL_OK;
}

extern "C" int b200rl_dropout_ln_relu_supported(int H) { return H >= 1 && H <= kMaxCols; }

extern "C" int b200rl_dropout_ln_relu_fwd(const float* z, const unsigned int* mask, float p, const float* gamma,
                                          const float* beta, long long stride_param, float eps, float* y, float* stats,
                                          int nets, int B, int H, cudaStream_t st) {
  RL_CHECK_ARG(z && gamma && beta && y && stats, "null pointer");
  RL_CHECK_ARG(nets > 0 && B > 0 && b200rl_dropout_ln_relu_supported(H), "bad dims (1 <= H <= 1024)");
  RL_CHECK_ARG(p >= 0.f && p < 1.f && ((p > 0.f) == (mask != nullptr)), "a mask is passed iff 0 < p < 1");
  const float scale = p > 0.f ? 1.f / (1.f - p) : 1.f;
  switch (cols_per_lane(H)) {
    case 1: dln_fwd_launch<1>(z, mask, scale, gamma, beta, stride_param, eps, y, stats, nets, B, H, st); break;
    case 2: dln_fwd_launch<2>(z, mask, scale, gamma, beta, stride_param, eps, y, stats, nets, B, H, st); break;
    case 4: dln_fwd_launch<4>(z, mask, scale, gamma, beta, stride_param, eps, y, stats, nets, B, H, st); break;
    case 8: dln_fwd_launch<8>(z, mask, scale, gamma, beta, stride_param, eps, y, stats, nets, B, H, st); break;
    case 16: dln_fwd_launch<16>(z, mask, scale, gamma, beta, stride_param, eps, y, stats, nets, B, H, st); break;
    default: dln_fwd_launch<32>(z, mask, scale, gamma, beta, stride_param, eps, y, stats, nets, B, H, st); break;
  }
  RL_CHECK_LAUNCH();
  return B200RL_OK;
}

extern "C" int b200rl_dropout_ln_relu_bwd(const float* dy, const float* y, const float* z, const unsigned int* mask,
                                          float p, const float* stats, const float* gamma, long long stride_param,
                                          float* dz, float* dgamma, float* dbeta, int nets, int B, int H,
                                          cudaStream_t st) {
  RL_CHECK_ARG(dy && y && z && stats && gamma && dz, "null pointer");
  RL_CHECK_ARG((dgamma == nullptr) == (dbeta == nullptr), "dgamma and dbeta are both given or both NULL");
  RL_CHECK_ARG(nets > 0 && B > 0 && b200rl_dropout_ln_relu_supported(H), "bad dims (1 <= H <= 1024)");
  RL_CHECK_ARG(p >= 0.f && p < 1.f && ((p > 0.f) == (mask != nullptr)), "a mask is passed iff 0 < p < 1");
  const float scale = p > 0.f ? 1.f / (1.f - p) : 1.f;
  // one CTA per critic reduces dgamma / dbeta: as many warps as the per-lane partials leave registers for
#define DLN_BWD(CPL, WARPS) \
  dln_bwd_launch<CPL, WARPS>(dy, y, z, mask, scale, stats, gamma, stride_param, dz, dgamma, dbeta, nets, B, H, st)
  switch (cols_per_lane(H)) {
    case 1: if (dgamma) DLN_BWD(1, 32); else DLN_BWD(1, 8); break;
    case 2: if (dgamma) DLN_BWD(2, 32); else DLN_BWD(2, 8); break;
    case 4: if (dgamma) DLN_BWD(4, 32); else DLN_BWD(4, 8); break;
    case 8: if (dgamma) DLN_BWD(8, 32); else DLN_BWD(8, 8); break;
    case 16: if (dgamma) DLN_BWD(16, 16); else DLN_BWD(16, 8); break;
    default: DLN_BWD(32, 8); break;
  }
#undef DLN_BWD
  RL_CHECK_LAUNCH();
  return B200RL_OK;
}
