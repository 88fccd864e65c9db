// LayerNorm(+SiLU) forward / backward and column sums (HBM-bound row kernels).
//
// Replaces: nn.LayerNorm(eps=1e-3) + nn.SiLU blocks built by `miniblock` (sheeprl/utils/model.py:34-88),
// `LayerNormChannelLast` (sheeprl/models/models.py:507-518; channel-last is the native layout here so no
// permute copies are needed) and their autograd backward; bias gradients (column sums).
// One warp per row: lanes stride over the C contiguous channels, statistics via warp shuffles.
#include "common.cuh"

namespace {

constexpr int ACT_NONE = 0, ACT_SILU = 1, ACT_TANH = 2, ACT_RELU = 3;   // (2, 3: the PPO MLPs with layer_norm=True)

__device__ __forceinline__ float act_fwd(int act, float o) {
  if (act == ACT_SILU) return siluf_(o);
  if (act == ACT_TANH) return tanhf(o);
  if (act == ACT_RELU) return fmaxf(o, 0.f);
  return o;
}
// dy * act'(ln)
__device__ __forceinline__ float act_bwd(int act, float ln, float dy) {
  if (act == ACT_SILU) {
    const float sg = sigmoidf_(ln);
    return dy * sg * (1.f + ln * (1.f - sg));
  }
  if (act == ACT_TANH) {
    const float t = tanhf(ln);
    return dy * (1.f - t * t);
  }
  if (act == ACT_RELU) return ln > 0.f ? dy : 0.f;
  return dy;
}

__global__ void __launch_bounds__(256)
ln_act_fwd_kernel(const float* __restrict__ X, const float* __restrict__ gamma, const float* __restrict__ beta,
                  float* __restrict__ Y, long long M, int C, long long ldx, long long ldy, float eps, int act) {
  const int lane = threadIdx.x & 31;
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  const float invC = 1.f / (float)C;
  for (long long r = warp; r < M; r += nwarps) {
    const float* x = X + r * ldx;
    float s = 0.f;
    for (int c = lane; c < C; c += 32) s += x[c];
    const float mu = warp_sum(s) * invC;
    float v = 0.f;
    for (int c = lane; c < C; c += 32) { const float d = x[c] - mu; v = fmaf(d, d, v); }
    const float rstd = rsqrtf(warp_sum(v) * invC + eps);
    float* y = Y + r * ldy;
    for (int c = lane; c < C; c += 32) {
      y[c] = act_fwd(act, (x[c] - mu) * rstd * gamma[c] + beta[c]);
    }
  }
}

// CPL = channels per lane held in registers for the dgamma/dbeta partial sums (C <= 32*CPL).
// DET: dgamma / dbeta are slot arrays with a row stride of 2*C floats, one slot per warp; each warp writes
// its own partials there (CPL == 0: accumulates them there, row by row) in place of the shared and global atomics.
template <int CPL, bool DET>
__global__ void __launch_bounds__(256)
ln_act_bwd_kernel(const float* __restrict__ X, const float* __restrict__ gamma, const float* __restrict__ beta,
                  const float* dY, float* dX, float* __restrict__ dgamma, float* __restrict__ dbeta,
                  long long M, int C, long long ldx, long long lddy, long long lddx, float eps, int act) {
  extern __shared__ float sacc[];  // CPL == 0: [2*C] shared accumulators
  const int lane = threadIdx.x & 31;
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  const float invC = 1.f / (float)C;
  constexpr int NACC = CPL > 0 ? CPL : 1;
  float ag[NACC], ab[NACC];
#pragma unroll
  for (int j = 0; j < NACC; ++j) { ag[j] = 0.f; ab[j] = 0.f; }
  const bool want_param = dgamma != nullptr;
  if (CPL == 0 && want_param) {
    if constexpr (DET) {
      for (int c = lane; c < C; c += 32) { dgamma[warp * 2 * C + c] = 0.f; dbeta[warp * 2 * C + c] = 0.f; }
    } else {
      for (int c = threadIdx.x; c < 2 * C; c += blockDim.x) sacc[c] = 0.f;
      __syncthreads();
    }
  }
  for (long long r = warp; r < M; r += nwarps) {
    const float* x = X + r * ldx;
    const float* dy = dY + r * lddy;
    float s = 0.f;
    for (int c = lane; c < C; c += 32) s += x[c];
    const float mu = warp_sum(s) * invC;
    float v = 0.f;
    for (int c = lane; c < C; c += 32) { const float d = x[c] - mu; v = fmaf(d, d, v); }
    const float rstd = rsqrtf(warp_sum(v) * invC + eps);
    float s1 = 0.f, s2 = 0.f;
    auto body = [&](int c, float& accg, float& accb) {
      const float xh = (x[c] - mu) * rstd;
      const float dln = (act == ACT_NONE) ? dy[c] : act_bwd(act, xh * gamma[c] + beta[c], dy[c]);
      const float dxh = dln * gamma[c];
      s1 += dxh;
      s2 = fmaf(dxh, xh, s2);
      accg = dln * xh;
      accb = dln;
    };
    if constexpr (CPL > 0) {
#pragma unroll
      for (int j = 0; j < NACC; ++j) {
        const int c = lane + 32 * j;
        if (c < C) {
          float g_, b_;
          body(c, g_, b_);
          ag[j] += g_;
          ab[j] += b_;
        }
      }
    } else {
      for (int c = lane; c < C; c += 32) {
        float g_, b_;
        body(c, g_, b_);
        if (want_param) {
          if constexpr (DET) { dgamma[warp * 2 * C + c] += g_; dbeta[warp * 2 * C + c] += b_; }
          else { atomicAdd(&sacc[c], g_); atomicAdd(&sacc[C + c], b_); }
        }
      }
    }
    s1 = warp_sum(s1) * invC;
    s2 = warp_sum(s2) * invC;
    float* dx = dX + r * lddx;
    for (int c = lane; c < C; c += 32) {
      const float xh = (x[c] - mu) * rstd;
      const float dln = (act == ACT_NONE) ? dy[c] : act_bwd(act, xh * gamma[c] + beta[c], dy[c]);
      dx[c] = rstd * (dln * gamma[c] - s1 - xh * s2);  // dX may alias dY: element c is read before it is written
    }
  }
  if (want_param) {
    if (CPL > 0) {
#pragma unroll
      for (int j = 0; j < NACC; ++j) {
        const int c = lane + 32 * j;
        if (c < C) {
          if constexpr (DET) { dgamma[warp * 2 * C + c] = ag[j]; dbeta[warp * 2 * C + c] = ab[j]; }
          else { atomicAdd(&dgamma[c], ag[j]); atomicAdd(&dbeta[c], ab[j]); }
        }
      }
    } else if constexpr (!DET) {
      __syncthreads();
      for (int c = threadIdx.x; c < C; c += blockDim.x) {
        atomicAdd(&dgamma[c], sacc[c]);
        atomicAdd(&dbeta[c], sacc[C + c]);
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------
// Wide rows (C > 1536, e.g. the XL GRU's joint LayerNorm over 3 x 4096 channels): one CTA of 512 threads per row at a
// time, the row held in registers (up to WNV float4 per thread), block-wide statistics.  The warp-per-row kernels above
// need many rows to fill the machine; the XL per-step scan has 64 rows of 12 288 floats (268 us -> HBM/latency bound).
// ---------------------------------------------------------------------------------------------------------
constexpr int WIDE_NT = 512, WNV = 8;   // C <= 4 * WIDE_NT * WNV = 16384

__device__ __forceinline__ float block_sum512(float v, float* red) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  v = warp_sum(v);
  __syncthreads();
  if (lane == 0) red[wid] = v;
  __syncthreads();
  float r = (lane < WIDE_NT / 32) ? red[lane] : 0.f;
  return warp_sum(r);
}

__global__ void __launch_bounds__(WIDE_NT)
ln_act_fwd_wide_kernel(const float* __restrict__ X, const float* __restrict__ gamma, const float* __restrict__ beta,
                       float* __restrict__ Y, long long M, int C, long long ldx, long long ldy, float eps, int act) {
  __shared__ float red[32];
  const int n4 = C >> 2;
  const float invC = 1.f / (float)C;
  for (long long r = blockIdx.x; r < M; r += gridDim.x) {
    const float4* x4 = reinterpret_cast<const float4*>(X + r * ldx);
    float4 v[WNV];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < WNV; ++i) {
      const int c = threadIdx.x + i * WIDE_NT;
      v[i] = (c < n4) ? x4[c] : make_float4(0.f, 0.f, 0.f, 0.f);
      s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
    }
    const float mu = block_sum512(s, red) * invC;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < WNV; ++i) {
      const int c = threadIdx.x + i * WIDE_NT;
      if (c < n4) {
        const float dx = v[i].x - mu, dy = v[i].y - mu, dz = v[i].z - mu, dw = v[i].w - mu;
        q += (dx * dx + dy * dy) + (dz * dz + dw * dw);
      }
    }
    const float rstd = rsqrtf(block_sum512(q, red) * invC + eps);
    float4* y4 = reinterpret_cast<float4*>(Y + r * ldy);
#pragma unroll
    for (int i = 0; i < WNV; ++i) {
      const int c = threadIdx.x + i * WIDE_NT;
      if (c < n4) {
        const float4 g = reinterpret_cast<const float4*>(gamma)[c], b = reinterpret_cast<const float4*>(beta)[c];
        float4 o;
        o.x = act_fwd(act, (v[i].x - mu) * rstd * g.x + b.x);
        o.y = act_fwd(act, (v[i].y - mu) * rstd * g.y + b.y);
        o.z = act_fwd(act, (v[i].z - mu) * rstd * g.z + b.z);
        o.w = act_fwd(act, (v[i].w - mu) * rstd * g.w + b.w);
        y4[c] = o;
      }
    }
  }
}

// DET: dgamma / dbeta are slot arrays with a row stride of 2*C floats, one slot per CTA (its threads own disjoint
// columns): plain stores in place of the global atomics.
template <bool DET>
__global__ void __launch_bounds__(WIDE_NT)
ln_act_bwd_wide_kernel(const float* __restrict__ X, const float* __restrict__ gamma, const float* __restrict__ beta,
                       const float* dY, float* dX, float* __restrict__ dgamma, float* __restrict__ dbeta, long long M, int C,
                       long long ldx, long long lddy, long long lddx, float eps, int act) {
  __shared__ float red[32];
  const int n4 = C >> 2;
  const float invC = 1.f / (float)C;
  const bool want_param = dgamma != nullptr;
  float4 ag[WNV], ab[WNV];
#pragma unroll
  for (int i = 0; i < WNV; ++i) { ag[i] = make_float4(0.f, 0.f, 0.f, 0.f); ab[i] = make_float4(0.f, 0.f, 0.f, 0.f); }
  for (long long r = blockIdx.x; r < M; r += gridDim.x) {
    const float4* x4 = reinterpret_cast<const float4*>(X + r * ldx);
    const float4* d4 = reinterpret_cast<const float4*>(dY + r * lddy);
    float4 v[WNV], d[WNV];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < WNV; ++i) {
      const int c = threadIdx.x + i * WIDE_NT;
      v[i] = (c < n4) ? x4[c] : make_float4(0.f, 0.f, 0.f, 0.f);
      d[i] = (c < n4) ? d4[c] : make_float4(0.f, 0.f, 0.f, 0.f);
      s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
    }
    const float mu = block_sum512(s, red) * invC;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < WNV; ++i) {
      const int c = threadIdx.x + i * WIDE_NT;
      if (c < n4) {
        const float dx = v[i].x - mu, dy = v[i].y - mu, dz = v[i].z - mu, dw = v[i].w - mu;
        q += (dx * dx + dy * dy) + (dz * dz + dw * dw);
      }
    }
    const float rstd = rsqrtf(block_sum512(q, red) * invC + eps);
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int i = 0; i < WNV; ++i) {
      const int c = threadIdx.x + i * WIDE_NT;
      if (c < n4) {
        const float4 g = reinterpret_cast<const float4*>(gamma)[c], b = reinterpret_cast<const float4*>(beta)[c];
        float4 xh, dl;
        xh.x = (v[i].x - mu) * rstd; xh.y = (v[i].y - mu) * rstd; xh.z = (v[i].z - mu) * rstd; xh.w = (v[i].w - mu) * rstd;
        dl.x = act_bwd(act, xh.x * g.x + b.x, d[i].x); dl.y = act_bwd(act, xh.y * g.y + b.y, d[i].y);
        dl.z = act_bwd(act, xh.z * g.z + b.z, d[i].z); dl.w = act_bwd(act, xh.w * g.w + b.w, d[i].w);
        ag[i].x += dl.x * xh.x; ag[i].y += dl.y * xh.y; ag[i].z += dl.z * xh.z; ag[i].w += dl.w * xh.w;
        ab[i].x += dl.x; ab[i].y += dl.y; ab[i].z += dl.z; ab[i].w += dl.w;
        d[i].x = dl.x * g.x; d[i].y = dl.y * g.y; d[i].z = dl.z * g.z; d[i].w = dl.w * g.w;
        v[i] = xh;
        s1 += (d[i].x + d[i].y) + (d[i].z + d[i].w);
        s2 += (d[i].x * xh.x + d[i].y * xh.y) + (d[i].z * xh.z + d[i].w * xh.w);
      }
    }
    s1 = block_sum512(s1, red) * invC;
    s2 = block_sum512(s2, red) * invC;
    float4* o4 = reinterpret_cast<float4*>(dX + r * lddx);
#pragma unroll
    for (int i = 0; i < WNV; ++i) {
      const int c = threadIdx.x + i * WIDE_NT;
      if (c < n4) {
        float4 o;
        o.x = rstd * (d[i].x - s1 - v[i].x * s2); o.y = rstd * (d[i].y - s1 - v[i].y * s2);
        o.z = rstd * (d[i].z - s1 - v[i].z * s2); o.w = rstd * (d[i].w - s1 - v[i].w * s2);
        o4[c] = o;
      }
    }
  }
  if (want_param) {
#pragma unroll
    for (int i = 0; i < WNV; ++i) {
      const int c = threadIdx.x + i * WIDE_NT;
      if (c < n4 && DET) {
        reinterpret_cast<float4*>(dgamma + (long long)blockIdx.x * 2 * C)[c] = ag[i];
        reinterpret_cast<float4*>(dbeta + (long long)blockIdx.x * 2 * C)[c] = ab[i];
      } else if (c < n4) {
        atomicAdd(&dgamma[4 * c + 0], ag[i].x); atomicAdd(&dgamma[4 * c + 1], ag[i].y);
        atomicAdd(&dgamma[4 * c + 2], ag[i].z); atomicAdd(&dgamma[4 * c + 3], ag[i].w);
        atomicAdd(&dbeta[4 * c + 0], ab[i].x); atomicAdd(&dbeta[4 * c + 1], ab[i].y);
        atomicAdd(&dbeta[4 * c + 2], ab[i].z); atomicAdd(&dbeta[4 * c + 3], ab[i].w);
      }
    }
  }
}

bool wide_ok(int C, long long ld0, long long ld1, long long ld2, const void* p0, const void* p1, const void* p2, const void* g,
             const void* b) {
  if (C <= 1536 || (C & 3) || C > 4 * WIDE_NT * WNV) return false;
  if ((ld0 | ld1 | ld2) & 3) return false;
  return ((reinterpret_cast<uintptr_t>(p0) | reinterpret_cast<uintptr_t>(p1) | reinterpret_cast<uintptr_t>(p2) |
           reinterpret_cast<uintptr_t>(g) | reinterpret_cast<uintptr_t>(b)) & 15) == 0;
}

// out[c] (+)= sum_m X[m,c]; blockDim = (32, 8); out pre-zeroed by the host wrapper unless accumulating.
// DET: `out` is the slot array, the CTA's partial goes to out[blockIdx.y * C + c] (det_sum_slots adds the slots).
template <bool DET>
__global__ void col_sum_kernel(const float* __restrict__ X, float* __restrict__ out, long long M, int C,
                               long long ldx, long long rows_per_block) {
  __shared__ float red[8][33];
  const int c = blockIdx.x * 32 + threadIdx.x;
  const long long r0 = (long long)blockIdx.y * rows_per_block;
  const long long r1 = min(M, r0 + rows_per_block);
  float s = 0.f;
  if (c < C)
    for (long long r = r0 + threadIdx.y; r < r1; r += 8) s += X[r * ldx + c];
  red[threadIdx.y][threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.y == 0 && c < C) {
    float t = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) t += red[i][threadIdx.x];
    if constexpr (DET) out[(long long)blockIdx.y * C + c] = t;
    else atomicAdd(&out[c], t);
  }
}

// Narrow contiguous matrices (C <= 32, ldx == C: the 3-channel image gradient behind the decoder's output bias): the
// matrix is read as one flat float4 stream.  The total thread count is a multiple of C, so the column of each of a
// thread's 4 vector slots never changes across its grid-stride iterations: 4 register accumulators, no per-element modulo.
// DET: the CTA's 1024 accumulators are staged in shared memory and thread c < C adds those of column c in thread order
// (then, in CTA 0, the unaligned tail) into slot out[blockIdx.x * C + c]: no shared or global atomics.
template <bool DET>
__global__ void __launch_bounds__(256)
col_sum_narrow_kernel(const float* __restrict__ X, float* __restrict__ out, long long total, int C) {
  __shared__ float bins[DET ? 1024 : 32];
  if constexpr (!DET) {
    if (threadIdx.x < 32) bins[threadIdx.x] = 0.f;
    __syncthreads();
  }
  const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x, nt = (long long)gridDim.x * blockDim.x;
  const long long n4 = total >> 2;
  float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
  for (long long j = tid; j < n4; j += nt) {
    const float4 v = __ldg(reinterpret_cast<const float4*>(X) + j);
    a0 += v.x; a1 += v.y; a2 += v.z; a3 += v.w;
  }
  if constexpr (DET) {
    float* b = bins + 4 * threadIdx.x;
    b[0] = a0; b[1] = a1; b[2] = a2; b[3] = a3;
    __syncthreads();
    if (threadIdx.x < C) {
      const int c = threadIdx.x;
      const long long base = 4LL * blockIdx.x * blockDim.x;      // flat element index of bins[0]
      float s = 0.f;
      for (int p = (int)((c - base % C + C) % C); p < 4 * (int)blockDim.x; p += C) s += bins[p];
      if (blockIdx.x == 0)
        for (long long i = (n4 << 2) + (c - (n4 << 2) % C + C) % C; i < total; i += C) s += X[i];
      out[(long long)blockIdx.x * C + c] = s;
    }
    return;
  }
  const int c0 = (int)((4 * tid) % C);
  if (tid < n4) {
    atomicAdd(&bins[c0], a0);
    atomicAdd(&bins[(c0 + 1) % C], a1);
    atomicAdd(&bins[(c0 + 2) % C], a2);
    atomicAdd(&bins[(c0 + 3) % C], a3);
  }
  if (tid == 0)
    for (long long i = n4 << 2; i < total; ++i) atomicAdd(&bins[(int)(i % C)], X[i]);
  __syncthreads();
  if (threadIdx.x < C && bins[threadIdx.x] != 0.f) atomicAdd(&out[threadIdx.x], bins[threadIdx.x]);
}


// ---------------------------------------------------------------------------------------------------------
// Vectorised row kernels: a row of C = 4*LPR*NV floats is held in registers by LPR lanes (NV float4 each), so X
// (and dY) are read exactly once with 128-bit accesses, 32/LPR rows are processed per warp at a time and the
// statistics are sub-warp shuffles.  These are the HBM-bound kernels of the conv stacks (C = 32..256, 1M rows).
// ---------------------------------------------------------------------------------------------------------
template <int LPR>
__device__ __forceinline__ float group_sum(float v) {
#pragma unroll
  for (int o = LPR / 2; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

template <int LPR, int NV>
__global__ void __launch_bounds__(256)
ln_act_fwd_vec_kernel(const float* __restrict__ X, const float* __restrict__ gamma, const float* __restrict__ beta,
                      float* __restrict__ Y, long long M, long long ldx, long long ldy, float eps, int act) {
  constexpr int RPW = 32 / LPR, C = 4 * LPR * NV;
  const int lane = threadIdx.x & 31, lr = lane % LPR, sub = lane / LPR;
  const long long gwarp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  float4 g[NV], b[NV];
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    g[i] = reinterpret_cast<const float4*>(gamma)[lr + i * LPR];
    b[i] = reinterpret_cast<const float4*>(beta)[lr + i * LPR];
  }
  const float invC = 1.f / (float)C;
  for (long long r0 = gwarp * RPW; r0 < M; r0 += nwarps * RPW) {
    const long long r = r0 + sub;
    const bool ok = r < M;
    float4 v[NV];
#pragma unroll
    for (int i = 0; i < NV; ++i)
      v[i] = ok ? reinterpret_cast<const float4*>(X + r * ldx)[lr + i * LPR] : make_float4(0.f, 0.f, 0.f, 0.f);
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
    const float mu = group_sum<LPR>(s) * invC;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const float dx = v[i].x - mu, dy = v[i].y - mu, dz = v[i].z - mu, dw = v[i].w - mu;
      q += (dx * dx + dy * dy) + (dz * dz + dw * dw);
    }
    const float rstd = rsqrtf(group_sum<LPR>(q) * invC + eps);
    if (ok) {
#pragma unroll
      for (int i = 0; i < NV; ++i) {
        float4 o;
        o.x = (v[i].x - mu) * rstd * g[i].x + b[i].x;
        o.y = (v[i].y - mu) * rstd * g[i].y + b[i].y;
        o.z = (v[i].z - mu) * rstd * g[i].z + b[i].z;
        o.w = (v[i].w - mu) * rstd * g[i].w + b[i].w;
        if (act != ACT_NONE) { o.x = act_fwd(act, o.x); o.y = act_fwd(act, o.y); o.z = act_fwd(act, o.z); o.w = act_fwd(act, o.w); }
        reinterpret_cast<float4*>(Y + r * ldy)[lr + i * LPR] = o;
      }
    }
  }
}

// DET: dgamma / dbeta are slot arrays with a row stride of 2*C floats, one slot per warp: the warp's row groups are
// added by a fixed butterfly and lanes 0..LPR-1 store the sums, in place of the shared and global atomics.
template <int LPR, int NV, bool DET>
__global__ void __launch_bounds__(256)
ln_act_bwd_vec_kernel(const float* __restrict__ X, const float* __restrict__ gamma, const float* __restrict__ beta,
                      const float* dY, float* dX, float* __restrict__ dgamma, float* __restrict__ dbeta, long long M,
                      long long ldx, long long lddy, long long lddx, float eps, int act) {
  constexpr int RPW = 32 / LPR, C = 4 * LPR * NV;
  __shared__ float sacc[DET ? 1 : 2 * C];
  const int lane = threadIdx.x & 31, lr = lane % LPR, sub = lane / LPR;
  const long long gwarp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  const bool want_param = dgamma != nullptr;
  if (want_param && !DET) {
    for (int c = threadIdx.x; c < 2 * C; c += blockDim.x) sacc[c] = 0.f;
    __syncthreads();
  }
  float4 g[NV], b[NV], ag[NV], ab[NV];
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    g[i] = reinterpret_cast<const float4*>(gamma)[lr + i * LPR];
    b[i] = reinterpret_cast<const float4*>(beta)[lr + i * LPR];
    ag[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    ab[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  const float invC = 1.f / (float)C;
  auto dact = [&](float ln, float dy) -> float { return act_bwd(act, ln, dy); };
  for (long long r0 = gwarp * RPW; r0 < M; r0 += nwarps * RPW) {
    const long long r = r0 + sub;
    const bool ok = r < M;
    float4 v[NV], d[NV];
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      v[i] = ok ? reinterpret_cast<const float4*>(X + r * ldx)[lr + i * LPR] : make_float4(0.f, 0.f, 0.f, 0.f);
      d[i] = ok ? reinterpret_cast<const float4*>(dY + r * lddy)[lr + i * LPR] : make_float4(0.f, 0.f, 0.f, 0.f);
    }
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
    const float mu = group_sum<LPR>(s) * invC;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const float dx = v[i].x - mu, dy = v[i].y - mu, dz = v[i].z - mu, dw = v[i].w - mu;
      q += (dx * dx + dy * dy) + (dz * dz + dw * dw);
    }
    const float rstd = rsqrtf(group_sum<LPR>(q) * invC + eps);
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      // v <- xh, d <- dxh ; accumulate parameter gradients
      float4 xh, dl;
      xh.x = (v[i].x - mu) * rstd; xh.y = (v[i].y - mu) * rstd; xh.z = (v[i].z - mu) * rstd; xh.w = (v[i].w - mu) * rstd;
      dl.x = dact(xh.x * g[i].x + b[i].x, d[i].x); dl.y = dact(xh.y * g[i].y + b[i].y, d[i].y);
      dl.z = dact(xh.z * g[i].z + b[i].z, d[i].z); dl.w = dact(xh.w * g[i].w + b[i].w, d[i].w);
      ag[i].x += dl.x * xh.x; ag[i].y += dl.y * xh.y; ag[i].z += dl.z * xh.z; ag[i].w += dl.w * xh.w;
      ab[i].x += dl.x; ab[i].y += dl.y; ab[i].z += dl.z; ab[i].w += dl.w;
      d[i].x = dl.x * g[i].x; d[i].y = dl.y * g[i].y; d[i].z = dl.z * g[i].z; d[i].w = dl.w * g[i].w;
      v[i] = xh;
      s1 += (d[i].x + d[i].y) + (d[i].z + d[i].w);
      s2 += (d[i].x * xh.x + d[i].y * xh.y) + (d[i].z * xh.z + d[i].w * xh.w);
    }
    s1 = group_sum<LPR>(s1) * invC;
    s2 = group_sum<LPR>(s2) * invC;
    if (ok) {
#pragma unroll
      for (int i = 0; i < NV; ++i) {
        float4 o;
        o.x = rstd * (d[i].x - s1 - v[i].x * s2); o.y = rstd * (d[i].y - s1 - v[i].y * s2);
        o.z = rstd * (d[i].z - s1 - v[i].z * s2); o.w = rstd * (d[i].w - s1 - v[i].w * s2);
        reinterpret_cast<float4*>(dX + r * lddx)[lr + i * LPR] = o;
      }
    }
  }
  if (want_param && DET) {
#pragma unroll
    for (int i = 0; i < NV; ++i) {
#pragma unroll
      for (int o = LPR; o < 32; o <<= 1) {
        ag[i].x += __shfl_xor_sync(0xffffffffu, ag[i].x, o); ag[i].y += __shfl_xor_sync(0xffffffffu, ag[i].y, o);
        ag[i].z += __shfl_xor_sync(0xffffffffu, ag[i].z, o); ag[i].w += __shfl_xor_sync(0xffffffffu, ag[i].w, o);
        ab[i].x += __shfl_xor_sync(0xffffffffu, ab[i].x, o); ab[i].y += __shfl_xor_sync(0xffffffffu, ab[i].y, o);
        ab[i].z += __shfl_xor_sync(0xffffffffu, ab[i].z, o); ab[i].w += __shfl_xor_sync(0xffffffffu, ab[i].w, o);
      }
      if (sub == 0) {
        reinterpret_cast<float4*>(dgamma + gwarp * 2 * C)[lr + i * LPR] = ag[i];
        reinterpret_cast<float4*>(dbeta + gwarp * 2 * C)[lr + i * LPR] = ab[i];
      }
    }
  } else if (want_param) {
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int c = 4 * (lr + i * LPR);
      atomicAdd(&sacc[c + 0], ag[i].x); atomicAdd(&sacc[c + 1], ag[i].y); atomicAdd(&sacc[c + 2], ag[i].z); atomicAdd(&sacc[c + 3], ag[i].w);
      atomicAdd(&sacc[C + c + 0], ab[i].x); atomicAdd(&sacc[C + c + 1], ab[i].y); atomicAdd(&sacc[C + c + 2], ab[i].z); atomicAdd(&sacc[C + c + 3], ab[i].w);
    }
    __syncthreads();
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
      atomicAdd(&dgamma[c], sacc[c]);
      atomicAdd(&dbeta[c], sacc[C + c]);
    }
  }
}

int vec_grid(long long M, int rows_per_warp) {
  long long warps = (M + rows_per_warp - 1) / rows_per_warp;
  long long blocks = (warps + 7) / 8;
  const long long cap = (long long)kNumSMs * 8;
  if (blocks > cap) blocks = cap;
  return (int)(blocks < 1 ? 1 : blocks);
}
bool vec_ok(int C, long long ld0, long long ld1, long long ld2, const void* p0, const void* p1, const void* p2, const void* g,
            const void* b) {
  // widths with a register-resident instantiation: powers of two 32..1024, 1536 (S GRU: 3*512) and the 3 * 2^k family
  // of the M / L / XL conv stacks and dense layers (48, 96, 192, 384, 768; cnn multipliers 48 / 96, dense 768), 640 (M)
  switch (C) {
    case 32: case 64: case 128: case 256: case 512: case 1024: case 1536:
    case 48: case 96: case 192: case 384: case 768: case 640: break;
    default: return false;
  }
  if ((ld0 | ld1 | ld2) & 3) return false;
  return ((reinterpret_cast<uintptr_t>(p0) | reinterpret_cast<uintptr_t>(p1) | reinterpret_cast<uintptr_t>(p2) |
           reinterpret_cast<uintptr_t>(g) | reinterpret_cast<uintptr_t>(b)) & 15) == 0;
}

int grid_for_rows(long long M) {
  long long blocks = (M + 7) / 8;  // 8 warps (rows) per 256-thread block
  const long long cap = (long long)kNumSMs * 8;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  return (int)blocks;
}

constexpr int ROUTE_GENERIC = 0, ROUTE_VEC = 1, ROUTE_WIDE = 2;

}  // namespace

extern "C" int b200rl_ln_act_route(int C, long long ld0, long long ld1, long long ld2, const float* p0, const float* p1,
                                   const float* p2, const float* gamma, const float* beta) {
  if (vec_ok(C, ld0, ld1, ld2, p0, p1, p2, gamma, beta)) return ROUTE_VEC;
  if (wide_ok(C, ld0, ld1, ld2, p0, p1, p2, gamma, beta)) return ROUTE_WIDE;
  return ROUTE_GENERIC;
}

extern "C" int b200rl_ln_act_fwd(const float* X, const float* gamma, const float* beta, float* Y, long long M, int C,
                                 long long ldx, long long ldy, float eps, int act, cudaStream_t st) {
  RL_CHECK_ARG(X && gamma && beta && Y, "null pointer");
  RL_CHECK_ARG(C > 0 && ldx >= C && ldy >= C, "bad C / ld");
  RL_CHECK_ARG(act >= ACT_NONE && act <= ACT_RELU, "act must be 0 (none), 1 (SiLU), 2 (tanh) or 3 (ReLU)");
  if (M <= 0) return B200RL_OK;
  const int route = b200rl_ln_act_route(C, ldx, ldy, 0, X, Y, nullptr, gamma, beta);
  if (route == ROUTE_VEC) {
#define LN_FWD_VEC(LPR_, NV_) \
  ln_act_fwd_vec_kernel<LPR_, NV_><<<vec_grid(M, 32 / LPR_), 256, 0, st>>>(X, gamma, beta, Y, M, ldx, ldy, eps, act)
    switch (C) {
      case 32: LN_FWD_VEC(8, 1); break;
      case 64: LN_FWD_VEC(16, 1); break;
      case 128: LN_FWD_VEC(32, 1); break;
      case 256: LN_FWD_VEC(32, 2); break;
      case 512: LN_FWD_VEC(32, 4); break;
      case 1024: LN_FWD_VEC(32, 8); break;
      case 48: LN_FWD_VEC(4, 3); break;
      case 96: LN_FWD_VEC(8, 3); break;
      case 192: LN_FWD_VEC(16, 3); break;
      case 384: LN_FWD_VEC(32, 3); break;
      case 640: LN_FWD_VEC(32, 5); break;
      case 768: LN_FWD_VEC(32, 6); break;
      default: LN_FWD_VEC(32, 12); break;
    }
#undef LN_FWD_VEC
    RL_CHECK_LAUNCH();
    return B200RL_OK;
  }
  if (route == ROUTE_WIDE) {
    const int grid = (int)(M < 4LL * kNumSMs ? M : 4LL * kNumSMs);
    ln_act_fwd_wide_kernel<<<grid, WIDE_NT, 0, st>>>(X, gamma, beta, Y, M, C, ldx, ldy, eps, act);
    RL_CHECK_LAUNCH();
    return B200RL_OK;
  }
  ln_act_fwd_kernel<<<grid_for_rows(M), 256, 0, st>>>(X, gamma, beta, Y, M, C, ldx, ldy, eps, act);
  RL_CHECK_LAUNCH();
  return B200RL_OK;
}

extern "C" int b200rl_ln_act_bwd(const float* X, const float* gamma, const float* beta, const float* dY, float* dX,
                                 float* dgamma, float* dbeta, long long M, int C, long long ldx, long long lddy,
                                 long long lddx, float eps, int act, int accumulate, cudaStream_t st) {
  RL_CHECK_ARG(X && gamma && beta && dY && dX, "null pointer");
  RL_CHECK_ARG((dgamma == nullptr) == (dbeta == nullptr), "dgamma/dbeta must both be given or both be null");
  RL_CHECK_ARG(C > 0 && ldx >= C && lddy >= C && lddx >= C, "bad C / ld");
  RL_CHECK_ARG(act >= ACT_NONE && act <= ACT_RELU, "act must be 0 (none), 1 (SiLU), 2 (tanh) or 3 (ReLU)");
  const int route = b200rl_ln_act_route(C, ldx, lddy, lddx, X, dY, dX, gamma, beta);
  // every refusal comes before the first write: a refused call leaves dgamma / dbeta as the caller had them
  RL_CHECK_ARG(route != ROUTE_GENERIC || C <= 28000, "C too large for the shared accumulator path");
  if (dgamma && !accumulate) {
    RL_CUDA(cudaMemsetAsync(dgamma, 0, sizeof(float) * C, st));
    RL_CUDA(cudaMemsetAsync(dbeta, 0, sizeof(float) * C, st));
  }
  if (M <= 0) return B200RL_OK;
  // deterministic mode: the kernels write per-warp (per-CTA on the wide route) partials to `slots` slots of 2*C floats
  // and det_sum_slots adds them to dgamma / dbeta in slot order
  const bool det = dgamma && det_mode();
  float* pg = dgamma;
  float* pb = dbeta;
  auto slots_ws = [&](long long slots) -> int {
    void* ws = nullptr;
    if (int rc = det_workspace(sizeof(float) * 2 * (size_t)C * slots, st, &ws)) return rc;
    pg = static_cast<float*>(ws);
    pb = pg + C;
    return B200RL_OK;
  };
  auto finish = [&](long long slots) -> int {
    RL_CHECK_LAUNCH();
    if (!det) return B200RL_OK;
    return det_sum_slots(pg, (int)slots, 2LL * C, dgamma, C, dbeta, st);
  };
  if (route == ROUTE_VEC) {
    // every CTA ends with 2*C global atomics into dgamma / dbeta: for wide rows (a warp already keeps >= 2 KB in flight) two
    // CTAs per SM saturate HBM and cut that traffic 4x (ncu: [16384,512] ran at 0.34 of the HBM peak with 1184 CTAs).
    // Deterministic mode takes the same cap at every width: it bounds the slots the reduction reads.
    const int bwd_cap = (dgamma && (C >= 256 || det)) ? 2 * kNumSMs : (1 << 30);
    int vgrid = 0;
#define LN_BWD_VEC(LPR_, NV_)                                                                                         \
  do {                                                                                                                \
    vgrid = min(vec_grid(M, 32 / LPR_), bwd_cap);                                                                     \
    if (!det) {                                                                                                       \
      ln_act_bwd_vec_kernel<LPR_, NV_, false><<<vgrid, 256, 0, st>>>(X, gamma, beta, dY, dX, dgamma, dbeta, M, ldx,   \
                                                                     lddy, lddx, eps, act);                           \
    } else {                                                                                                          \
      if (int rc = slots_ws(8LL * vgrid)) return rc;                                                                  \
      ln_act_bwd_vec_kernel<LPR_, NV_, true><<<vgrid, 256, 0, st>>>(X, gamma, beta, dY, dX, pg, pb, M, ldx, lddy, lddx,\
                                                                    eps, act);                                        \
    }                                                                                                                 \
  } while (0)
    switch (C) {
      case 32: LN_BWD_VEC(8, 1); break;
      case 64: LN_BWD_VEC(16, 1); break;
      case 128: LN_BWD_VEC(32, 1); break;
      case 256: LN_BWD_VEC(32, 2); break;
      case 512: LN_BWD_VEC(32, 4); break;
      case 1024: LN_BWD_VEC(32, 8); break;
      case 48: LN_BWD_VEC(4, 3); break;
      case 96: LN_BWD_VEC(8, 3); break;
      case 192: LN_BWD_VEC(16, 3); break;
      case 384: LN_BWD_VEC(32, 3); break;
      case 640: LN_BWD_VEC(32, 5); break;
      case 768: LN_BWD_VEC(32, 6); break;
      default: LN_BWD_VEC(32, 12); break;
    }
#undef LN_BWD_VEC
    return finish(8LL * vgrid);
  }
  if (route == ROUTE_WIDE) {
    const int wgrid = (int)(M < 2LL * kNumSMs ? M : 2LL * kNumSMs);
    if (det) {
      if (int rc = slots_ws(wgrid)) return rc;
      ln_act_bwd_wide_kernel<true><<<wgrid, WIDE_NT, 0, st>>>(X, gamma, beta, dY, dX, pg, pb, M, C, ldx, lddy, lddx, eps,
                                                              act);
    } else {
      ln_act_bwd_wide_kernel<false><<<wgrid, WIDE_NT, 0, st>>>(X, gamma, beta, dY, dX, dgamma, dbeta, M, C, ldx, lddy,
                                                               lddx, eps, act);
    }
    return finish(wgrid);
  }
  int grid = grid_for_rows(M);
  if (dgamma && grid > 2 * kNumSMs) grid = 2 * kNumSMs;  // fewer, longer-lived warps -> fewer flush atomics
  // deterministic mode, C > 512: a slot of 2*C floats per warp, so fewer warps (the route no engine width takes)
  if (det && C > 512 && grid > 32) grid = 32;
  if (det)
    if (int rc = slots_ws(8LL * grid)) return rc;
  // the default instances are instantiated first: that keeps their code the default path's code before DET
#define LN_BWD(CPL_, SMEM_)                                                                                           \
  do {                                                                                                                \
    if (!det)                                                                                                         \
      ln_act_bwd_kernel<CPL_, false><<<grid, 256, SMEM_, st>>>(X, gamma, beta, dY, dX, dgamma, dbeta, M, C, ldx, lddy,\
                                                               lddx, eps, act);                                       \
    else                                                                                                              \
      ln_act_bwd_kernel<CPL_, true><<<grid, 256, 0, st>>>(X, gamma, beta, dY, dX, pg, pb, M, C, ldx, lddy, lddx, eps, \
                                                          act);                                                       \
  } while (0)
  if (C <= 32) LN_BWD(1, 0);
  else if (C <= 64) LN_BWD(2, 0);
  else if (C <= 128) LN_BWD(4, 0);
  else if (C <= 256) LN_BWD(8, 0);
  else if (C <= 512) LN_BWD(16, 0);
  else {
    // wide rows (XL: the GRU's joint LayerNorm spans 3*4096 channels): per-CTA gamma/beta partials in opted-in smem
    // (C <= 28000, checked above)
    const size_t smem = sizeof(float) * 2 * (size_t)C;
    if (smem > 48 * 1024 && !det)
      RL_CUDA(cudaFuncSetAttribute(ln_act_bwd_kernel<0, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    LN_BWD(0, smem);
  }
#undef LN_BWD
  return finish(8LL * grid);
}

extern "C" int b200rl_col_sum(const float* X, float* out, long long M, int C, long long ldx, int accumulate,
                              cudaStream_t st) {
  RL_CHECK_ARG(X && out, "null pointer");
  RL_CHECK_ARG(C > 0 && ldx >= C, "bad C / ld");
  if (!accumulate) RL_CUDA(cudaMemsetAsync(out, 0, sizeof(float) * C, st));
  if (M <= 0) return B200RL_OK;
  const bool det = det_mode();
  void* ws = nullptr;
  if (C <= 32 && ldx == C && M * C >= (1 << 16) && (reinterpret_cast<uintptr_t>(X) & 15) == 0) {
    int blocks = 4 * kNumSMs;
    blocks = (blocks + C - 1) / C * C;             // thread count divisible by C: fixed column per vector slot
    if (det) {
      if (int rc = det_workspace(sizeof(float) * blocks * C, st, &ws)) return rc;
      col_sum_narrow_kernel<true><<<blocks, 256, 0, st>>>(X, static_cast<float*>(ws), M * C, C);
      RL_CHECK_LAUNCH();
      return det_sum_slots(static_cast<const float*>(ws), blocks, C, out, C, nullptr, st);
    }
    col_sum_narrow_kernel<false><<<blocks, 256, 0, st>>>(X, out, M * C, C);
    RL_CHECK_LAUNCH();
    return B200RL_OK;
  }
  const int cb = ceil_div(C, 32);
  long long rb = (2LL * kNumSMs + cb - 1) / cb;
  long long rows_per_block = (M + rb - 1) / rb;
  if (rows_per_block < 64) rows_per_block = 64;
  rb = (M + rows_per_block - 1) / rows_per_block;
  if (det) {
    if (int rc = det_workspace(sizeof(float) * rb * C, st, &ws)) return rc;
    col_sum_kernel<true><<<dim3(cb, (unsigned)rb), dim3(32, 8), 0, st>>>(X, static_cast<float*>(ws), M, C, ldx,
                                                                         rows_per_block);
    RL_CHECK_LAUNCH();
    return det_sum_slots(static_cast<const float*>(ws), (int)rb, C, out, C, nullptr, st);
  }
  col_sum_kernel<false><<<dim3(cb, (unsigned)rb), dim3(32, 8), 0, st>>>(X, out, M, C, ldx, rows_per_block);
  RL_CHECK_LAUNCH();
  return B200RL_OK;
}
