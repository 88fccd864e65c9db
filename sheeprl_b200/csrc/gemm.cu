// fp32 SIMT GEMM family: C[M,N] = op(A) * op(B) (+bias) (+C)
//
// This is the exact-fp32 (FFMA) path used for (a) the latency-bound skinny GEMMs of the RSSM scan
// (M = batch 16) and (b) every shape the tensor-core path (gemm_tc.cu, 3xTF32 wgmma) does not take.
// Register-blocked, shared-memory tiled, register-prefetch double buffered, optional split-K
// (fp32 atomics) so that weight-gradient GEMMs (tiny output, reduction over T*B rows) fill the SMs.
//
// Reference ops replaced: nn.Linear forward / its autograd backward as used throughout
// sheeprl/algos/dreamer_v3/agent.py (MLP, RecurrentModel, representation/transition models).
#include <stdlib.h>

#include "common.cuh"

namespace {

template <int BM, int BN, int BK, int TM, int TN, bool TA, bool TB>
__global__ void __launch_bounds__((BM / TM) * (BN / TN))
sgemm_kernel(const float* __restrict__ A, const float* __restrict__ B, float* __restrict__ C,
             const float* __restrict__ bias, int M, int N, int K, int lda, int ldb, int ldc,
             int accumulate, int kchunk) {
  constexpr int NT = (BM / TM) * (BN / TN);
  constexpr int PAD = 4;
  constexpr int RCH = (TM >= 4) ? 4 : TM, NRC = TM / RCH;
  constexpr int CCH = (TN >= 4) ? 4 : TN, NCC = TN / CCH;
  constexpr int LA = (BM * BK) / NT, LB = (BN * BK) / NT;
  static_assert((BM * BK) % NT == 0 && (BN * BK) % NT == 0, "tile/thread mismatch");
  __shared__ __align__(16) float As[BK][BM + PAD];
  __shared__ __align__(16) float Bs[BK][BN + PAD];

  const int tid = threadIdx.x;
  const int tx = tid % (BN / TN), ty = tid / (BN / TN);
  const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
  const int kbeg = blockIdx.z * kchunk;
  const int kend = min(K, kbeg + kchunk);

  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

  float ra[LA], rb[LB];

  auto load_tiles = [&](int k0) {
#pragma unroll
    for (int l = 0; l < LA; ++l) {
      const int e = tid + l * NT;
      int mm, kk;
      if (TA) { mm = e % BM; kk = e / BM; } else { kk = e % BK; mm = e / BK; }
      const int gm = m0 + mm, gk = k0 + kk;
      float v = 0.f;
      if (gm < M && gk < kend) v = TA ? A[(size_t)gk * lda + gm] : A[(size_t)gm * lda + gk];
      ra[l] = v;
    }
#pragma unroll
    for (int l = 0; l < LB; ++l) {
      const int e = tid + l * NT;
      int nn, kk;
      if (TB) { kk = e % BK; nn = e / BK; } else { nn = e % BN; kk = e / BN; }
      const int gn = n0 + nn, gk = k0 + kk;
      float v = 0.f;
      if (gn < N && gk < kend) v = TB ? B[(size_t)gn * ldb + gk] : B[(size_t)gk * ldb + gn];
      rb[l] = v;
    }
  };
  auto store_tiles = [&]() {
#pragma unroll
    for (int l = 0; l < LA; ++l) {
      const int e = tid + l * NT;
      int mm, kk;
      if (TA) { mm = e % BM; kk = e / BM; } else { kk = e % BK; mm = e / BK; }
      As[kk][mm] = ra[l];
    }
#pragma unroll
    for (int l = 0; l < LB; ++l) {
      const int e = tid + l * NT;
      int nn, kk;
      if (TB) { kk = e % BK; nn = e / BK; } else { nn = e % BN; kk = e / BN; }
      Bs[kk][nn] = rb[l];
    }
  };

  if (kbeg < kend) {
    load_tiles(kbeg);
    for (int k0 = kbeg; k0 < kend; k0 += BK) {
      store_tiles();
      __syncthreads();
      if (k0 + BK < kend) load_tiles(k0 + BK);  // prefetch next tile into registers during the math
#pragma unroll
      for (int kk = 0; kk < BK; ++kk) {
        float a[TM], b[TN];
#pragma unroll
        for (int c = 0; c < NRC; ++c)
#pragma unroll
          for (int i = 0; i < RCH; ++i) a[c * RCH + i] = As[kk][c * (BM / NRC) + ty * RCH + i];
#pragma unroll
        for (int c = 0; c < NCC; ++c)
#pragma unroll
          for (int j = 0; j < CCH; ++j) b[c * CCH + j] = Bs[kk][c * (BN / NCC) + tx * CCH + j];
#pragma unroll
        for (int i = 0; i < TM; ++i)
#pragma unroll
          for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
      }
      __syncthreads();
    }
  }

  const bool split = gridDim.z > 1;
#pragma unroll
  for (int i = 0; i < TM; ++i) {
    const int gm = m0 + (i / RCH) * (BM / NRC) + ty * RCH + (i % RCH);
    if (gm >= M) continue;
#pragma unroll
    for (int j = 0; j < TN; ++j) {
      const int gn = n0 + (j / CCH) * (BN / NCC) + tx * CCH + (j % CCH);
      if (gn >= N) continue;
      float* p = C + (size_t)gm * ldc + gn;
      if (split) {
        atomicAdd(p, acc[i][j]);  // C was initialised (bias / zero / kept) by init2d_kernel
      } else {
        float v = acc[i][j];
        if (bias) v += bias[gn];
        if (accumulate) v += *p;
        *p = v;
      }
    }
  }
}

__global__ void init2d_kernel(float* __restrict__ C, const float* __restrict__ bias, int M, int N, int ldc) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)M * N) return;
  const int m = (int)(idx / N), n = (int)(idx % N);
  C[(size_t)m * ldc + n] = bias ? bias[n] : 0.f;
}

__global__ void addbias2d_kernel(float* __restrict__ C, const float* __restrict__ bias, int M, int N, int ldc) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)M * N) return;
  const int m = (int)(idx / N), n = (int)(idx % N);
  C[(size_t)m * ldc + n] += bias[n];
}

template <int BM, int BN, int BK, int TM, int TN>
int launch_cfg(const float* A, const float* B, float* C, const float* bias, int M, int N, int K, int lda, int ldb,
               int ldc, int transA, int transB, int accumulate, cudaStream_t st) {
  const int tm = ceil_div(M, BM), tn = ceil_div(N, BN);
  const int tiles = tm * tn;
  int splits = 1;
  if (tiles < kNumSMs && K >= 8 * BK) {
    splits = min(ceil_div(2 * kNumSMs, tiles), K / (4 * BK));
    if (splits < 1) splits = 1;
  }
  int kchunk = ceil_div(ceil_div(K, splits), BK) * BK;
  splits = ceil_div(K, kchunk);
  if (splits > 1) {
    const long long tot = (long long)M * N;
    if (!accumulate)
      init2d_kernel<<<ceil_div(tot, 256), 256, 0, st>>>(C, bias, M, N, ldc);
    else if (bias)
      addbias2d_kernel<<<ceil_div(tot, 256), 256, 0, st>>>(C, bias, M, N, ldc);
  }
  dim3 grid(tn, tm, splits), block((BM / TM) * (BN / TN));
#define LAUNCH(TA_, TB_)                                                                                    \
  sgemm_kernel<BM, BN, BK, TM, TN, TA_, TB_><<<grid, block, 0, st>>>(A, B, C, bias, M, N, K, lda, ldb, ldc, \
                                                                     accumulate, kchunk)
  if (transA) { if (transB) LAUNCH(true, true); else LAUNCH(true, false); }
  else        { if (transB) LAUNCH(false, true); else LAUNCH(false, false); }
#undef LAUNCH
  RL_CHECK_LAUNCH();
  return B200RL_OK;
}

}  // namespace

extern "C" int b200rl_gemm_tc_supported(const float* A, const float* B, int M, int N, int K, int lda, int ldb,
                                        int transA, int transB);
extern "C" int b200rl_gemm_tc(const float* A, const float* B, float* C, const float* bias, int M, int N, int K, int lda,
                              int ldb, int ldc, int transA, int transB, int accumulate, cudaStream_t st);

static bool tc_enabled() {
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("B200RL_DISABLE_TC");
    v = (e && e[0] == '1') ? 0 : 1;
  }
  return v == 1;
}

// Rank-K update for tiny K (input gradient of a policy head with a handful of actions: [rows, A] x [A, hidden]):
// C[m, n..n+3] (+)= bias + sum_k A[m, k] * B[k, n..n+3], one float4 of C per thread, B rows through the read-only cache.
// The tiled kernels below spend a whole 16-deep k-step on K = 2.
template <int KMAX>
__global__ void __launch_bounds__(256)
rank_k_nn_kernel(const float* __restrict__ A, const float* __restrict__ B, float* __restrict__ C, const float* __restrict__ bias,
                 int M, int N, int K, int lda, int ldb, int ldc, int accumulate) {
  const int n4 = N >> 2;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)M * n4) return;
  const int m = (int)(idx / n4), c = (int)(idx - (long long)m * n4);
  float4 acc = bias ? reinterpret_cast<const float4*>(bias)[c] : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
  for (int k = 0; k < KMAX; ++k) {
    if (k < K) {
      const float a = __ldg(A + (size_t)m * lda + k);
      const float4 b = __ldg(reinterpret_cast<const float4*>(B + (size_t)k * ldb) + c);
      acc.x = fmaf(a, b.x, acc.x); acc.y = fmaf(a, b.y, acc.y); acc.z = fmaf(a, b.z, acc.z); acc.w = fmaf(a, b.w, acc.w);
    }
  }
  float4* out = reinterpret_cast<float4*>(C + (size_t)m * ldc) + c;
  if (accumulate) { const float4 o = *out; acc.x += o.x; acc.y += o.y; acc.z += o.z; acc.w += o.w; }
  *out = acc;
}

// include/b200rl.h: b200rl_gemm_f32.  Large NT products go to the wgmma 3xTF32 kernel (gemm_tc.cu); everything
// else (skinny, transposed, unaligned) runs on the exact-fp32 FFMA kernels below.
extern "C" int b200rl_gemm_f32(const float* A, const float* B, float* C, const float* bias, int M, int N, int K,
                               int lda, int ldb, int ldc, int transA, int transB, int accumulate,
                               cudaStream_t st) {
  RL_CHECK_ARG(A && B && C, "null pointer");
  RL_CHECK_ARG(M >= 0 && N >= 0 && K >= 0, "negative dimension");
  if (M == 0 || N == 0) return B200RL_OK;
  RL_CHECK_ARG(lda >= (transA ? M : K) && ldb >= (transB ? K : N) && ldc >= N, "leading dimension too small");
  if (K == 0) {   // empty product: C = bias (or 0), or C += bias when accumulating
    if (!accumulate)
      init2d_kernel<<<ceil_div((long long)M * N, 256), 256, 0, st>>>(C, bias, M, N, ldc);
    else if (bias)
      addbias2d_kernel<<<ceil_div((long long)M * N, 256), 256, 0, st>>>(C, bias, M, N, ldc);
    else
      return B200RL_OK;
    RL_CHECK_LAUNCH();
    return B200RL_OK;
  }
  if (tc_enabled() && b200rl_gemm_tc_supported(A, B, M, N, K, lda, ldb, transA, transB))
    return b200rl_gemm_tc(A, B, C, bias, M, N, K, lda, ldb, ldc, transA, transB, accumulate, st);
  if (!transA && !transB && K <= 8 && M >= 1024 && (N & 3) == 0 && (ldb & 3) == 0 && (ldc & 3) == 0 &&
      ((reinterpret_cast<uintptr_t>(B) | reinterpret_cast<uintptr_t>(C) | reinterpret_cast<uintptr_t>(bias)) & 15) == 0) {
    rank_k_nn_kernel<8><<<ceil_div((long long)M * (N >> 2), 256), 256, 0, st>>>(A, B, C, bias, M, N, K, lda, ldb, ldc, accumulate);
    RL_CHECK_LAUNCH();
    return B200RL_OK;
  }
  if (M <= 32) return launch_cfg<16, 64, 32, 1, 8>(A, B, C, bias, M, N, K, lda, ldb, ldc, transA, transB, accumulate, st);
  if (N <= 32) return launch_cfg<128, 32, 16, 8, 2>(A, B, C, bias, M, N, K, lda, ldb, ldc, transA, transB, accumulate, st);
  if (M <= 64 || N <= 64)
    return launch_cfg<64, 64, 16, 4, 4>(A, B, C, bias, M, N, K, lda, ldb, ldc, transA, transB, accumulate, st);
  return launch_cfg<128, 128, 16, 8, 8>(A, B, C, bias, M, N, K, lda, ldb, ldc, transA, transB, accumulate, st);
}
