// Batched strided small-GEMM with fused epilogues: the Linear layers of the SAC / PPO updates.
//
// Replaces (reference): every nn.Linear + activation of sheeprl/models/models.py:16-119 (MLP) as used by
// SACActor / SACCritic (sheeprl/algos/sac/agent.py:19-108) and PPOAgent (sheeprl/algos/ppo/agent.py:84-177), forward
// and the three autograd products of each layer.  These updates are launch-latency bound (B = 64..256 rows, 64..256
// units: ~40 MFLOP per layer), so the design goal is FEW launches, not tensor-core tiles:
//   * `nets` independent networks (the twin critics and their targets) run in ONE launch (blockIdx.z) with a constant
//     stride between their parameter blocks in the flat group;
//   * bias, ReLU / Tanh, and the activation derivative of the backward-data product are epilogues;
//   * the bias gradient (column sum of dY) is produced by the weight-gradient launch itself (row sums of its A
//     operand), so a layer's backward is exactly two launches.
// All operands are addressed through (row stride, column stride) pairs, which covers NN / NT / TN without copies.
#include "common.cuh"

namespace {

enum { EPI_NONE = 0, EPI_RELU = 1, EPI_TANH = 2, EPI_DRELU = 3, EPI_DTANH = 4 };

struct BG {
  const float* A; long long sam, sak, strideA;      // A(m,k) = A[m*sam + k*sak]
  const float* B; long long sbk, sbn, strideB;      // B(k,n) = B[k*sbk + n*sbn]
  float* C; long long ldc, strideC;                 // C(m,n) = C[m*ldc + n]
  const float* bias; long long strideBias;          // + bias[n]            (may be null)
  const float* aux; long long ldaux, strideAux;     // activation output of the layer, for EPI_D*
  float* rsum; long long strideRsum;                // rsum[m] = sum_k A(m,k) (may be null)
  int M, N, K, epi, accumulate;
};

// Tile kernel: BMxBN outputs per CTA, TMxTN per thread, 256 threads, BK-deep k-steps, double-buffered shared
// tiles with register prefetch of the next k-step (these products are latency- not throughput-bound: without the
// prefetch every k-step pays a full L2 round trip).  blockIdx.z = net * ksplit + split; with ksplit > 1 each CTA
// reduces a K-slice and adds its partial tile with fp32 atomics (weight gradients: long K, tiny output).
template <int BM, int BN, int TM, int TN, int BK>
__global__ void __launch_bounds__(256) bgemm_kernel(const BG g, const int ksplit, const int kper) {
  constexpr int NT = (BM / TM) * (BN / TN);
  static_assert(NT == 256, "256 threads");
  constexpr int EA = BM * BK / NT, EB = BN * BK / NT;
  __shared__ float As[2][BK][BM + 1];
  __shared__ float Bs[2][BK][BN + 1];
  const int net = blockIdx.z / ksplit, ks = blockIdx.z - net * ksplit;
  const float* __restrict__ A = g.A + net * g.strideA;
  const float* __restrict__ B = g.B + net * g.strideB;
  const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
  const int kbeg = ks * kper, kend = min(g.K, kbeg + kper);
  const int tid = threadIdx.x;
  const int tx = tid % (BN / TN), ty = tid / (BN / TN);
  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;
  float rs = 0.f;                                    // row sum of A for row m0 + tid (tid < BM)
  const bool want_rsum = g.rsum != nullptr && blockIdx.x == 0;
  const bool a_kfast = g.sak == 1, b_nfast = g.sbn == 1;
  float ra[EA], rb[EB];
  auto fetch = [&](int k0) {
#pragma unroll
    for (int e = 0; e < EA; ++e) {                   // consecutive threads walk the unit-stride dimension
      const int idx = tid + e * NT;
      const int m = a_kfast ? idx / BK : idx % BM;
      const int k = a_kfast ? idx % BK : idx / BM;
      const int gm = m0 + m, gk = k0 + k;
      ra[e] = (gm < g.M && gk < kend) ? __ldg(A + gm * g.sam + gk * g.sak) : 0.f;
    }
#pragma unroll
    for (int e = 0; e < EB; ++e) {
      const int idx = tid + e * NT;
      const int n = b_nfast ? idx % BN : idx / BK;
      const int k = b_nfast ? idx / BN : idx % BK;
      const int gn = n0 + n, gk = k0 + k;
      rb[e] = (gn < g.N && gk < kend) ? __ldg(B + gk * g.sbk + gn * g.sbn) : 0.f;
    }
  };
  auto stash = [&](int buf) {
#pragma unroll
    for (int e = 0; e < EA; ++e) {
      const int idx = tid + e * NT;
      const int m = a_kfast ? idx / BK : idx % BM;
      const int k = a_kfast ? idx % BK : idx / BM;
      As[buf][k][m] = ra[e];
    }
#pragma unroll
    for (int e = 0; e < EB; ++e) {
      const int idx = tid + e * NT;
      const int n = b_nfast ? idx % BN : idx / BK;
      const int k = b_nfast ? idx / BN : idx % BK;
      Bs[buf][k][n] = rb[e];
    }
  };
  int cur = 0;
  if (kbeg < kend) {
    fetch(kbeg);
    stash(0);
  }
  __syncthreads();
  for (int k0 = kbeg; k0 < kend; k0 += BK) {
    const bool more = k0 + BK < kend;
    if (more) fetch(k0 + BK);
    if (want_rsum && tid < BM) {
#pragma unroll
      for (int k = 0; k < BK; ++k) rs += As[cur][k][tid];
    }
#pragma unroll
    for (int k = 0; k < BK; ++k) {
      float a[TM], b[TN];
#pragma unroll
      for (int i = 0; i < TM; ++i) a[i] = As[cur][k][ty * TM + i];
#pragma unroll
      for (int j = 0; j < TN; ++j) b[j] = Bs[cur][k][tx * TN + j];
#pragma unroll
      for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    if (more) stash(cur ^ 1);
    __syncthreads();
    cur ^= 1;
  }
  float* __restrict__ C = g.C + net * g.strideC;
  const float* __restrict__ bias = g.bias ? g.bias + net * g.strideBias : nullptr;
  const float* __restrict__ aux = g.aux ? g.aux + net * g.strideAux : nullptr;
  if (ksplit > 1) {
    // partial tile of a split-K product (plain epilogue, checked by the host): float2 reductions where the row allows.
    // Only the 32x32 tile (TN = 2) is ever split: the host takes wider tiles only when they already fill the SMs.
#pragma unroll
    for (int i = 0; i < TM; ++i) {
      const int m = m0 + ty * TM + i;
      if (m >= g.M) continue;
      const int n = n0 + tx * TN;
      float* c = C + m * g.ldc + n;
      bool done = false;
      if constexpr (TN == 2) {
        if (n + 1 < g.N && ((reinterpret_cast<uintptr_t>(c) & 7) == 0)) {
          atomicAdd(reinterpret_cast<float2*>(c), make_float2(acc[i][0], acc[i][1]));
          done = true;
        }
      }
      if (!done) {
#pragma unroll
        for (int j = 0; j < TN; ++j)
          if (n + j < g.N) atomicAdd(c + j, acc[i][j]);
      }
    }
  } else
#pragma unroll
  for (int i = 0; i < TM; ++i) {
    const int m = m0 + ty * TM + i;
    if (m >= g.M) continue;
#pragma unroll
    for (int j = 0; j < TN; ++j) {
      const int n = n0 + tx * TN + j;
      if (n >= g.N) continue;
      float v = acc[i][j];
      float* c = C + m * g.ldc + n;
      if (bias) v += bias[n];
      if (g.epi == EPI_RELU) v = fmaxf(v, 0.f);
      else if (g.epi == EPI_TANH) v = tanhf(v);
      else if (g.epi == EPI_DRELU) v = (aux[m * g.ldaux + n] > 0.f) ? v : 0.f;
      else if (g.epi == EPI_DTANH) { const float y = aux[m * g.ldaux + n]; v *= (1.f - y * y); }
      *c = g.accumulate ? *c + v : v;
    }
  }
  if (want_rsum && tid < BM && m0 + tid < g.M) {
    float* r = g.rsum + net * g.strideRsum + m0 + tid;
    if (ksplit > 1) atomicAdd(r, rs);
    else *r = g.accumulate ? *r + rs : rs;
  }
}

// zero C (and rsum) ahead of a split-K launch that does not accumulate
__global__ void bgemm_zero_kernel(const BG g) {
  const int net = blockIdx.z;
  float* C = g.C + net * g.strideC;
  const long long total = (long long)g.M * g.N;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x)
    C[(i / g.N) * g.ldc + (i % g.N)] = 0.f;
  if (g.rsum && blockIdx.x == 0)
    for (int m = threadIdx.x; m < g.M; m += blockDim.x) g.rsum[net * g.strideRsum + m] = 0.f;
}

}  // namespace

extern "C" int b200rl_bgemm(const float* A, long long sam, long long sak, long long strideA, const float* B,
                            long long sbk, long long sbn, long long strideB, float* C, long long ldc, long long strideC,
                            const float* bias, long long strideBias, const float* aux, long long ldaux,
                            long long strideAux, float* rsum, long long strideRsum, int M, int N, int K, int nets,
                            int epilogue, int accumulate, cudaStream_t st) {
  RL_CHECK_ARG(A && B && C, "null pointer");
  RL_CHECK_ARG(M > 0 && N > 0 && K > 0 && nets > 0, "bad dims");
  RL_CHECK_ARG(epilogue >= EPI_NONE && epilogue <= EPI_DTANH, "unknown epilogue");
  RL_CHECK_ARG(epilogue < EPI_DRELU || aux, "derivative epilogue needs the saved activation");
  BG g{A, sam, sak, strideA, B, sbk, sbn, strideB, C, ldc, strideC, bias, strideBias, aux, ldaux, strideAux,
       rsum, strideRsum, M, N, K, epilogue, accumulate};
  // tile shape: wide tiles once they fill the machine, narrow N for thin outputs (conv1: N = 32), else 32x32
  const long long tiles64 = (long long)((M + 63) / 64) * ((N + 63) / 64) * nets;
  int BMv = 32, BNv = 32;
  if (N <= 32 && (long long)((M + 63) / 64) * nets >= kNumSMs) { BMv = 64; BNv = 32; }
  else if (tiles64 >= kNumSMs) { BMv = 64; BNv = 64; }
  constexpr int BK = 32;
  const int tx = (N + BNv - 1) / BNv, ty = (M + BMv - 1) / BMv;
  const long long tiles = (long long)tx * ty * nets;
  // split-K: only for plain products (weight gradients) whose output tiles cannot fill the SMs
  int ksplit = 1;
  if (epilogue == EPI_NONE && !bias && tiles < kNumSMs && K >= 8 * BK) {
    ksplit = (int)((4LL * kNumSMs + tiles - 1) / tiles);
    if (ksplit > K / (2 * BK)) ksplit = K / (2 * BK);
    if (ksplit > 128) ksplit = 128;
    if (ksplit < 1) ksplit = 1;
  }
  int kper = ((K + ksplit - 1) / ksplit + BK - 1) / BK * BK;
  ksplit = (K + kper - 1) / kper;
  RL_CHECK_ARG((long long)nets * ksplit <= 65535, "too many networks x K-splits for grid.z");
  if (ksplit > 1 && !accumulate) {
    const long long total = (long long)M * N;
    int zb = (int)((total + 255) / 256);
    if (zb > 64) zb = 64;
    bgemm_zero_kernel<<<dim3(zb, 1, nets), 256, 0, st>>>(g);
  }
  dim3 grid(tx, ty, nets * ksplit);
  if (BMv == 64 && BNv == 64) bgemm_kernel<64, 64, 4, 4, BK><<<grid, 256, 0, st>>>(g, ksplit, kper);
  else if (BMv == 64) bgemm_kernel<64, 32, 4, 2, BK><<<grid, 256, 0, st>>>(g, ksplit, kper);
  else bgemm_kernel<32, 32, 2, 2, BK><<<grid, 256, 0, st>>>(g, ksplit, kper);
  RL_CHECK_LAUNCH();
  return B200RL_OK;
}
