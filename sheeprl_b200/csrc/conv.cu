// Stride-2, kernel-4, padding-1 convolutions on channel-last images (fp32 SIMT implicit GEMM).
//
// All of Dreamer-V3's image layers are this one geometry (agent.py:78-91 encoder Conv2d k4 s2 p1,
// agent.py:199-222 decoder ConvTranspose2d k4 s2 p1).  With weights kept in the reference layouts
//   Conv2d          W[Cout, Cin, 4, 4]   (Cout = small-image channels, Cin = big-image channels)
//   ConvTranspose2d W[Cin, Cout, 4, 4]   (Cin  = small-image channels, Cout = big-image channels)
// i.e. always W[Cs, Cb, ky, kx], three kernels cover forward and backward of both layer kinds:
//   down : small[n,y,x,cs]  = sum_{ky,kx,cb} big[n,2y-1+ky,2x-1+kx,cb] * W[cs,cb,ky,kx]
//          (Conv2d forward; ConvTranspose2d backward-data)
//   up   : big[n,Y,X,cb]    = sum_{cs,(y,ky):2y-1+ky=Y,(x,kx):2x-1+kx=X} small[n,y,x,cs] * W[cs,cb,ky,kx] (+bias)
//          (ConvTranspose2d forward; Conv2d backward-data) -- 4 output-parity classes, 2x2 taps each
//   wgrad: dW[cs,cb,ky,kx] = sum_{n,y,x} small[n,y,x,cs] * big[n,2y-1+ky,2x-1+kx,cb]
//          (weight gradient of both)
// plus the uint8/float NCHW -> normalised NHWC input conversion (dreamer_v3.py:98) and batched transposes.
#include "common.cuh"

namespace {

constexpr int MODE_DOWN = 0, MODE_UP = 1;

// Implicit GEMM: rows = pixels of the small-image grid (per parity class for UP), cols = output channels.
template <int MODE, int BN, int TN>
__global__ void __launch_bounds__(256)
conv_igemm_kernel(const float* __restrict__ In, const float* __restrict__ W, float* __restrict__ Out,
                  const float* __restrict__ bias, int NB, int h, int w, int Cs, int Cb) {
  constexpr int BM = 128, BK = 16, TM = 8, PAD = 4;
  constexpr int NT = (BM / TM) * (BN / TN);
  static_assert(NT == 256, "256 threads expected");
  constexpr int CCH = (TN >= 4) ? 4 : TN, NCC = TN / CCH;
  constexpr int LB = (BN * BK) / NT;
  __shared__ __align__(16) float As[BK][BM + PAD];
  __shared__ __align__(16) float Bs[BK][BN + PAD];

  const int tid = threadIdx.x;
  const int tx = tid % (BN / TN), ty = tid / (BN / TN);
  const long long Mtot = (long long)NB * h * w;
  const long long m0 = (long long)blockIdx.y * BM;
  const int n0 = blockIdx.x * BN;
  const int py = (MODE == MODE_UP) ? (blockIdx.z >> 1) : 0, px = (MODE == MODE_UP) ? (blockIdx.z & 1) : 0;
  const int Cin = (MODE == MODE_DOWN) ? Cb : Cs;    // channels of the gathered image
  const int Cout = (MODE == MODE_DOWN) ? Cs : Cb;
  const int K = (MODE == MODE_DOWN) ? 16 * Cb : 4 * Cs;
  const int Hin = (MODE == MODE_DOWN) ? 2 * h : h, Win = (MODE == MODE_DOWN) ? 2 * w : w;

  // A loader: this thread gathers 8 consecutive k for row (m0 + tid%128)
  const int a_mm = tid % BM, a_kh = tid / BM;
  const long long a_m = m0 + a_mm;
  const bool a_row_ok = a_m < Mtot;
  int a_n = 0, a_y = 0, a_x = 0;
  if (a_row_ok) {
    a_x = (int)(a_m % w);
    const long long t = a_m / w;
    a_y = (int)(t % h);
    a_n = (int)(t / h);
  }
  const bool fast = (Cin % 8) == 0;

  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;
  float ra[8], rb[LB];

  auto src_offset = [&](int tap, bool& ok) -> long long {
    int yy, xx;
    if (MODE == MODE_DOWN) {
      yy = 2 * a_y - 1 + (tap >> 2);
      xx = 2 * a_x - 1 + (tap & 3);
    } else {
      yy = a_y + py - (tap >> 1);
      xx = a_x + px - (tap & 1);
    }
    ok = a_row_ok && yy >= 0 && yy < Hin && xx >= 0 && xx < Win;
    return (((long long)a_n * Hin + yy) * Win + xx) * Cin;
  };
  auto w_index = [&](int k, int col) -> long long {
    const int tap = k / Cin, ch = k - tap * Cin;
    if (MODE == MODE_DOWN) return ((long long)col * Cb + ch) * 16 + tap;  // W[cs=col][cb=ch][tap]
    const int ky = (1 - py) + 2 * (tap >> 1), kx = (1 - px) + 2 * (tap & 1);
    return ((long long)ch * Cb + col) * 16 + ky * 4 + kx;                 // W[cs=ch][cb=col][ky][kx]
  };

  auto load_tiles = [&](int k0) {
    const int kb = k0 + a_kh * 8;
    if (fast) {
      if (kb < K) {
        const int tap = kb / Cin, ch = kb - tap * Cin;
        bool ok;
        const long long off = src_offset(tap, ok);
        if (ok) {
          const float4 v0 = *reinterpret_cast<const float4*>(In + off + ch);
          const float4 v1 = *reinterpret_cast<const float4*>(In + off + ch + 4);
          ra[0] = v0.x; ra[1] = v0.y; ra[2] = v0.z; ra[3] = v0.w;
          ra[4] = v1.x; ra[5] = v1.y; ra[6] = v1.z; ra[7] = v1.w;
        } else {
#pragma unroll
          for (int q = 0; q < 8; ++q) ra[q] = 0.f;
        }
      } else {
#pragma unroll
        for (int q = 0; q < 8; ++q) ra[q] = 0.f;
      }
    } else {
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        const int k = kb + q;
        float v = 0.f;
        if (k < K) {
          const int tap = k / Cin, ch = k - tap * Cin;
          bool ok;
          const long long off = src_offset(tap, ok);
          if (ok) v = In[off + ch];
        }
        ra[q] = v;
      }
    }
#pragma unroll
    for (int l = 0; l < LB; ++l) {
      const int e = tid + l * NT;
      const int nn = e % BN, kk = e / BN;
      const int k = k0 + kk, col = n0 + nn;
      rb[l] = (k < K && col < Cout) ? W[w_index(k, col)] : 0.f;
    }
  };
  auto store_tiles = [&]() {
#pragma unroll
    for (int q = 0; q < 8; ++q) As[a_kh * 8 + q][a_mm] = ra[q];
#pragma unroll
    for (int l = 0; l < LB; ++l) {
      const int e = tid + l * NT;
      Bs[e / BN][e % BN] = rb[l];
    }
  };

  load_tiles(0);
  for (int k0 = 0; k0 < K; k0 += BK) {
    store_tiles();
    __syncthreads();
    if (k0 + BK < K) load_tiles(k0 + BK);
#pragma unroll
    for (int kk = 0; kk < BK; ++kk) {
      float a[TM], b[TN];
#pragma unroll
      for (int c = 0; c < 2; ++c)
#pragma unroll
        for (int i = 0; i < 4; ++i) a[c * 4 + i] = As[kk][c * 64 + ty * 4 + i];
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

#pragma unroll
  for (int i = 0; i < TM; ++i) {
    const long long gm = m0 + (i / 4) * 64 + ty * 4 + (i % 4);
    if (gm >= Mtot) continue;
    long long obase;
    if (MODE == MODE_DOWN) {
      obase = gm * Cs;
    } else {
      const int x = (int)(gm % w);
      const long long t = gm / w;
      const int y = (int)(t % h);
      const long long n = t / h;
      obase = ((n * (2 * h) + (2 * y + py)) * (2 * w) + (2 * x + px)) * (long long)Cb;
    }
#pragma unroll
    for (int j = 0; j < TN; ++j) {
      const int gn = n0 + (j / CCH) * (BN / NCC) + tx * CCH + (j % CCH);
      if (gn >= Cout) continue;
      float v = acc[i][j];
      if (MODE == MODE_UP && bias) v += bias[gn];
      Out[obase + gn] = v;
    }
  }
}

// dW[cs,cb,tap] += sum_m small[m,cs] * big[row(m,tap),cb]; 64x64 (cs x cb) tiles, 16 pixel rows per k-step.
__global__ void __launch_bounds__(256)
conv_wgrad_kernel(const float* __restrict__ Small, const float* __restrict__ Big, float* __restrict__ dW, int NB,
                  int h, int w, int Cs, int Cb, long long rows_per_split) {
  constexpr int BT = 64, BK = 16, PAD = 4;
  __shared__ __align__(16) float As[BK][BT + PAD];
  __shared__ __align__(16) float Bs[BK][BT + PAD];
  const int tid = threadIdx.x;
  const int tx = tid % 16, ty = tid / 16;
  const int cs0 = blockIdx.y * BT, cb0 = blockIdx.x * BT;
  const int tap = blockIdx.z % 16, split = blockIdx.z / 16;
  const int ky = tap >> 2, kx = tap & 3;
  const long long Mtot = (long long)NB * h * w;
  const long long mbeg = (long long)split * rows_per_split;
  const long long mend = min(Mtot, mbeg + rows_per_split);
  const int Hb = 2 * h, Wb = 2 * w;

  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  float ra[4], rb[4];
  const int l_c = tid % BT, l_k = tid / BT;  // this thread loads channel l_c of rows l_k, l_k+4, l_k+8, l_k+12

  auto load_tiles = [&](long long mb) {
#pragma unroll
    for (int l = 0; l < 4; ++l) {
      const long long m = mb + l_k + 4 * l;
      float va = 0.f, vb = 0.f;
      if (m < mend) {
        if (cs0 + l_c < Cs) va = Small[m * Cs + cs0 + l_c];
        const int x = (int)(m % w);
        const long long t = m / w;
        const int y = (int)(t % h);
        const long long n = t / h;
        const int yy = 2 * y - 1 + ky, xx = 2 * x - 1 + kx;
        if (yy >= 0 && yy < Hb && xx >= 0 && xx < Wb && cb0 + l_c < Cb)
          vb = Big[((n * Hb + yy) * Wb + xx) * (long long)Cb + cb0 + l_c];
      }
      ra[l] = va;
      rb[l] = vb;
    }
  };

  if (mbeg < mend) {
    load_tiles(mbeg);
    for (long long mb = mbeg; mb < mend; mb += BK) {
#pragma unroll
      for (int l = 0; l < 4; ++l) {
        As[l_k + 4 * l][l_c] = ra[l];
        Bs[l_k + 4 * l][l_c] = rb[l];
      }
      __syncthreads();
      if (mb + BK < mend) load_tiles(mb + BK);
#pragma unroll
      for (int kk = 0; kk < BK; ++kk) {
        const float4 a = *reinterpret_cast<const float4*>(&As[kk][ty * 4]);
        const float4 b = *reinterpret_cast<const float4*>(&Bs[kk][tx * 4]);
        const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
      }
      __syncthreads();
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int cs = cs0 + ty * 4 + i;
    if (cs >= Cs) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int cb = cb0 + tx * 4 + j;
      if (cb >= Cb) continue;
      atomicAdd(&dW[((long long)cs * Cb + cb) * 16 + tap], acc[i][j]);
    }
  }
}

// Weight gradient when the big image has very few channels (RGB input / output layers): all 16*CB
// (tap, channel) columns of a pixel are staged once and shared by every small-image channel.
template <int CB>
__global__ void __launch_bounds__(256)
conv_wgrad_smallcb_kernel(const float* __restrict__ Small, const float* __restrict__ Big, float* __restrict__ dW,
                          int NB, int h, int w, int Cs, long long rows_per_block) {
  constexpr int RB = 32, Q = 16 * CB, MAXACC = 24;
  extern __shared__ float sm[];
  float* S = sm;            // [RB][Cs]
  float* P = sm + RB * Cs;  // [RB][Q]
  const int tid = threadIdx.x;
  const long long Mtot = (long long)NB * h * w;
  const long long mbeg = (long long)blockIdx.x * rows_per_block;
  const long long mend = min(Mtot, mbeg + rows_per_block);
  const int Hb = 2 * h, Wb = 2 * w;
  const int nout = Cs * Q;
  float acc[MAXACC];
#pragma unroll
  for (int i = 0; i < MAXACC; ++i) acc[i] = 0.f;
  for (long long mb = mbeg; mb < mend; mb += RB) {
    const int rows = (int)min((long long)RB, mend - mb);
    for (int e = tid; e < RB * Cs; e += 256) {
      const int r = e / Cs;
      S[e] = (r < rows) ? Small[(mb + r) * Cs + (e - r * Cs)] : 0.f;
    }
    for (int e = tid; e < RB * Q; e += 256) {
      const int r = e / Q, q = e - r * Q;
      float v = 0.f;
      if (r < rows) {
        const long long m = mb + r;
        const int tap = q / CB, c = q - tap * CB;
        const int x = (int)(m % w);
        const long long t = m / w;
        const int y = (int)(t % h);
        const long long n = t / h;
        const int yy = 2 * y - 1 + (tap >> 2), xx = 2 * x - 1 + (tap & 3);
        if (yy >= 0 && yy < Hb && xx >= 0 && xx < Wb) v = Big[((n * Hb + yy) * Wb + xx) * (long long)CB + c];
      }
      P[e] = v;
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < MAXACC; ++i) {
      const int o = tid + i * 256;
      if (o < nout) {
        const int cs = o % Cs, q = o / Cs;
        float a = acc[i];
        for (int r = 0; r < RB; ++r) a = fmaf(S[r * Cs + cs], P[r * Q + q], a);
        acc[i] = a;
      }
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < MAXACC; ++i) {
    const int o = tid + i * 256;
    if (o < nout) {
      const int cs = o % Cs, q = o / Cs;
      const int tap = q / CB, c = q - tap * CB;
      atomicAdd(&dW[((long long)cs * CB + c) * 16 + tap], acc[i]);
    }
  }
}

template <typename T>
__global__ void obs_prep_kernel(const T* __restrict__ obs, float* __restrict__ out, long long NB, int C, int HW) {
  // out[n, p, c] = obs[n, c, p] / 255 - 0.5 ; one thread per output element (writes coalesced)
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long tot = NB * C * HW;
  if (idx >= tot) return;
  const int c = (int)(idx % C);
  const long long t = idx / C;
  const int p = (int)(t % HW);
  const long long n = t / HW;
  out[idx] = (float)obs[(n * C + c) * HW + p] / 255.0f - 0.5f;
}

// Same result, one thread per 4 consecutive pixels of one image and all C channels: 32-bit loads per channel plane
// (uint8) / 128-bit (float), 4*C contiguous floats written as C 128-bit stores, no per-element 64-bit div/mod.
template <typename T, int C>
__global__ void __launch_bounds__(256) obs_prep_vec_kernel(const T* __restrict__ obs, float* __restrict__ out, int HW) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;        // quad of pixels inside image blockIdx.y
  if (q * 4 >= HW) return;
  const long long n = blockIdx.y;
  const int p = q * 4;
  float v[4 * C];
#pragma unroll
  for (int c = 0; c < C; ++c) {
    const T* src = obs + (n * C + c) * (long long)HW + p;
    float x0, x1, x2, x3;
    if constexpr (sizeof(T) == 1) {
      const uchar4 u = *reinterpret_cast<const uchar4*>(src);
      x0 = (float)u.x; x1 = (float)u.y; x2 = (float)u.z; x3 = (float)u.w;
    } else {
      const float4 u = *reinterpret_cast<const float4*>(src);
      x0 = u.x; x1 = u.y; x2 = u.z; x3 = u.w;
    }
    v[0 * C + c] = x0 / 255.0f - 0.5f;
    v[1 * C + c] = x1 / 255.0f - 0.5f;
    v[2 * C + c] = x2 / 255.0f - 0.5f;
    v[3 * C + c] = x3 / 255.0f - 0.5f;
  }
  float4* dst = reinterpret_cast<float4*>(out + (n * HW + p) * (long long)C);
#pragma unroll
  for (int i = 0; i < C; ++i) dst[i] = make_float4(v[4 * i], v[4 * i + 1], v[4 * i + 2], v[4 * i + 3]);
}

template <typename T>
bool launch_obs_prep_vec(const T* obs, float* out, long long NB, int C, int HW, cudaStream_t st) {
  const size_t in_align = sizeof(T) == 1 ? 3 : 15;
  if (HW % 4 || NB > 65535 || (reinterpret_cast<uintptr_t>(obs) & in_align) || (reinterpret_cast<uintptr_t>(out) & 15)) return false;
  const dim3 grid(ceil_div(HW / 4, 256), (unsigned)NB);
  switch (C) {
    case 1: obs_prep_vec_kernel<T, 1><<<grid, 256, 0, st>>>(obs, out, HW); return true;
    case 3: obs_prep_vec_kernel<T, 3><<<grid, 256, 0, st>>>(obs, out, HW); return true;
    case 4: obs_prep_vec_kernel<T, 4><<<grid, 256, 0, st>>>(obs, out, HW); return true;
    case 12: obs_prep_vec_kernel<T, 12><<<grid, 256, 0, st>>>(obs, out, HW); return true;
    default: return false;
  }
}

// Y[n, j, i] = X[n, i, j]; X [NB, a, b]; 32x32 smem tiles
__global__ void transpose_batched_kernel(const float* __restrict__ X, float* __restrict__ Y, int a, int b) {
  __shared__ float tile[32][33];
  const long long n = blockIdx.z;
  const float* x = X + n * (long long)a * b;
  float* y = Y + n * (long long)a * b;
  const int i0 = blockIdx.y * 32, j0 = blockIdx.x * 32;
  for (int r = threadIdx.y; r < 32; r += 8) {
    const int i = i0 + r, j = j0 + threadIdx.x;
    if (i < a && j < b) tile[r][threadIdx.x] = x[(long long)i * b + j];
  }
  __syncthreads();
  for (int r = threadIdx.y; r < 32; r += 8) {
    const int j = j0 + r, i = i0 + threadIdx.x;
    if (i < a && j < b) y[(long long)j * a + i] = tile[threadIdx.x][r];
  }
}

// Y[j*ldy + i] = X[i*ldx + j]; X [rows][cols] with row stride ldx; 32x32 smem tiles
__global__ void transpose2d_kernel(const float* __restrict__ X, float* __restrict__ Y, int rows, int cols,
                                   long long ldx, long long ldy) {
  __shared__ float tile[32][33];
  const int i0 = blockIdx.y * 32, j0 = blockIdx.x * 32;
  for (int r = threadIdx.y; r < 32; r += 8) {
    const int i = i0 + r, j = j0 + threadIdx.x;
    if (i < rows && j < cols) tile[r][threadIdx.x] = X[(long long)i * ldx + j];
  }
  __syncthreads();
  for (int r = threadIdx.y; r < 32; r += 8) {
    const int j = j0 + r, i = i0 + threadIdx.x;
    if (i < rows && j < cols) Y[(long long)j * ldy + i] = tile[threadIdx.x][r];
  }
}

// Transposed im2col for the weight-gradient GEMM: out[(tap*Cb + cb)][pix] = big[n, 2y-1+ky, 2x-1+kx, cb] (0 outside).
// One block = 128 pixels x 32 channels of one tap: 128-byte channel reads, smem transpose, 512-byte pixel runs written
// as float4 (the matrix is 4x the activation it is gathered from, so the write side is what has to be wide).
__global__ void __launch_bounds__(256)
im2col_t_kernel(const float* __restrict__ Big, float* __restrict__ out, int NB, int h, int w, int Cb, long long ldo) {
  constexpr int PT = 128;
  __shared__ __align__(16) float tile[32][PT + 4];
  __shared__ long long src[PT];                     // source pixel offset (in pixels) or -1 outside the image
  const int tap = blockIdx.z, ky = tap >> 2, kx = tap & 3;
  const long long p0 = (long long)blockIdx.x * PT;
  const int c0 = blockIdx.y * 32;
  const long long P = (long long)NB * h * w;
  const int Hb = 2 * h, Wb = 2 * w;
  const int c = c0 + threadIdx.x;
  // the (n, y, x) decomposition costs two 64-bit divisions: do it once per pixel, not once per element
  const int tid = threadIdx.y * 32 + threadIdx.x;
  if (tid < PT) {
    const long long p = p0 + tid;
    long long off = -1;
    if (p < P) {
      const int x = (int)(p % w);
      const long long t = p / w;
      const int y = (int)(t % h);
      const long long n = t / h;
      const int yy = 2 * y - 1 + ky, xx = 2 * x - 1 + kx;
      if (yy >= 0 && yy < Hb && xx >= 0 && xx < Wb) off = (n * Hb + yy) * Wb + xx;
    }
    src[tid] = off;
  }
  __syncthreads();
#pragma unroll 4
  for (int r = threadIdx.y; r < PT; r += 8) {
    const long long off = src[r];
    tile[threadIdx.x][r] = (off >= 0 && c < Cb) ? __ldg(Big + off * Cb + c) : 0.f;
  }
  __syncthreads();
  // 32 channel rows x 32 float4 per row: warp ty writes rows ty, ty+8, ...
  for (int r = threadIdx.y; r < 32; r += 8) {
    const int cc = c0 + r;
    const long long p = p0 + 4 * threadIdx.x;
    if (cc >= Cb || p >= P) continue;
    float* dst = out + ((long long)tap * Cb + cc) * ldo + p;
    const float4 v = *reinterpret_cast<const float4*>(&tile[r][4 * threadIdx.x]);
    if (p + 3 < P) *reinterpret_cast<float4*>(dst) = v;
    else {
      dst[0] = v.x;
      if (p + 1 < P) dst[1] = v.y;
      if (p + 2 < P) dst[2] = v.z;
    }
  }
}

// dW[cs][cb][tap] = G[tap*Cb + cb][cs]
__global__ void wgrad_unpack_kernel(const float* __restrict__ G, float* __restrict__ dW, int Cs, int Cb, int accumulate) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)Cs * Cb * 16) return;
  const int tap = (int)(idx % 16);
  const int cb = (int)((idx / 16) % Cb);
  const int cs = (int)(idx / (16LL * Cb));
  const float v = G[((long long)tap * Cb + cb) * Cs + cs];
  dW[idx] = accumulate ? dW[idx] + v : v;
}

}  // namespace

extern "C" int b200rl_gemm_tc(const float* A, const float* B, float* C, const float* bias, int M, int N, int K, int lda,
                              int ldb, int ldc, int transA, int transB, int accumulate, cudaStream_t st);

// Weight gradient on the tensor cores: dW = small^T (x) im2col(big) as ONE K-major GEMM with K = all pixels.
// workspace: (Cs + 16*Cb) * Ppad + 16*Cs*Cb floats, Ppad = pixels rounded up to 4.
extern "C" int b200rl_conv_wgrad_mn_supported(int NB, int h, int w, int Cs, int Cb);
extern "C" long long b200rl_conv_wgrad_tc_workspace(int NB, int h, int w, int Cs, int Cb) {
  if (b200rl_conv_wgrad_mn_supported(NB, h, w, Cs, Cb)) return 16LL * Cs * Cb;   // only the [16*Cb][Cs] result
  const long long P = ((long long)NB * h * w + 3) / 4 * 4;
  return (Cs + 16LL * Cb) * P + 16LL * Cs * Cb;
}
extern "C" int b200rl_conv_wgrad_mn(const float* small_, const float* big, float* G, int NB, int h, int w, int Cs, int Cb,
                                    cudaStream_t st);

extern "C" int b200rl_conv_wgrad_tc_supported(int NB, int h, int w, int Cs, int Cb) {
  const long long P = (long long)NB * h * w;
  return P >= 1024 && P <= 2000000000LL && Cs >= 48 && Cb >= 8;
}

extern "C" int b200rl_conv_wgrad_tc(const float* small_, const float* big, float* dW, float* workspace, int NB, int h,
                                    int w, int Cs, int Cb, int accumulate, cudaStream_t st) {
  RL_CHECK_ARG(small_ && big && dW && workspace, "null pointer");
  RL_CHECK_ARG(b200rl_conv_wgrad_tc_supported(NB, h, w, Cs, Cb), "shape not eligible for the tensor-core wgrad path");
  const long long P = (long long)NB * h * w, Pp = (P + 3) / 4 * 4;
  if (b200rl_conv_wgrad_mn_supported(NB, h, w, Cs, Cb)) {
    // operands read in place: the gathered big image and the small image are both MN-major tiles
    float* G = workspace;                      // [16*Cb][Cs]
    if (int rc = b200rl_conv_wgrad_mn(small_, big, G, NB, h, w, Cs, Cb, st)) return rc;
    wgrad_unpack_kernel<<<ceil_div(16LL * Cs * Cb, 256), 256, 0, st>>>(G, dW, Cs, Cb, accumulate);
    RL_CHECK_LAUNCH();
    return B200RL_OK;
  }
  float* St = workspace;                       // [Cs][Pp]
  float* Bt = workspace + (long long)Cs * Pp;  // [16*Cb][Pp]
  float* G = Bt + 16LL * Cb * Pp;              // [16*Cb][Cs]
  RL_CHECK_ARG(ceil_div(P, 32) <= 2147483647LL && ceil_div(Cb, 32) <= 65535, "grid too large");
  // small [P][Cs] -> St [Cs][Pp]
  {
    const long long rows = P;
    for (long long r0 = 0; r0 < rows; r0 += 32LL * 65535) {   // transpose2d launches are limited to 65535 row tiles
      const int nr = (int)min((long long)32 * 65535, rows - r0);
      transpose2d_kernel<<<dim3(ceil_div(Cs, 32), ceil_div(nr, 32)), dim3(32, 8), 0, st>>>(small_ + r0 * Cs, St + r0, nr, Cs, Cs, Pp);
    }
  }
  im2col_t_kernel<<<dim3((unsigned)ceil_div(P, 128), ceil_div(Cb, 32), 16), dim3(32, 8), 0, st>>>(big, Bt, NB, h, w, Cb, Pp);
  RL_CHECK_LAUNCH();
  // rows = (tap, cb) (>= 128), columns = cs: G = im2col^T . small
  if (int rc = b200rl_gemm_tc(Bt, St, G, nullptr, 16 * Cb, Cs, (int)P, (int)Pp, (int)Pp, Cs, 0, 1, 0, st)) return rc;
  wgrad_unpack_kernel<<<ceil_div(16LL * Cs * Cb, 256), 256, 0, st>>>(G, dW, Cs, Cb, accumulate);
  RL_CHECK_LAUNCH();
  return B200RL_OK;
}

extern "C" int b200rl_transpose2d(const float* X, float* Y, int rows, int cols, long long ldx, long long ldy,
                                  cudaStream_t st) {
  RL_CHECK_ARG(X && Y, "null pointer");
  if (rows <= 0 || cols <= 0) return B200RL_OK;
  RL_CHECK_ARG(ldx >= cols && ldy >= rows, "leading dimension too small");
  RL_CHECK_ARG(ceil_div(rows, 32) <= 65535, "too many rows for one launch");
  transpose2d_kernel<<<dim3(ceil_div(cols, 32), ceil_div(rows, 32)), dim3(32, 8), 0, st>>>(X, Y, rows, cols, ldx, ldy);
  RL_CHECK_LAUNCH();
  return B200RL_OK;
}

// thin-channel specialisations (conv_thin.cu)
extern "C" int b200rl_thin_up_supported(int Cs, int Cb);
extern "C" int b200rl_thin_wgrad_supported(int Cs, int Cb);
extern "C" int b200rl_thin_down_supported(int w, int Cs, int Cb);
int b200rl_conv_down_thin(const float* big, const float* W, float* small, int NB, int h, int w, int Cs, int Cb, cudaStream_t st);
int b200rl_conv_up_thin(const float* small, const float* W, float* big, const float* bias, int NB, int h, int w, int Cs,
                        int Cb, cudaStream_t st);
int b200rl_conv_wgrad_thin(const float* small, const float* big, float* dW, int NB, int h, int w, int Cs, int Cb,
                           cudaStream_t st);

extern "C" int b200rl_conv_down(const float* big, const float* W, float* small, int NB, int h, int w, int Cs, int Cb,
                                cudaStream_t st) {
  RL_CHECK_ARG(big && W && small, "null pointer");
  RL_CHECK_ARG(NB > 0 && h > 0 && w > 0 && Cs > 0 && Cb > 0, "bad dims");
  if (b200rl_thin_down_supported(w, Cs, Cb)) return b200rl_conv_down_thin(big, W, small, NB, h, w, Cs, Cb, st);
  const long long Mtot = (long long)NB * h * w;
  const int gm = ceil_div(Mtot, 128);
  if (Cs <= 32)
    conv_igemm_kernel<MODE_DOWN, 32, 2><<<dim3(ceil_div(Cs, 32), gm, 1), 256, 0, st>>>(big, W, small, nullptr, NB, h, w, Cs, Cb);
  else if (Cs <= 64)
    conv_igemm_kernel<MODE_DOWN, 64, 4><<<dim3(ceil_div(Cs, 64), gm, 1), 256, 0, st>>>(big, W, small, nullptr, NB, h, w, Cs, Cb);
  else
    conv_igemm_kernel<MODE_DOWN, 128, 8><<<dim3(ceil_div(Cs, 128), gm, 1), 256, 0, st>>>(big, W, small, nullptr, NB, h, w, Cs, Cb);
  RL_CHECK_LAUNCH();
  return B200RL_OK;
}

extern "C" int b200rl_conv_up(const float* small, const float* W, float* big, const float* bias, int NB, int h, int w,
                              int Cs, int Cb, cudaStream_t st) {
  RL_CHECK_ARG(big && W && small, "null pointer");
  RL_CHECK_ARG(NB > 0 && h > 0 && w > 0 && Cs > 0 && Cb > 0, "bad dims");
  if (b200rl_thin_up_supported(Cs, Cb)) return b200rl_conv_up_thin(small, W, big, bias, NB, h, w, Cs, Cb, st);
  const long long Mtot = (long long)NB * h * w;
  const int gm = ceil_div(Mtot, 128);
  if (Cb <= 32)
    conv_igemm_kernel<MODE_UP, 32, 2><<<dim3(ceil_div(Cb, 32), gm, 4), 256, 0, st>>>(small, W, big, bias, NB, h, w, Cs, Cb);
  else if (Cb <= 64)
    conv_igemm_kernel<MODE_UP, 64, 4><<<dim3(ceil_div(Cb, 64), gm, 4), 256, 0, st>>>(small, W, big, bias, NB, h, w, Cs, Cb);
  else
    conv_igemm_kernel<MODE_UP, 128, 8><<<dim3(ceil_div(Cb, 128), gm, 4), 256, 0, st>>>(small, W, big, bias, NB, h, w, Cs, Cb);
  RL_CHECK_LAUNCH();
  return B200RL_OK;
}

extern "C" int b200rl_conv_wgrad(const float* small, const float* big, float* dW, int NB, int h, int w, int Cs, int Cb,
                                 int accumulate, cudaStream_t st) {
  RL_CHECK_ARG(big && dW && small, "null pointer");
  RL_CHECK_ARG(NB > 0 && h > 0 && w > 0 && Cs > 0 && Cb > 0, "bad dims");
  if (!accumulate) RL_CUDA(cudaMemsetAsync(dW, 0, sizeof(float) * (size_t)Cs * Cb * 16, st));
  if (b200rl_thin_wgrad_supported(Cs, Cb)) return b200rl_conv_wgrad_thin(small, big, dW, NB, h, w, Cs, Cb, st);
  const long long Mtot = (long long)NB * h * w;
  if (Cb <= 4 && Cs * 16 * Cb <= 24 * 256) {
    long long blocks = min((long long)4 * kNumSMs, (Mtot + 31) / 32);
    long long rpb = ((Mtot + blocks - 1) / blocks + 31) / 32 * 32;
    blocks = (Mtot + rpb - 1) / rpb;
    const size_t smem = sizeof(float) * 32 * (Cs + 16 * Cb);
    switch (Cb) {
      case 1: conv_wgrad_smallcb_kernel<1><<<(unsigned)blocks, 256, smem, st>>>(small, big, dW, NB, h, w, Cs, rpb); break;
      case 2: conv_wgrad_smallcb_kernel<2><<<(unsigned)blocks, 256, smem, st>>>(small, big, dW, NB, h, w, Cs, rpb); break;
      case 3: conv_wgrad_smallcb_kernel<3><<<(unsigned)blocks, 256, smem, st>>>(small, big, dW, NB, h, w, Cs, rpb); break;
      default: conv_wgrad_smallcb_kernel<4><<<(unsigned)blocks, 256, smem, st>>>(small, big, dW, NB, h, w, Cs, rpb); break;
    }
    RL_CHECK_LAUNCH();
    return B200RL_OK;
  }
  const int tcs = ceil_div(Cs, 64), tcb = ceil_div(Cb, 64);
  const int base = tcs * tcb * 16;
  long long splits = max(1LL, min((long long)ceil_div(4 * kNumSMs, base), Mtot / 256));
  long long rps = ((Mtot + splits - 1) / splits + 15) / 16 * 16;
  splits = (Mtot + rps - 1) / rps;
  conv_wgrad_kernel<<<dim3(tcb, tcs, (unsigned)(16 * splits)), 256, 0, st>>>(small, big, dW, NB, h, w, Cs, Cb, rps);
  RL_CHECK_LAUNCH();
  return B200RL_OK;
}

extern "C" int b200rl_obs_prep(const void* obs, int is_uint8, float* out, long long NB, int C, int HW,
                               cudaStream_t st) {
  RL_CHECK_ARG(obs && out, "null pointer");
  const long long tot = NB * C * HW;
  if (tot <= 0) return B200RL_OK;
  const bool vec = is_uint8 ? launch_obs_prep_vec((const unsigned char*)obs, out, NB, C, HW, st)
                            : launch_obs_prep_vec((const float*)obs, out, NB, C, HW, st);
  if (vec) {
    RL_CHECK_LAUNCH();
    return B200RL_OK;
  }
  if (is_uint8)
    obs_prep_kernel<unsigned char><<<ceil_div(tot, 256), 256, 0, st>>>((const unsigned char*)obs, out, NB, C, HW);
  else
    obs_prep_kernel<float><<<ceil_div(tot, 256), 256, 0, st>>>((const float*)obs, out, NB, C, HW);
  RL_CHECK_LAUNCH();
  return B200RL_OK;
}

extern "C" int b200rl_transpose_batched(const float* X, float* Y, int NB, int a, int b, cudaStream_t st) {
  RL_CHECK_ARG(X && Y, "null pointer");
  if (NB <= 0 || a <= 0 || b <= 0) return B200RL_OK;
  RL_CHECK_ARG(NB <= 65535, "batch too large for grid.z");
  transpose_batched_kernel<<<dim3(ceil_div(b, 32), ceil_div(a, 32), NB), dim3(32, 8), 0, st>>>(X, Y, a, b);
  RL_CHECK_LAUNCH();
  return B200RL_OK;
}
