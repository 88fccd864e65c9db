// Image layers whose big-image side has only a few channels (the RGB ends of the Dreamer-V3 encoder / decoder):
//   up_thin   : ConvTranspose2d(Cs -> CB, k4 s2 p1) forward  (decoder output layer, agent.py:199-222)
//   wgrad_thin: weight gradient of Conv2d(CB -> Cs) / ConvTranspose2d(Cs -> CB)  (encoder first / decoder last layer)
// With CB = 3 these are not tensor-core shapes (K or N of 3..48) and they move the two largest activations of the
// model (1024 x 32x32x32 fp32 = 134 MB and the 50 MB image), so they are written as FMA/LDS-balanced SIMT kernels
// that read every activation once with full 128-byte lines:
//   bound: max(HBM: 184 MB / launch, FMA: 1.6 GFMA / launch) (not measured on the H100); the generic implicit-GEMM kernels
//   they replace took 1.5 ms (up) and 0.7 ms (wgrad) per launch.
// Weights keep the reference layout W[Cs][CB][ky][kx] (see conv.cu header for the index conventions).
#include "common.cuh"

namespace {

// ---------------------------------------------------------------------------------------------------------
// up_thin: one thread per small-grid position (i, j) -> the 2x2 output block (2i+a, 2j+b), all CB channels.
// Output (2i+a) takes small rows i+dy with kernel row ky = a - 2dy + 1: dy=-1 -> a=0,ky=3; dy=0 -> a,ky=a+1;
// dy=+1 -> a=1,ky=0 (same along x).  Per neighbour the (a, b, cb) weights are packed contiguously in shared memory
// (padded to a multiple of 4) so one broadcast LDS.128 feeds 4 FMAs.
// ---------------------------------------------------------------------------------------------------------
template <int D> struct Nb { static constexpr int n = (D == 0) ? 2 : 1; static constexpr int a0 = (D == 1) ? 1 : 0; };

template <int CB> __host__ __device__ constexpr int nb_slots(int p) {   // padded weight count of neighbour p = (dy+1)*3+(dx+1)
  const int ny = (p / 3 == 1) ? 2 : 1, nx = (p % 3 == 1) ? 2 : 1;
  return (ny * nx * CB + 3) / 4 * 4;
}
template <int CB> __host__ __device__ constexpr int nb_base(int p) {
  int s = 0;
  for (int q = 0; q < p; ++q) s += nb_slots<CB>(q);
  return s;
}

template <int CB, int CS, int DY, int DX>
__device__ __forceinline__ void up_neighbour(const float* __restrict__ small, const float* __restrict__ Wn, int i, int j,
                                             int h, int w, long long img_base, float (&acc)[2][2][CB]) {
  const int iy = i + DY, ix = j + DX;
  if (iy < 0 || iy >= h || ix < 0 || ix >= w) return;
  constexpr int P = (DY + 1) * 3 + (DX + 1);
  constexpr int NY = Nb<DY>::n, NX = Nb<DX>::n, A0 = Nb<DY>::a0, B0 = Nb<DX>::a0;
  constexpr int CNT = NY * NX * CB, PADDED = nb_slots<CB>(P), BASE = nb_base<CB>(P), WSTRIDE = nb_base<CB>(9);
  const float4* __restrict__ src = reinterpret_cast<const float4*>(small + (img_base + (long long)iy * w + ix) * CS);
#pragma unroll 2
  for (int c4 = 0; c4 < CS / 4; ++c4) {
    const float4 v = __ldg(src + c4);
    const float vs[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const float4* wp = reinterpret_cast<const float4*>(Wn + (c4 * 4 + q) * WSTRIDE + BASE);
      float wv[PADDED];
#pragma unroll
      for (int e = 0; e < PADDED / 4; ++e) {
        const float4 t = wp[e];
        wv[4 * e] = t.x; wv[4 * e + 1] = t.y; wv[4 * e + 2] = t.z; wv[4 * e + 3] = t.w;
      }
#pragma unroll
      for (int s = 0; s < CNT; ++s) {
        const int cb = s % CB, b = (s / CB) % NX, a = s / (CB * NX);
        acc[A0 + a][B0 + b][cb] = fmaf(vs[q], wv[s], acc[A0 + a][B0 + b][cb]);
      }
    }
  }
}

template <int CB, int CS>
__global__ void __launch_bounds__(128)
conv_up_thin_kernel(const float* __restrict__ small, const float* __restrict__ W, const float* __restrict__ bias,
                    float* __restrict__ big, int NB, int h, int w) {
  constexpr int WSTRIDE = nb_base<CB>(9);
  __shared__ __align__(16) float Wn[CS * WSTRIDE];
  for (int e = threadIdx.x; e < CS * WSTRIDE; e += blockDim.x) Wn[e] = 0.f;
  __syncthreads();
  // pack: Wn[cs][base(p) + (a*NX + b)*CB + cb] = W[cs][cb][ky][kx]
  for (int e = threadIdx.x; e < CS * CB * 16; e += blockDim.x) {
    const int tap = e % 16, cb = (e / 16) % CB, cs = e / (16 * CB);
    const int ky = tap >> 2, kx = tap & 3;
    // ky = a - 2dy + 1  ->  (ky=3: dy=-1,a=0) (ky=1: dy=0,a=0) (ky=2: dy=0,a=1) (ky=0: dy=1,a=1)
    const int dy = (ky == 3) ? -1 : ((ky == 0) ? 1 : 0), a = (ky == 2 || ky == 0) ? 1 : 0;
    const int dx = (kx == 3) ? -1 : ((kx == 0) ? 1 : 0), b = (kx == 2 || kx == 0) ? 1 : 0;
    const int p = (dy + 1) * 3 + (dx + 1);
    const int nx = (dx == 0) ? 2 : 1;
    const int la = (dy == 0) ? a : 0, lb = (dx == 0) ? b : 0;     // local index inside the neighbour's (a, b) set
    Wn[cs * WSTRIDE + nb_base<CB>(p) + (la * nx + lb) * CB + cb] = W[e];
  }
  __syncthreads();
  const long long total = (long long)NB * h * w;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
    const int j = (int)(t % w);
    const long long r = t / w;
    const int i = (int)(r % h);
    const long long n = r / h;
    float acc[2][2][CB];
#pragma unroll
    for (int a = 0; a < 2; ++a)
#pragma unroll
      for (int b = 0; b < 2; ++b)
#pragma unroll
        for (int c = 0; c < CB; ++c) acc[a][b][c] = bias ? bias[c] : 0.f;
    const long long img = n * h * w;
    up_neighbour<CB, CS, -1, -1>(small, Wn, i, j, h, w, img, acc);
    up_neighbour<CB, CS, -1, 0>(small, Wn, i, j, h, w, img, acc);
    up_neighbour<CB, CS, -1, 1>(small, Wn, i, j, h, w, img, acc);
    up_neighbour<CB, CS, 0, -1>(small, Wn, i, j, h, w, img, acc);
    up_neighbour<CB, CS, 0, 0>(small, Wn, i, j, h, w, img, acc);
    up_neighbour<CB, CS, 0, 1>(small, Wn, i, j, h, w, img, acc);
    up_neighbour<CB, CS, 1, -1>(small, Wn, i, j, h, w, img, acc);
    up_neighbour<CB, CS, 1, 0>(small, Wn, i, j, h, w, img, acc);
    up_neighbour<CB, CS, 1, 1>(small, Wn, i, j, h, w, img, acc);
    const int Wb = 2 * w;
#pragma unroll
    for (int a = 0; a < 2; ++a) {
      float* dst = big + ((n * 2 * h + 2 * i + a) * Wb + 2 * j) * (long long)CB;   // 2*CB contiguous floats
#pragma unroll
      for (int b = 0; b < 2; ++b)
#pragma unroll
        for (int c = 0; c < CB; ++c) dst[b * CB + c] = acc[a][b][c];
    }
  }
}

// ---------------------------------------------------------------------------------------------------------
// wgrad_thin: dW[cs][cb][ky][kx] += sum over small pixels of small[p][cs] * big[patch(p)][ky][kx][cb].
// CTA tile = up to 32 consecutive small pixels of one image row; the 4 big rows they touch are staged (zero-padded)
// in shared memory, lane = small channel, each warp walks 4 of the pixels: per pixel 1 LDS + 8*CB broadcast LDS.64
// feed 16*CB FMAs on register accumulators; one cross-warp + atomic reduction per CTA at the very end.
// ---------------------------------------------------------------------------------------------------------
template <int CB>
__global__ void __launch_bounds__(256, 2)
conv_wgrad_thin_kernel(const float* __restrict__ small, const float* __restrict__ big, float* __restrict__ dW, int NB,
                       int h, int w, int Cs, int tiles_per_row) {
  constexpr int TX = 32, ROWF = (2 * TX + 2) * CB;              // floats per staged big row (even)
  extern __shared__ __align__(16) float sm[];
  float* Bt = sm;                                                // [4][ROWF]
  float* St = sm + 4 * ROWF;                                     // [TX][Cs]
  float* Red = St + TX * 32;                                     // [16*CB][Cs]
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int groups = Cs / 32;
  const int Hb = 2 * h, Wb = 2 * w;
  const long long ntiles = (long long)NB * h * tiles_per_row;
  for (int e = threadIdx.x; e < 16 * CB * Cs; e += blockDim.x) Red[e] = 0.f;
  for (int g = 0; g < groups; ++g) {
    float acc[4][4 * CB];
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
      for (int b = 0; b < 4 * CB; ++b) acc[a][b] = 0.f;
    // software pipeline: the next tile's global loads are issued into registers before the current tile is consumed
    // (the kernel is otherwise stalled on their latency: 3 CTAs per SM cannot hide it)
    constexpr int NBR = (4 * ROWF + 255) / 256, NSR = TX * 32 / 256;
    float rb[NBR], rs[NSR];
    auto fetch = [&](long long tile) {
      const int tx = (int)(tile % tiles_per_row);
      const long long r = tile / tiles_per_row;
      const int y = (int)(r % h);
      const long long n = r / h;
      const int x0 = tx * TX, npx = min(TX, w - x0);
#pragma unroll
      for (int u = 0; u < NBR; ++u) {
        const int e = threadIdx.x + u * 256;
        float v = 0.f;
        if (e < 4 * ROWF) {
          const int row = e / ROWF, f = e - row * ROWF;
          const int col = f / CB, c = f - col * CB;
          const int yy = 2 * y - 1 + row, xx = 2 * x0 - 1 + col;
          if (yy >= 0 && yy < Hb && xx >= 0 && xx < Wb) v = __ldg(big + ((n * Hb + yy) * Wb + xx) * (long long)CB + c);
        }
        rb[u] = v;
      }
#pragma unroll
      for (int u = 0; u < NSR; ++u) {
        const int e = threadIdx.x + u * 256, p = e >> 5, c = e & 31;
        rs[u] = (p < npx) ? __ldg(small + ((n * h + y) * (long long)w + x0 + p) * Cs + g * 32 + c) : 0.f;
      }
    };
    long long tile = blockIdx.x;
    if (tile < ntiles) fetch(tile);
    for (; tile < ntiles; tile += gridDim.x) {
      __syncthreads();                                         // the previous tile has been consumed
#pragma unroll
      for (int u = 0; u < NBR; ++u) {
        const int e = threadIdx.x + u * 256;
        if (e < 4 * ROWF) Bt[e] = rb[u];
      }
#pragma unroll
      for (int u = 0; u < NSR; ++u) St[threadIdx.x + u * 256] = rs[u];
      __syncthreads();
      if (tile + gridDim.x < ntiles) fetch(tile + gridDim.x);  // in flight while this tile is multiplied
#pragma unroll
      for (int q = 0; q < TX / 8; ++q) {
        const int p = warp + 8 * q;
        const float s = St[p * 32 + lane];
#pragma unroll
        for (int ky = 0; ky < 4; ++ky) {
          const float2* bp = reinterpret_cast<const float2*>(Bt + ky * ROWF + 2 * p * CB);
#pragma unroll
          for (int e = 0; e < 2 * CB; ++e) {
            const float2 b2 = bp[e];
            acc[ky][2 * e] = fmaf(s, b2.x, acc[ky][2 * e]);
            acc[ky][2 * e + 1] = fmaf(s, b2.y, acc[ky][2 * e + 1]);
          }
        }
      }
    }
    // cross-warp reduction in shared memory, then one atomic per output element and CTA
#pragma unroll
    for (int ky = 0; ky < 4; ++ky)
#pragma unroll
      for (int f = 0; f < 4 * CB; ++f) atomicAdd(&Red[(ky * 4 * CB + f) * Cs + g * 32 + lane], acc[ky][f]);
  }
  __syncthreads();
  for (int e = threadIdx.x; e < 16 * CB * Cs; e += blockDim.x) {
    const int cs = e % Cs, q = e / Cs;                      // q = ky*(4*CB) + kx*CB + cb
    const int ky = q / (4 * CB), rem = q - ky * 4 * CB, kx = rem / CB, cb = rem - kx * CB;
    atomicAdd(&dW[((long long)cs * CB + cb) * 16 + ky * 4 + kx], Red[e]);
  }
}


// ---------------------------------------------------------------------------------------------------------
// Paired-FMA versions for 32-wide small grids (the 64x64 images of Dreamer-V3): one warp per pair of small-grid rows,
// lane = column.  The generic kernels above issue ~4 instructions per FMA; here every weight LDS.128 (warp-uniform, one
// wavefront) feeds 8-16 FMAs on 64-bit register pairs and the image rows are staged once per warp in shared memory in a
// conflict-free layout.
// ---------------------------------------------------------------------------------------------------------
typedef unsigned long long u64;
__device__ __forceinline__ float lo32(u64 v) { return __uint_as_float((unsigned)v); }
__device__ __forceinline__ float hi32(u64 v) { return __uint_as_float((unsigned)(v >> 32)); }
__device__ __forceinline__ u64 pack2(float lo, float hi) {
  return ((u64)__float_as_uint(hi) << 32) | (u64)__float_as_uint(lo);
}
// two independent round-to-nearest FMAs on the halves of a register pair
__device__ __forceinline__ void fma2(u64& acc, u64 x, u64 w) {
  acc = pack2(fmaf(lo32(x), lo32(w), lo32(acc)), fmaf(hi32(x), hi32(w), hi32(acc)));
}
__device__ __forceinline__ u64 dup2(float x) { return pack2(x, x); }

// down_thin: Conv2d(3 -> CS, k4 s2 p1) on [NB][2h][64][3] -> [NB][h][32][CS]  (CNNEncoder first layer, agent.py:78-91; also
// the input-gradient pass of the decoder's last ConvTranspose2d).  A warp owns two output rows (64 pixels) x 32 channels.
// Staged rows: [6 rows][3 ch][column parity][33] so that output column x reads input column 2x-1+kx at slot x + (kx >> 1) of
// plane kx & 1 (conflict-free, no index arithmetic per element).
constexpr int DT_PLANE = 33, DT_ROWF = 3 * 2 * DT_PLANE, DT_STAGE = 6 * DT_ROWF;
template <int CS>
__global__ void __launch_bounds__(128, 3)
conv_down_thin_kernel(const float* __restrict__ big, const float* __restrict__ W, float* __restrict__ small_, int NB, int h) {
  extern __shared__ __align__(16) float sm[];
  float* Wk = sm;                                  // [48][CS], k = (ky*4+kx)*3 + cb
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float* stg = sm + 48 * CS + warp * DT_STAGE;
  for (int e = threadIdx.x; e < CS * 48; e += blockDim.x) {
    const int cs = e / 48, rem = e - cs * 48, cb = rem >> 4, tap = rem & 15;    // W[cs][cb][ky][kx]
    Wk[(tap * 3 + cb) * CS + cs] = W[e];
  }
  __syncthreads();
  const int Hb = 2 * h, pairs = (h + 1) >> 1;
  const long long units = (long long)NB * pairs;
  for (long long u = (long long)blockIdx.x * 4 + warp; u < units; u += (long long)gridDim.x * 4) {
    const long long n = u / pairs;
    const int y0 = (int)(u - n * pairs) * 2;
    __syncwarp();
    // stage big rows 2*y0-1 .. 2*y0+4 (zero outside the image), 48 float4 per row
    for (int idx = lane; idx < 6 * 48; idx += 32) {
      const int r = idx / 48, f4 = idx - r * 48, iy = 2 * y0 - 1 + r;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (iy >= 0 && iy < Hb) v = __ldg(reinterpret_cast<const float4*>(big + ((n * Hb + iy) * 64) * 3) + f4);
      const float vs[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int e = f4 * 4 + j, col = e / 3, ch = e - col * 3, pc = col + 1;
        stg[r * DT_ROWF + (ch * 2 + (pc & 1)) * DT_PLANE + (pc >> 1)] = vs[j];
      }
    }
    if (lane < 18) {                                 // the two padding columns (-1 and 64) of every (row, channel)
      const int r = lane / 3, ch = lane - r * 3;
      stg[r * DT_ROWF + (ch * 2 + 0) * DT_PLANE + 0] = 0.f;
      stg[r * DT_ROWF + (ch * 2 + 1) * DT_PLANE + 32] = 0.f;
    }
    __syncwarp();
    const bool two = y0 + 1 < h;
    // lane = (pixel group pg = lane >> 2: columns 4pg .. 4pg+3 of both rows, channel octet cg = lane & 3): 8 pixels x 8
    // channels of packed accumulators.  Per patch element a lane loads 8 inputs (LDS.32, shared by the 4 lanes of a pixel
    // group) and 8 weights (2 LDS.128, shared by the 8 lanes of an octet): 16 words for 64 FMAs (the lane-per-pixel mapping
    // loaded 34 for 64 and sat on the shared-memory return path).
    const int pg = lane >> 2, cg = lane & 3;
#pragma unroll 1
    for (int c0 = 0; c0 < CS; c0 += 32) {
      u64 acc[8][4];
#pragma unroll
      for (int p = 0; p < 8; ++p)
#pragma unroll
        for (int q = 0; q < 4; ++q) acc[p][q] = 0ull;
#pragma unroll 1
      for (int ky = 0; ky < 4; ++ky)
#pragma unroll
        for (int kx = 0; kx < 4; ++kx)
#pragma unroll
          for (int cb = 0; cb < 3; ++cb) {
            const int off = (cb * 2 + (kx & 1)) * DT_PLANE + 4 * pg + (kx >> 1);
            const ulonglong2* wp = reinterpret_cast<const ulonglong2*>(Wk + ((ky * 4 + kx) * 3 + cb) * CS + c0 + cg * 8);
            const ulonglong2 w0 = wp[0], w1 = wp[1];
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              const u64 x0 = dup2(stg[ky * DT_ROWF + off + j]), x1 = dup2(stg[(ky + 2) * DT_ROWF + off + j]);
              fma2(acc[j][0], x0, w0.x); fma2(acc[j][1], x0, w0.y); fma2(acc[j][2], x0, w1.x); fma2(acc[j][3], x0, w1.y);
              fma2(acc[4 + j][0], x1, w0.x); fma2(acc[4 + j][1], x1, w0.y); fma2(acc[4 + j][2], x1, w1.x); fma2(acc[4 + j][3], x1, w1.y);
            }
          }
#pragma unroll
      for (int p = 0; p < 8; ++p) {
        const int row = y0 + (p >> 2), x = 4 * pg + (p & 3);
        if (row < h && (two || p < 4)) {
          float4* o = reinterpret_cast<float4*>(small_ + ((n * h + row) * 32 + x) * (long long)CS + c0 + cg * 8);
          o[0] = make_float4(lo32(acc[p][0]), hi32(acc[p][0]), lo32(acc[p][1]), hi32(acc[p][1]));
          o[1] = make_float4(lo32(acc[p][2]), hi32(acc[p][2]), lo32(acc[p][3]), hi32(acc[p][3]));
        }
      }
    }
  }
}

// up_thin2: ConvTranspose2d(CS -> 3, k4 s2 p1) on [NB][h][32][CS] -> [NB][2h][64][3] (CNNDecoder last layer, agent.py:199-222).
// Lane j owns small-grid positions (i, j) and (i+1, j), i.e. 2 x (2x2x3) outputs.  Packed FMAs pair EVEN/ODD input channels
// (both operands are natural 64-bit pairs of the channel-last layouts, no duplication moves); the two partial sums of an
// output are added at the end.  Per neighbour column dx the four staged rows are loaded once (4 LDS.128) and every weight
// LDS.128 (4 channels of one (dy, dx, a, b, c) combination, warp-uniform) feeds 4 packed FMAs.
// Output (2i+a) takes small rows i+dy with kernel row ky = a - 2dy + 1 (dy=-1: a=0, ky=3; dy=0: ky=a+1; dy=+1: a=1, ky=0).
// A CTA (4 warps) owns 8 consecutive small rows and stages the 10 rows they touch once: [10][34 positions][32 ch + 4 pad].
constexpr int UT_POS = 34, UT_CH = 36, UT_ROWS = 10, UT_STAGE = UT_ROWS * UT_POS * UT_CH;
template <int CS>
__global__ void __launch_bounds__(128)
conv_up_thin2_kernel(const float* __restrict__ small_, const float* __restrict__ W, const float* __restrict__ bias,
                     float* __restrict__ big, int NB, int h) {
  extern __shared__ __align__(16) float sm[];
  float* Wn = sm;                                  // [3 dy][3 dx][2 a][2 b][3 c][CS] (unused (a, b) slots stay zero)
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float* stg = sm + 108 * CS;
  for (int e = threadIdx.x; e < 108 * CS; e += blockDim.x) Wn[e] = 0.f;
  __syncthreads();
  for (int e = threadIdx.x; e < CS * 48; e += blockDim.x) {
    const int cs = e / 48, rem = e - cs * 48, c = rem >> 4, ky = (rem >> 2) & 3, kx = rem & 3;   // W[cs][c][ky][kx]
    const int dy = (ky == 3) ? -1 : ((ky == 0) ? 1 : 0), a = (ky == 2 || ky == 0) ? 1 : 0;
    const int dx = (kx == 3) ? -1 : ((kx == 0) ? 1 : 0), b = (kx == 2 || kx == 0) ? 1 : 0;
    Wn[(((((dy + 1) * 3 + (dx + 1)) * 2 + a) * 2 + b) * 3 + c) * CS + cs] = W[e];
  }
  __syncthreads();
  const int octs = (h + 7) >> 3, Hb = 2 * h;
  const long long units = (long long)NB * octs;
  for (long long u = blockIdx.x; u < units; u += gridDim.x) {
    const long long n = u / octs;
    const int ib = (int)(u - n * octs) * 8, i0 = ib + 2 * warp;
    u64 acc[2][2][2][3];
#pragma unroll
    for (int p = 0; p < 2; ++p)
#pragma unroll
      for (int a = 0; a < 2; ++a)
#pragma unroll
        for (int b = 0; b < 2; ++b)
#pragma unroll
          for (int c = 0; c < 3; ++c) acc[p][a][b][c] = 0ull;
#pragma unroll 1
    for (int c0 = 0; c0 < CS; c0 += 32) {
      __syncthreads();
      // stage small rows ib-1 .. ib+8, 32 channels [c0, c0+32): 8 float4 per position
      for (int idx = threadIdx.x; idx < UT_ROWS * 32 * 8; idx += blockDim.x) {
        const int r = idx >> 8, pos = (idx >> 3) & 31, f4 = idx & 7, iy = ib - 1 + r;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (iy >= 0 && iy < h) v = __ldg(reinterpret_cast<const float4*>(small_ + ((n * h + iy) * 32 + pos) * (long long)CS + c0) + f4);
        *reinterpret_cast<float4*>(stg + (r * UT_POS + pos + 1) * UT_CH + f4 * 4) = v;
      }
      for (int idx = threadIdx.x; idx < UT_ROWS * 2 * 8; idx += blockDim.x) {      // zero the border positions -1 and 32
        const int r = idx >> 4, side = (idx >> 3) & 1, f4 = idx & 7;
        *reinterpret_cast<float4*>(stg + (r * UT_POS + side * 33) * UT_CH + f4 * 4) = make_float4(0.f, 0.f, 0.f, 0.f);
      }
      __syncthreads();
      const float* wst = stg + 2 * warp * UT_POS * UT_CH;     // this warp's rows i0-1 .. i0+2
#pragma unroll 1
      for (int cq = 0; cq < 8; ++cq) {                   // 4 channels per step
#pragma unroll
        for (int dx = -1; dx <= 1; ++dx) {
          ulonglong2 x[4];
#pragma unroll
          for (int r = 0; r < 4; ++r)
            x[r] = *reinterpret_cast<const ulonglong2*>(wst + (r * UT_POS + lane + 1 + dx) * UT_CH + cq * 4);
#pragma unroll
          for (int dy = -1; dy <= 1; ++dy)
#pragma unroll
            for (int a = (dy == 1 ? 1 : 0); a <= (dy == -1 ? 0 : 1); ++a)
#pragma unroll
              for (int b = (dx == 1 ? 1 : 0); b <= (dx == -1 ? 0 : 1); ++b)
#pragma unroll
                for (int c = 0; c < 3; ++c) {
                  const ulonglong2 wv = *reinterpret_cast<const ulonglong2*>(
                      Wn + (((((dy + 1) * 3 + (dx + 1)) * 2 + a) * 2 + b) * 3 + c) * CS + c0 + cq * 4);
                  fma2(acc[0][a][b][c], x[dy + 1].x, wv.x); fma2(acc[0][a][b][c], x[dy + 1].y, wv.y);
                  fma2(acc[1][a][b][c], x[dy + 2].x, wv.x); fma2(acc[1][a][b][c], x[dy + 2].y, wv.y);
                }
        }
      }
    }
    float bv[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) bv[c] = bias ? bias[c] : 0.f;
#pragma unroll
    for (int p = 0; p < 2; ++p) {
      if (i0 + p >= h) break;
#pragma unroll
      for (int a = 0; a < 2; ++a) {
        float2* dst = reinterpret_cast<float2*>(big + ((n * Hb + 2 * (i0 + p) + a) * 64 + 2 * lane) * 3LL);   // 6 floats
        float o[6];
#pragma unroll
        for (int b = 0; b < 2; ++b)
#pragma unroll
          for (int c = 0; c < 3; ++c) o[b * 3 + c] = lo32(acc[p][a][b][c]) + hi32(acc[p][a][b][c]) + bv[c];
        dst[0] = make_float2(o[0], o[1]); dst[1] = make_float2(o[2], o[3]); dst[2] = make_float2(o[4], o[5]);
      }
    }
  }
}


// wgrad_thin2: dW[cs][cb][ky][kx] += sum over small pixels of small[p][cs] * big[patch(p)][ky][kx][cb] for 3-channel big images
// and 32-wide small grids (weight gradient of the encoder's first Conv2d / the decoder's last ConvTranspose2d).  One warp per
// small row (blockIdx.y = 32-channel group).  The 4 image rows a small row touches are staged twice, left-padded by 3 and by
// 5 floats: pixel x's 12-float patch row starts at float 6x (even x, first copy) or 6x+2 (odd x, second copy), both 16-byte
// aligned LDS.128.  One shared-memory + global atomic flush per CTA.
constexpr int WT_ROW = 200;
template <int NWARPS>
__global__ void __launch_bounds__(NWARPS * 32)
conv_wgrad_thin2_kernel(const float* __restrict__ small_, const float* __restrict__ big, float* __restrict__ dW, int NB, int h,
                        int Cs) {
  __shared__ __align__(16) float R[NWARPS][2][4][WT_ROW];
  __shared__ __align__(16) float S[NWARPS][32 * 32];
  __shared__ float Red[48 * 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, g = blockIdx.y;
  const int Hb = 2 * h;
  for (int e = threadIdx.x; e < 48 * 32; e += blockDim.x) Red[e] = 0.f;
  for (int e = threadIdx.x; e < NWARPS * 2 * 4 * WT_ROW; e += blockDim.x) (&R[0][0][0][0])[e] = 0.f;   // the pads stay zero
  __syncthreads();
  // lane = (patch row ky = lane >> 3, channel quad csg = lane & 7): 12 patch floats x 4 channels of accumulators, packed
  // over patch-float pairs.  Per pixel a lane loads its 12 patch floats (3 LDS.128, shared by the 8 lanes of a ky) and its
  // 4 channel values (1 LDS.128, shared by the 4 lanes of a quad): 16 words for 48 FMAs — the warp-per-channel mapping
  // loaded 49 words for 48 FMAs and sat on the 128 B/clk shared-memory return path.
  const int kg = lane >> 3, csg = lane & 7;
  u64 acc[6][4];
#pragma unroll
  for (int q = 0; q < 6; ++q)
#pragma unroll
    for (int c = 0; c < 4; ++c) acc[q][c] = 0ull;
  const long long rows = (long long)NB * h;
  for (long long u = (long long)blockIdx.x * NWARPS + warp; u < rows; u += (long long)gridDim.x * NWARPS) {
    const long long n = u / h;
    const int y = (int)(u - n * h);
    __syncwarp();
#pragma unroll
    for (int i = 0; i < 6; ++i) {                    // image rows 2y-1 .. 2y+2: 4 x 48 float4
      const int idx = lane + 32 * i, ky = idx / 48, f4 = idx - ky * 48, iy = 2 * y - 1 + ky;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (iy >= 0 && iy < Hb) v = __ldg(reinterpret_cast<const float4*>(big + (n * Hb + iy) * 192) + f4);
      float* ra = &R[warp][0][ky][4 * f4 + 3];
      float* rb = &R[warp][1][ky][4 * f4 + 5];
      ra[0] = v.x; ra[1] = v.y; ra[2] = v.z; ra[3] = v.w;
      rb[0] = v.x; rb[1] = v.y; rb[2] = v.z; rb[3] = v.w;
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {                    // small row: 32 pixels x 32 channels of group g
      const int idx = lane + 32 * i, px = idx >> 3, f4 = idx & 7;
      *reinterpret_cast<float4*>(&S[warp][px * 32 + f4 * 4]) =
          __ldg(reinterpret_cast<const float4*>(small_ + ((n * h + y) * 32 + px) * (long long)Cs + g * 32) + f4);
    }
    __syncwarp();
#pragma unroll 2
    for (int px = 0; px < 32; px += 2) {
#pragma unroll
      for (int o = 0; o < 2; ++o) {
        const float4 sv = *reinterpret_cast<const float4*>(&S[warp][(px + o) * 32 + csg * 4]);
        const u64 s0 = dup2(sv.x), s1 = dup2(sv.y), s2 = dup2(sv.z), s3 = dup2(sv.w);
        const ulonglong2* pp = reinterpret_cast<const ulonglong2*>(&R[warp][o][kg][6 * (px + o) + 2 * o]);
#pragma unroll
        for (int q = 0; q < 3; ++q) {
          const ulonglong2 bv = pp[q];
          fma2(acc[2 * q][0], s0, bv.x); fma2(acc[2 * q][1], s1, bv.x); fma2(acc[2 * q][2], s2, bv.x); fma2(acc[2 * q][3], s3, bv.x);
          fma2(acc[2 * q + 1][0], s0, bv.y); fma2(acc[2 * q + 1][1], s1, bv.y);
          fma2(acc[2 * q + 1][2], s2, bv.y); fma2(acc[2 * q + 1][3], s3, bv.y);
        }
      }
    }
  }
  // acc[q][c]: patch floats f = 2q, 2q+1 of row kg (k = kg*12 + f), channel csg*4 + c
#pragma unroll
  for (int q = 0; q < 6; ++q)
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      atomicAdd(&Red[(kg * 12 + 2 * q) * 32 + csg * 4 + c], lo32(acc[q][c]));
      atomicAdd(&Red[(kg * 12 + 2 * q + 1) * 32 + csg * 4 + c], hi32(acc[q][c]));
    }
  __syncthreads();
  for (int e = threadIdx.x; e < 48 * 32; e += blockDim.x) {
    const int cs = g * 32 + (e & 31), k = e >> 5, tap = k / 3, cb = k - tap * 3;      // k = tap * 3 + cb
    atomicAdd(&dW[((long long)cs * 3 + cb) * 16 + tap], Red[e]);
  }
}

}  // namespace

// dispatch predicates of conv.cu's b200rl_conv_{up,wgrad,down} (include/b200rl.h); the launchers below are internal
extern "C" int b200rl_thin_up_supported(int Cs, int Cb) { return Cb == 3 && (Cs == 32 || Cs == 48 || Cs == 64 || Cs == 96); }
extern "C" int b200rl_thin_wgrad_supported(int Cs, int Cb) { return Cb >= 1 && Cb <= 4 && Cs % 32 == 0 && Cs <= 128; }

extern "C" int b200rl_thin_down_supported(int w, int Cs, int Cb) { return Cb == 3 && w == 32 && (Cs == 32 || Cs == 64 || Cs == 96); }

int b200rl_conv_down_thin(const float* big, const float* W, float* small, int NB, int h, int w, int Cs, int Cb, cudaStream_t st) {
  (void)w; (void)Cb;
  const long long units = (long long)NB * ((h + 1) / 2);
  long long blocks = (units + 3) / 4;
  if (blocks > 4LL * kNumSMs) blocks = 4LL * kNumSMs;
  const size_t smem = sizeof(float) * (48 * Cs + 4 * DT_STAGE);
#define DOWN_THIN(CS_)                                                                                               \
  do {                                                                                                               \
    RL_CUDA(cudaFuncSetAttribute(conv_down_thin_kernel<CS_>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
    conv_down_thin_kernel<CS_><<<(unsigned)blocks, 128, smem, st>>>(big, W, small, NB, h);                         \
  } while (0)
  if (Cs == 32) DOWN_THIN(32); else if (Cs == 64) DOWN_THIN(64); else DOWN_THIN(96);
#undef DOWN_THIN
  RL_CHECK_LAUNCH();
  return B200RL_OK;
}

int b200rl_conv_up_thin(const float* small, const float* W, float* big, const float* bias, int NB, int h, int w, int Cs,
                        int Cb, cudaStream_t st) {
  if (w == 32 && (Cs == 32 || Cs == 64 || Cs == 96)) {
    const long long units = (long long)NB * ((h + 7) / 8);
    long long blocks = units < 3LL * kNumSMs ? units : 3LL * kNumSMs;
    const size_t smem = sizeof(float) * (108 * Cs + UT_STAGE);
#define UP_THIN2(CS_)                                                                                                \
  do {                                                                                                               \
    RL_CUDA(cudaFuncSetAttribute(conv_up_thin2_kernel<CS_>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
    conv_up_thin2_kernel<CS_><<<(unsigned)blocks, 128, smem, st>>>(small, W, bias, big, NB, h);                    \
  } while (0)
    if (Cs == 32) UP_THIN2(32); else if (Cs == 64) UP_THIN2(64); else UP_THIN2(96);
#undef UP_THIN2
    RL_CHECK_LAUNCH();
    return B200RL_OK;
  }
  const long long total = (long long)NB * h * w;
  long long blocks = (total + 127) / 128;
  if (blocks > (long long)kNumSMs * 16) blocks = (long long)kNumSMs * 16;
  switch (Cs) {
    case 32: conv_up_thin_kernel<3, 32><<<(unsigned)blocks, 128, 0, st>>>(small, W, bias, big, NB, h, w); break;
    case 48: conv_up_thin_kernel<3, 48><<<(unsigned)blocks, 128, 0, st>>>(small, W, bias, big, NB, h, w); break;
    case 64: conv_up_thin_kernel<3, 64><<<(unsigned)blocks, 128, 0, st>>>(small, W, bias, big, NB, h, w); break;
    default: conv_up_thin_kernel<3, 96><<<(unsigned)blocks, 128, 0, st>>>(small, W, bias, big, NB, h, w); break;
  }
  RL_CHECK_LAUNCH();
  return B200RL_OK;
}

int b200rl_conv_wgrad_thin(const float* small, const float* big, float* dW, int NB, int h, int w, int Cs, int Cb,
                           cudaStream_t st) {
  if (Cb == 3 && w == 32 && Cs % 32 == 0) {
    constexpr int NW = 4;
    const long long rows = (long long)NB * h;
    long long bx = (rows + NW - 1) / NW;
    const long long cap = (4LL * kNumSMs) / (Cs / 32) > 0 ? (4LL * kNumSMs) / (Cs / 32) : 1;
    if (bx > cap) bx = cap;
    conv_wgrad_thin2_kernel<NW><<<dim3((unsigned)bx, Cs / 32), NW * 32, 0, st>>>(small, big, dW, NB, h, Cs);
    RL_CHECK_LAUNCH();
    return B200RL_OK;
  }
  const int tiles_per_row = (w + 31) / 32;
  const long long ntiles = (long long)NB * h * tiles_per_row;
  // ~13 KB of smem and 80 registers per thread: 6 CTAs per SM hide the stage -> compute latency of a 32-pixel tile
  long long blocks = ntiles < 6LL * kNumSMs ? ntiles : 6LL * kNumSMs;
  const size_t smem = sizeof(float) * (4 * (2 * 32 + 2) * Cb + 32 * 32 + 16 * Cb * Cs);
  switch (Cb) {
    case 1: conv_wgrad_thin_kernel<1><<<(unsigned)blocks, 256, smem, st>>>(small, big, dW, NB, h, w, Cs, tiles_per_row); break;
    case 2: conv_wgrad_thin_kernel<2><<<(unsigned)blocks, 256, smem, st>>>(small, big, dW, NB, h, w, Cs, tiles_per_row); break;
    case 3: conv_wgrad_thin_kernel<3><<<(unsigned)blocks, 256, smem, st>>>(small, big, dW, NB, h, w, Cs, tiles_per_row); break;
    default: conv_wgrad_thin_kernel<4><<<(unsigned)blocks, 256, smem, st>>>(small, big, dW, NB, h, w, Cs, tiles_per_row); break;
  }
  RL_CHECK_LAUNCH();
  return B200RL_OK;
}
