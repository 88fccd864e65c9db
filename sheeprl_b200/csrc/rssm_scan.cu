// Persistent RSSM scan: all T steps of RSSM.dynamic (forward) and their BPTT (backward), each as ONE
// cooperative kernel.
//
// Replaces the Python loop `for i in range(sequence_length): rssm.dynamic(...)`
// (sheeprl/algos/dreamer_v3/dreamer_v3.py:131-145 -> agent.py:396-435: is_first masking, RecurrentModel +
// LayerNormGRUCell models.py:396-403, representation MLP, unimix, straight-through sampling) and the autograd
// replay of it inside `fabric.backward(rec_loss)` (dreamer_v3.py:191).
//
// What is on the recurrence and what is not.  Only the POSTERIOR feeds the next step (z_t -> x_{t+1} -> h_{t+1});
// the prior (transition model on h_t, agent.py:433) is a function of the finished h sequence, so its forward and
// its backward (its gradient comes from the KL term only) are batched tensor-core products over all T*B rows
// OUTSIDE this kernel (engine.py: _prior_forward / _prior_backward).  The kernels below carry the dependent
// chain only:
//   forward   z_{t-1} --gather W_in--> x (LN, SiLU) --W_g--> gates (LN over 3R) --> h_t --W_r1--> rp (LN, SiLU)
//             --W_r2--> logits --unimix, sample--> z_t
//   backward  the reverse chain, LayerNorm corrections applied by the CONSUMER of each gradient row.
//
// Design (B200).  The batch is tiny (B <= 16 rows), the steps strictly sequential: the scan is latency-bound, so
// the design minimises the number and the cost of cross-SM hand-offs per step.
//   * 128 co-resident CTAs (one per SM, cooperative launch), each owning a fixed slice of OUTPUT COLUMNS of every
//     weight matrix, resident in shared memory for the whole scan (weights are read from HBM once per scan).
//   * No grid barriers.  Every cross-CTA hand-off is a flag-carrying data exchange ("LL": each 8-byte element is
//     {fp32 value, 32-bit step tag}, written with one 64-bit store and polled with 64-bit loads straight from L2):
//     the consumer spins on the very data it needs, so a hand-off costs one L2 store + one L2 load latency instead of
//     release-fence + atomic counter + acquire + a dependent load.  Four hand-offs per forward step (z indices, x rows,
//     GRU LayerNorm partial statistics, h rows; then rp rows to the sampling units), four per backward step.
//   * Work that does not depend on the newest hand-off is issued before waiting for it (the h-part of the GRU product
//     runs while the x rows are still being built; input prefetches at step start).
//   * z_{t-1} is one-hot per group, so z W_in^T is a gather of S weights per output from the CTA's W_in slice.  Every
//     CTA receives all x rows anyway (the x-part of the GRU product needs them), so each computes the x LayerNorm
//     statistics itself, with the same code and summation order: bit-identical on every CTA, no CTA is a row owner.
//   * Products: the batch is one MMA tile high, so a warp takes an (8-column tile) x (K slice) item of m16n8k8 TF32 MMAs
//     with the 3xTF32 split (fp32-accurate); K-slice partials are summed in a fixed order (bit-reproducible).
#include "b200rl.h"
#include "common.cuh"

namespace {

constexpr int SCAN_G = 128;    // CTAs (one per SM; 132 SMs available)
constexpr int SCAN_NT = 512;   // threads per CTA: the scan is latency-bound (ncu: 11 stall cycles per issued instruction at
                               // 8 warps / SM), so every phase is spread over 32 warps with short per-warp instruction streams
constexpr int SCAN_NW = SCAN_NT / 32;
constexpr int MAXB = 16;
constexpr int MAXRPU = 8;      // rows of one sampling unit (S <= 64 groups over 128 CTAs -> >= 2 row splits)
constexpr int KS_MAX = 8;      // K slices of a product (rows of the partial buffer)
constexpr int CLS_SLICES = 8;  // K slices of the class-per-lane products (logits / dz)

typedef unsigned long long u64;

__host__ __device__ inline int r4(int x) { return (x + 3) / 4 * 4; }
__host__ __device__ inline int imax(int a, int b) { return a > b ? a : b; }
__host__ __device__ inline int imin(int a, int b) { return a < b ? a : b; }

__host__ __device__ inline int owned_groups(int width, int cta) {
  const int groups = (width + 3) / 4;
  return (groups > cta) ? (groups - cta + SCAN_G - 1) / SCAN_G : 0;
}
// number of valid columns of `width` owned by `cta`
__host__ __device__ inline int owned_cols(int width, int cta) {
  int n = 0;
  for (int gi = cta; gi * 4 < width; gi += SCAN_G) n += (width - gi * 4 < 4) ? width - gi * 4 : 4;
  return n;
}

// ---------------------------------------------------------------------------------------------------------------
// workspace: [header 256 B | profile | LL exchange region (zeroed at every launch) | saves shared by fwd and bwd]
// ---------------------------------------------------------------------------------------------------------------
struct Workspace {
  int* error;
  long long* prof;       // [2][32] cycle counters of CTA 0 and CTA 1 (profiling aid)
  u64* ll;               // LL region base
  int* zidx;             // [T][B][S] sampled class per group
  float* ln_stats;       // [3][T*B][2] (mean, rstd) of the x / g / representation LayerNorms
};

struct LLGeo {           // offsets (in u64 elements) inside the LL region; every buffer is double-buffered by step parity
  size_t z, x, s, h, r, a, b, c, d, sb, sc, sd, total;
};

__host__ __device__ inline LLGeo make_ll(int S, int Dx, int R, int Dr, int Z) {
  LLGeo g;
  size_t o = 0;
  g.z = o; o += 2 * (size_t)MAXB * S;            // forward: sampled class indices
  g.x = o; o += 2 * (size_t)MAXB * Dx;           //          x_pre rows
  g.s = o; o += 2 * (size_t)MAXB * SCAN_G * 2;   //          partial statistics of the GRU LayerNorm
  g.h = o; o += 2 * (size_t)MAXB * R;            //          h rows
  g.r = o; o += 2 * (size_t)MAXB * Dr;           //          rp_pre rows
  g.a = o; o += 2 * (size_t)MAXB * Z;            // backward: d_post_raw rows
  g.b = o; o += 2 * (size_t)MAXB * Dr;           //           dxh of the representation LayerNorm
  g.c = o; o += 2 * (size_t)MAXB * 3 * R;        //           dxh of the GRU LayerNorm
  g.d = o; o += 2 * (size_t)MAXB * Dx;           //           dxh of the x LayerNorm
  g.sb = o; o += 2 * (size_t)MAXB * SCAN_G * 2;  //           per-CTA row sums (sum dxh, sum dxh*xh) of the three
  g.sc = o; o += 2 * (size_t)MAXB * SCAN_G * 2;
  g.sd = o; o += 2 * (size_t)MAXB * SCAN_G * 2;
  g.total = o;
  return g;
}

constexpr size_t WS_HEADER = 256, WS_PROF = 2 * 32 * sizeof(long long);

__host__ __device__ inline size_t ws_ll_bytes(int S, int D, int Dx, int R, int Dr) {
  return make_ll(S, Dx, R, Dr, S * D).total * sizeof(u64);
}
__host__ __device__ inline size_t ws_bytes(int T, int B, int S, int D, int Dx, int R, int Dr) {
  return WS_HEADER + WS_PROF + ws_ll_bytes(S, D, Dx, R, Dr) + sizeof(int) * (size_t)T * B * S +
         sizeof(float) * 3 * (size_t)T * B * 2 + 256;
}

__host__ __device__ inline Workspace carve(void* ws, int T, int B, int S, int D, int Dx, int R, int Dr) {
  Workspace w;
  char* p = (char*)ws;
  w.error = (int*)(p + 64);
  p += WS_HEADER;
  w.prof = (long long*)p;   p += WS_PROF;
  w.ll = (u64*)p;           p += ws_ll_bytes(S, D, Dx, R, Dr);
  w.zidx = (int*)p;         p += sizeof(int) * (size_t)T * B * S;
  w.ln_stats = (float*)p;
  return w;
}

// ---------------------------------------------------------------------------------------------------------------
// LL exchange primitives
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ u64 ll_pack(float v, unsigned tag) { return ((u64)tag << 32) | (u64)__float_as_uint(v); }
__device__ __forceinline__ void ll_store(u64* p, float v, unsigned tag) {
  asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(ll_pack(v, tag)) : "memory");
}
__device__ __forceinline__ void ll_store2(u64* p, float v0, float v1, unsigned tag) {   // p 16-byte aligned
  asm volatile("st.relaxed.gpu.global.v2.u64 [%0], {%1, %2};" ::"l"(p), "l"(ll_pack(v0, tag)), "l"(ll_pack(v1, tag)) : "memory");
}
__device__ __forceinline__ u64 ll_load(const u64* p) {
  u64 x;
  asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(x) : "l"(p) : "memory");
  return x;
}
__device__ __forceinline__ void ll_load2(const u64* p, u64& a, u64& b) {                // p 16-byte aligned
  asm volatile("ld.relaxed.gpu.global.v2.u64 {%0, %1}, [%2];" : "=l"(a), "=l"(b) : "l"(p) : "memory");
}

struct Spin {            // bounded polling: a lost hand-off must never hang the device
  int* error;
  unsigned polls;
  long long t0;
  bool dead;
  __device__ __forceinline__ void init(int* e) { error = e; polls = 0; t0 = 0; dead = false; }
  // called on every failed poll; returns true when the wait must be abandoned
  __device__ __forceinline__ bool fail() {
    if (dead) return true;
    if ((++polls & 255u) == 0u) {
      if (t0 == 0) t0 = clock64();
      if (clock64() - t0 > 4000000000LL) { atomicExch(error, 1); dead = true; }               // ~2 s
      else if (*(volatile int*)error != 0) dead = true;                                        // another CTA gave up
    }
    return dead;
  }
};

__device__ __forceinline__ float ll_wait(const u64* p, unsigned tag, Spin& sp) {
  u64 v = ll_load(p);
  while ((unsigned)(v >> 32) != tag) {
    if (sp.fail()) break;
    v = ll_load(p);
  }
  return __uint_as_float((unsigned)v);
}

// Receives rows x n values (n even; LL rows of stride ss elements, 16-byte aligned) into shared memory rows of stride ds.
// Thread (row group, column pair): LL_UNROLL 16-byte loads in flight before the first tag is checked (one L2 round trip
// per batch; 8 in the forward kernel, 4 in the register-tighter backward kernel where 8 spilled and measured slower).
// With `sums` (the backward's LayerNorm hand-offs: the producers send their per-CTA row sums (sum dxh, sum dxh*xh) right
// after the rows), warp w also polls the SCAN_G partials of row sr0 + w (< sr0 + rows) in the same wave: they are loaded
// before the rows, every retry re-polls the stale rows and partials together, and the partials are then summed in a
// fixed order, scaled by `inv` into out1 / out2 [sr0 + w].  `sums` points at the row-sum block of the step's parity.
// (inlined, like every helper of the step loops: as calls, ptxas saved and restored the step's live values around each
// one, and with ~225 KB of shared memory per SM those spills miss L1.  Inlined, the S model's forward and backward took
// 1.66 / 1.65 ms per launch on an H100 instead of 1.72 / 2.07 ms.)
template <int LL_UNROLL>
__device__ __forceinline__ void ll_recv(float* dst, int ds, const u64* src, int ss, int rows, int n, unsigned tag, int tid, Spin& sp,
                                     const u64* sums = nullptr, int sr0 = 0, float inv = 0.f, float* out1 = nullptr,
                                     float* out2 = nullptr) {
  static_assert(MAXB <= SCAN_NW, "one warp per row of the row sums");
  const int lane = tid & 31, wid = tid >> 5;
  const bool has_s = sums != nullptr && wid < rows;              // warp-uniform
  const u64* sp_row = has_s ? sums + ((size_t)(sr0 + wid) * SCAN_G + lane) * 2 : nullptr;
  u64 sx[SCAN_G / 32], sy[SCAN_G / 32];
  bool s_stale = has_s;
  if (has_s)
#pragma unroll
    for (int i = 0; i < SCAN_G / 32; ++i) ll_load2(sp_row + 64 * i, sx[i], sy[i]);
  // the stale partials of this lane are re-issued (true while any is stale)
  auto poll_sums = [&]() {
    if (!s_stale) return false;
    bool st = false;
#pragma unroll
    for (int i = 0; i < SCAN_G / 32; ++i)
      if ((unsigned)(sx[i] >> 32) != tag || (unsigned)(sy[i] >> 32) != tag) { st = true; ll_load2(sp_row + 64 * i, sx[i], sy[i]); }
    s_stale = st;
    return st;
  };
  const int half = n >> 1;
  int rg = 0, kp = tid, nrg = 1, kstep = SCAN_NT;
  if (half < SCAN_NT) { rg = tid / half; kp = tid - rg * half; nrg = SCAN_NT / half; kstep = half; }
  if (rg < nrg)
    for (int k = 2 * kp; k < n; k += 2 * kstep) {
      for (int r0 = rg; r0 < rows; r0 += nrg * LL_UNROLL) {
        u64 a[LL_UNROLL], b[LL_UNROLL];
#pragma unroll
        for (int u = 0; u < LL_UNROLL; ++u)
          if (r0 + u * nrg < rows) ll_load2(src + (size_t)(r0 + u * nrg) * ss + k, a[u], b[u]);
        // elements that came back with an old tag are re-polled TOGETHER (one L2 round trip per retry of the whole batch,
        // not one per element), the row-sum partials with them
        for (;;) {
          bool stale = false;
#pragma unroll
          for (int u = 0; u < LL_UNROLL; ++u)
            if (r0 + u * nrg < rows && ((unsigned)(a[u] >> 32) != tag || (unsigned)(b[u] >> 32) != tag)) stale = true;
          if (!stale || sp.fail()) break;
#pragma unroll
          for (int u = 0; u < LL_UNROLL; ++u)
            if (r0 + u * nrg < rows && ((unsigned)(a[u] >> 32) != tag || (unsigned)(b[u] >> 32) != tag))
              ll_load2(src + (size_t)(r0 + u * nrg) * ss + k, a[u], b[u]);
          poll_sums();
        }
#pragma unroll
        for (int u = 0; u < LL_UNROLL; ++u)
          if (r0 + u * nrg < rows)
            *reinterpret_cast<float2*>(dst + (r0 + u * nrg) * ds + k) =
                make_float2(__uint_as_float((unsigned)a[u]), __uint_as_float((unsigned)b[u]));
      }
    }
  if (!has_s) return;
  while (poll_sums() && !sp.fail()) {}
  float v0 = 0.f, v1 = 0.f;
#pragma unroll
  for (int i = 0; i < SCAN_G / 32; ++i) {
    v0 += __uint_as_float((unsigned)sx[i]);
    v1 += __uint_as_float((unsigned)sy[i]);
  }
  v0 = warp_sum(v0); v1 = warp_sum(v1);
  if (lane == 0) { out1[sr0 + wid] = v0 * inv; out2[sr0 + wid] = v1 * inv; }
}

// (row, owned-column) element a thread is responsible for during the whole scan: e = b * per_row + cj
struct Slot {
  int b, cj, col;
  bool ok;
};
__device__ __forceinline__ Slot make_slot(int e, int per_row, int B, int cta, int width) {
  Slot s;
  s.b = per_row > 0 ? e / per_row : 0;
  s.cj = e - s.b * per_row;
  s.col = (cta + (s.cj >> 2) * SCAN_G) * 4 + (s.cj & 3);
  s.ok = per_row > 0 && s.b < B && s.col < width;
  return s;
}

// fast transcendental form for SiLU; rel. error ~1e-6
__device__ __forceinline__ float fsilu(float x) { return __fdividef(x, 1.f + __expf(-x)); }

// ---- products on the warp-level tensor-core path -------------------------------------------------------------------
// The batch is exactly one MMA tile high (B <= 16 rows), so a product is a row of m16n8k8 TF32 MMAs per 8 output columns.
// fp32 accuracy comes from the same 3xTF32 split as the large GEMMs (x = hi + lo, hi = x with the 13 low mantissa bits
// cleared; hi*lo + lo*hi + hi*hi, fp32 accumulate), the K reduction happens inside the MMA (the FFMA2 version spent most of
// a product item in its 62-shuffle cross-lane reduction and was bound by the 128 B/clk shared-memory return path: every
// loaded word fed only two FMAs), and a K slice's partial tile goes to PART like before (fixed-order sum by the caller).
// k permutation: within a 16-wide k step lane (g, t) owns k = 4t..4t+3 of BOTH operands (one LDS.128 each); the first MMA
// of the step consumes words 0, 1 as fragment columns (t, t+4), the second words 2, 3 — any pairing is valid as long as A
// and B agree, the MMA sums over k.
__device__ __forceinline__ void mma_tf32(float (&d)[4], const unsigned (&a)[4], unsigned b0, unsigned b1) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ unsigned tf32_hi(float x) { return __float_as_uint(x) & 0xffffe000u; }
__device__ __forceinline__ unsigned tf32_lo(float x) { return __float_as_uint(x - __uint_as_float(__float_as_uint(x) & 0xffffe000u)); }

// One (8-column tile, K slice) item.  X rows [0, 16) of stride xs (rows >= B are never read: their fragments are zero), weight
// rows w + n * wst for n < nvalid (missing rows read as zero).  k0, k1 multiples of 4; the tail of a slice is zero padded
// (both operands are zero padded to r4(K) by their producers, reads stay below k1).
__device__ __forceinline__ void mma_item(const float* __restrict__ X, int xs, int B, const float* __restrict__ w, int wst,
                                         int nvalid, int k0, int k1, float* part, int ldp, int c0, int lane) {
  const int g = lane >> 2, t = lane & 3;
  const bool r_lo = g < B, r_hi = g + 8 < B, n_ok = g < nvalid;
  const float* xa = X + (size_t)g * xs;
  const float* xb = X + (size_t)(g + 8) * xs;
  const float* wr = w + (size_t)g * wst;
  // three independent accumulators (hi*lo, lo*hi, hi*hi): a step's 6 MMAs form chains of 2 instead of 6 dependent MMAs
  float d[4] = {0.f, 0.f, 0.f, 0.f}, dx[4] = {0.f, 0.f, 0.f, 0.f}, dy[4] = {0.f, 0.f, 0.f, 0.f};
  for (int kb = k0; kb < k1; kb += 16) {             // warp-uniform trip count (mma.sync needs the whole warp)
    const int k = kb + 4 * t;
    const bool k_ok = k < k1;
    float4 va = make_float4(0.f, 0.f, 0.f, 0.f), vb = va, vw = va;
    if (r_lo && k_ok) va = *reinterpret_cast<const float4*>(xa + k);
    if (r_hi && k_ok) vb = *reinterpret_cast<const float4*>(xb + k);
    if (n_ok && k_ok) vw = *reinterpret_cast<const float4*>(wr + k);
    {
      const unsigned ah[4] = {tf32_hi(va.x), tf32_hi(vb.x), tf32_hi(va.y), tf32_hi(vb.y)};
      const unsigned al[4] = {tf32_lo(va.x), tf32_lo(vb.x), tf32_lo(va.y), tf32_lo(vb.y)};
      const unsigned bh0 = tf32_hi(vw.x), bh1 = tf32_hi(vw.y), bl0 = tf32_lo(vw.x), bl1 = tf32_lo(vw.y);
      mma_tf32(dx, ah, bl0, bl1);
      mma_tf32(dy, al, bh0, bh1);
      mma_tf32(d, ah, bh0, bh1);
    }
    {
      const unsigned ah[4] = {tf32_hi(va.z), tf32_hi(vb.z), tf32_hi(va.w), tf32_hi(vb.w)};
      const unsigned al[4] = {tf32_lo(va.z), tf32_lo(vb.z), tf32_lo(va.w), tf32_lo(vb.w)};
      const unsigned bh0 = tf32_hi(vw.z), bh1 = tf32_hi(vw.w), bl0 = tf32_lo(vw.z), bl1 = tf32_lo(vw.w);
      mma_tf32(dx, ah, bl0, bl1);
      mma_tf32(dy, al, bh0, bh1);
      mma_tf32(d, ah, bh0, bh1);
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) d[i] += dx[i] + dy[i];
  // accumulator fragment: d0 (row g, col 2t), d1 (g, 2t+1), d2 (g+8, 2t), d3 (g+8, 2t+1)
  const int c = 2 * t;
  if (c < nvalid) {
    part[(size_t)g * ldp + c0 + c] = d[0];
    part[(size_t)(g + 8) * ldp + c0 + c] = d[2];
  }
  if (c + 1 < nvalid) {
    part[(size_t)g * ldp + c0 + c + 1] = d[1];
    part[(size_t)(g + 8) * ldp + c0 + c + 1] = d[3];
  }
}

// Runs all (8-column tile, K slice) items of one product over the CTA's warps.  Slice s writes its partial sums to
// PART[s][b][cbase + column] for all MAXB rows (every element written by exactly one lane); the caller sums the slices in
// order (bit-reproducible).  `wbase`: first weight row; column n is row wbase + n*wst (groups of 4 columns are contiguous
// rows).  Returns the number of slices.  No barrier inside: the caller synchronises before (X complete) and after.
__device__ __forceinline__ int product(const float* X, int xs, const float* wbase, int wst, int ngroups, int K, int B,
                                       float* PART, int ldp, int cbase, int tid) {
  if (ngroups <= 0) return 0;
  const int lane = tid & 31, wid = tid >> 5;
  const int ncols = ngroups * 4, ntiles = (ncols + 7) >> 3, Kp = r4(K);
  int ks = imin(KS_MAX, imax(1, SCAN_NW / ntiles));
  const int kchunk = ((Kp + ks - 1) / ks + 15) / 16 * 16;
  ks = (Kp + kchunk - 1) / kchunk;
  for (int item = wid; item < ntiles * ks; item += SCAN_NW) {
    const int sl = item / ntiles, tile = item - sl * ntiles;
    const int k0 = sl * kchunk, k1 = imin(Kp, k0 + kchunk);
    mma_item(X, xs, B, wbase + (size_t)tile * 8 * wst, wst, imin(8, ncols - tile * 8), k0, k1,
             PART + (size_t)sl * MAXB * ldp, ldp, cbase + tile * 8, lane);
  }
  return ks;
}

__device__ __forceinline__ float part_sum(const float* PART, int ldp, int ks, int b, int c) {
  float v = 0.f;
  for (int s = 0; s < ks; ++s) v += PART[((size_t)s * MAXB + b) * ldp + c];
  return v;
}

// Class-per-column product (forward logits, backward dz): out[row][class] = sum_k X[row][k] * W[class][k] for nr <= MAXRPU
// rows and D <= 32 classes, on the same m16n8k8 3xTF32 MMAs as `product` (rows 8..15 of the tile are unused).  Warp
// (K slice s = wid % CLS_SLICES, class half wid / CLS_SLICES: two 8-class tiles sharing the A fragments); partials go to
// PART[s][row][class] (fixed-order sum by the caller).
__device__ __forceinline__ void class_product(const float* X, int xs, const float* W, int wst, int D, int Kp, int nr, float* PART,
                                              int tid) {
  const int lane = tid & 31, wid = tid >> 5, g = lane >> 2, t = lane & 3;
  const int sl = wid % CLS_SLICES, half = wid / CLS_SLICES;           // SCAN_NW == 2 * CLS_SLICES
  const int kc = ((Kp + CLS_SLICES - 1) / CLS_SLICES + 15) / 16 * 16;
  const int k0 = sl * kc, k1 = imin(Kp, k0 + kc);
  const int n0 = half * 16;                                           // classes [n0, n0 + 16)
  if (n0 >= D) return;
  const bool r_ok = g < nr, n_ok0 = n0 + g < D, n_ok1 = n0 + 8 + g < D;
  const float* xa = X + (size_t)g * xs;
  const float* w0 = W + (size_t)(n0 + g) * wst;
  const float* w1 = W + (size_t)(n0 + 8 + g) * wst;
  float d0[4] = {0.f, 0.f, 0.f, 0.f}, d1[4] = {0.f, 0.f, 0.f, 0.f};
  float e0[4] = {0.f, 0.f, 0.f, 0.f}, e1[4] = {0.f, 0.f, 0.f, 0.f};     // cross terms (hi*lo + lo*hi), separate chains
  for (int kb = k0; kb < k1; kb += 16) {
    const int k = kb + 4 * t;
    const bool k_ok = k < k1;
    float4 va = make_float4(0.f, 0.f, 0.f, 0.f), v0 = va, v1 = va;
    if (r_ok && k_ok) va = *reinterpret_cast<const float4*>(xa + k);
    if (n_ok0 && k_ok) v0 = *reinterpret_cast<const float4*>(w0 + k);
    if (n_ok1 && k_ok) v1 = *reinterpret_cast<const float4*>(w1 + k);
    {
      const unsigned ah[4] = {tf32_hi(va.x), 0u, tf32_hi(va.y), 0u}, al[4] = {tf32_lo(va.x), 0u, tf32_lo(va.y), 0u};
      mma_tf32(e0, ah, tf32_lo(v0.x), tf32_lo(v0.y)); mma_tf32(e1, ah, tf32_lo(v1.x), tf32_lo(v1.y));
      mma_tf32(d0, ah, tf32_hi(v0.x), tf32_hi(v0.y)); mma_tf32(d1, ah, tf32_hi(v1.x), tf32_hi(v1.y));
      mma_tf32(e0, al, tf32_hi(v0.x), tf32_hi(v0.y)); mma_tf32(e1, al, tf32_hi(v1.x), tf32_hi(v1.y));
    }
    {
      const unsigned ah[4] = {tf32_hi(va.z), 0u, tf32_hi(va.w), 0u}, al[4] = {tf32_lo(va.z), 0u, tf32_lo(va.w), 0u};
      mma_tf32(e0, ah, tf32_lo(v0.z), tf32_lo(v0.w)); mma_tf32(e1, ah, tf32_lo(v1.z), tf32_lo(v1.w));
      mma_tf32(d0, ah, tf32_hi(v0.z), tf32_hi(v0.w)); mma_tf32(d1, ah, tf32_hi(v1.z), tf32_hi(v1.w));
      mma_tf32(e0, al, tf32_hi(v0.z), tf32_hi(v0.w)); mma_tf32(e1, al, tf32_hi(v1.z), tf32_hi(v1.w));
    }
  }
  if (g < nr) {                                        // accumulator rows g (d[0], d[1]); rows g + 8 are padding
    float* out = PART + ((size_t)sl * MAXRPU + g) * 32 + n0 + 2 * t;
    out[0] = d0[0] + e0[0]; out[1] = d0[1] + e0[1];
    out[8] = d1[0] + e1[0]; out[9] = d1[1] + e1[1];
  }
}

// Copies 4 rows (row0..row0+3) of a row-major [rows][ld] weight, columns [c0, c0+K), into smem rows of stride `wst` at
// offset koff, zero padded to Kp.
__device__ __forceinline__ void load_rows4(float* dst, int wst, int koff, const float* W, size_t ld, int row0, int nrows_valid,
                                           int c0, int K, int Kp, int tid) {
  for (int j = 0; j < 4; ++j)
    for (int k = tid; k < Kp; k += SCAN_NT)
      dst[j * wst + koff + k] = (row0 + j < nrows_valid && k < K) ? W[(size_t)(row0 + j) * ld + c0 + k] : 0.f;
}
// Copies 4 COLUMNS (col0..col0+3) of a row-major [K][ld] weight into 4 smem rows (transposed slice) at offset koff.
__device__ __forceinline__ void load_cols4(float* dst, int wst, const float* W, size_t ld, int col0, int ncols_valid,
                                           int K, int koff, int tid) {
  for (int e = tid; e < K * 4; e += SCAN_NT) {
    const int k = e >> 2, j = e & 3;
    dst[j * wst + koff + k] = (col0 + j < ncols_valid) ? W[(size_t)k * ld + col0 + j] : 0.f;
  }
}

// per-phase cycle counters: accumulated in SHARED memory by thread 0 of CTA 0 / 1 (a global read-modify-write per mark
// would stall that warp for an L2 round trip ~16 times per step and make the instrumented CTAs the stragglers of every
// hand-off), flushed to the workspace when the kernel ends
__device__ __forceinline__ void prof_mark(long long* prof, int slot, long long& last, bool on) {
  if (on) {
    const long long now = clock64();
    prof[slot] += now - last;
    last = now;
  }
}

// =====================================================================================================
// forward
// =====================================================================================================
struct GeoF {
  int ngh, ngr, ngx;            // owned 4-column groups of R (GRU output columns), Dr (representation layer 1), Dx (x_pre)
  int sR, sDx, sDr, wgst, w2st; // padded widths; smem row strides of the W_g / W_r2 slices
  int nsplit, rpu;              // sampling units: S groups x nsplit row blocks of rpu rows
  int unit_g, unit_r0, unit_nr; // this CTA's unit: group (-1: none), first row, row count
  int ldp;                      // row length of the product partial buffers
  int kin;                      // row length of the W_in slice: S*D + A, padded
  int oWg, oWr1, oW2, oWin, oXh, oXx, oPart, oAcc, oX0, oPar, oMisc, oInt, total;
};

struct Dims { int B, S, D, R, Dx, Dr, A; };

__host__ __device__ inline GeoF make_geo_f(const Dims& a, int cta) {
  GeoF g;
  g.ngh = owned_groups(a.R, cta);
  g.ngr = owned_groups(a.Dr, cta);
  g.ngx = owned_groups(a.Dx, cta);
  g.kin = r4(a.S * a.D + a.A);
  g.sR = r4(a.R); g.sDx = r4(a.Dx); g.sDr = r4(a.Dr);
  g.wgst = g.sR + g.sDx;
  g.w2st = g.sDr + 4;           // +4: the 8 lanes of a quarter-warp hit 8 distinct 16-byte bank groups
  g.nsplit = imax(1, imin(a.B, SCAN_G / a.S));
  g.rpu = (a.B + g.nsplit - 1) / g.nsplit;
  g.unit_g = -1; g.unit_r0 = 0; g.unit_nr = 0;
  if (cta < a.S * g.nsplit) {
    const int sp = cta / a.S;
    g.unit_r0 = sp * g.rpu;
    g.unit_nr = imin(g.rpu, a.B - g.unit_r0);
    if (g.unit_nr > 0) g.unit_g = cta % a.S; else g.unit_nr = 0;
  }
  const int mh = owned_groups(a.R, 0), mr = owned_groups(a.Dr, 0), mx = owned_groups(a.Dx, 0);
  g.ldp = imax(imax(mh * 12, mr * 4), 4);
  int o = 0;
  g.oWg = o;   o += mh * 12 * g.wgst;
  g.oWr1 = o;  o += mr * 4 * g.sR;
  g.oW2 = o;   o += a.D * g.w2st;
  g.oWin = o;  o += mx * 4 * g.kin;            // W_in rows of the owned x_pre columns
  g.oXh = o;   o += MAXB * g.sR;
  g.oXx = o;   o += MAXB * imax(g.sDx, g.sDr);
  g.oPart = o; o += imax(KS_MAX * MAXB * g.ldp, CLS_SLICES * MAXRPU * 32);
  g.oAcc = o;  o += MAXB * g.ldp;
  g.oX0 = o;   o += imax(mx * 4, 4);           // x_pre of the learned initial posterior z0, owned columns
  g.oPar = o;  o += g.sR + 2 * g.sDx + 2 * g.sDr;   // h0 | lnx gamma, beta | lnr gamma, beta (read every step)
  g.oMisc = o; o += 8 * MAXB + 64;           // [0,48) flags / statistics; [48,80) and [80,112) per-warp reduction scratch
  // z0 class indices, z_{t-1} indices of every row, GRU column counts; SCAN_G more words than that, so that the
  // shared-memory need, and with it the envelope scan_check admits, is the one of the x-statistics exchange it replaced
  g.oInt = o;  o += r4(64 + MAXB * 64 + 2 * SCAN_G);
  g.total = o;
  return g;
}

// FIX: the model widths are compile-time constants (the BASELINE S model: stochastic 32x32, recurrent / dense / hidden
// 512) — index arithmetic and loop bounds fold; the generic instantiation reads them from the arguments.
template <bool FIX>
__global__ void __launch_bounds__(SCAN_NT, 1) rssm_scan_fwd_kernel(const b200rl_rssm_scan_args a) {
  extern __shared__ __align__(16) float sm[];
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int cta = blockIdx.x;
  const int T = a.T, B = a.B, A = a.A;
  const int S = FIX ? 32 : a.S, D = FIX ? 32 : a.D, Z = S * D, R = FIX ? 512 : a.R, Dx = FIX ? 512 : a.Dx, Dr = FIX ? 512 : a.Dr;
  const int NB = T * B;
  const GeoF g = make_geo_f(Dims{B, S, D, R, Dx, Dr, a.A}, cta);
  const Workspace ws = carve(a.workspace, T, B, S, D, Dx, R, Dr);
  const LLGeo L = make_ll(S, Dx, R, Dr, Z);
  float* Wg = sm + g.oWg;       // [ngh*12][wgst]  rows: (group, part r/c/u, col-in-group); cols [h (sR) | x (sDx)]
  float* Wr1 = sm + g.oWr1;     // [ngr*4][sR]
  float* W2 = sm + g.oW2;       // [D][w2st] rows of W_r2 of this CTA's categorical group
  float* Xh = sm + g.oXh;       // [MAXB][sR]  h rows (carried from one step to the next)
  float* Xx = sm + g.oXx;       // [MAXB][sDx] x rows; reused for the unit's rp rows
  float* PART = sm + g.oPart;
  float* ACC = sm + g.oAcc;     // [MAXB][ldp] finished g_pre columns (for the row statistics)
  float* Win = sm + g.oWin;     // [ngx*4][kin] rows of W_in of the owned x_pre columns
  float* X0 = sm + g.oX0;       // [ngx*4] x_pre contribution of the learned initial posterior z0 (owned columns)
  float* H0 = sm + g.oPar;      // [R] tanh(initial_recurrent_state)
  float* LNXG = H0 + g.sR;      // [Dx] x LayerNorm gamma, beta
  float* LNXB = LNXG + g.sDx;
  float* LNRG = LNXB + g.sDx;   // [Dr] representation LayerNorm gamma, beta
  float* LNRB = LNRG + g.sDr;
  float* misc = sm + g.oMisc;   // [0,16) first flags; [16,32) mean; [32,48) rstd; [48,80) reduction scratch
  int* z0idx = (int*)(sm + g.oInt);
  int* zall = z0idx + 64;       // [MAXB][64] class indices of z_{t-1}, every row
  int* nctab = zall + MAXB * 64;   // valid GRU columns per CTA
  const int ldp = g.ldp, xxs = imax(g.sDx, g.sDr);
  const bool sampler = g.unit_g >= 0;
  __shared__ long long sprof[32];
  const bool prof_on = (cta < 2) && tid == 0;
  long long* prof = sprof;
  if (tid < 32) sprof[tid] = 0;
  long long tlast = prof_on ? clock64() : 0;
  Spin sp;
  sp.init(ws.error);

  // ---------------- prologue: weight slices and per-step parameters -> shared memory (read from HBM once per scan)
  for (int e = tid; e < g.total; e += SCAN_NT) sm[e] = 0.f;
  __syncthreads();
  for (int gi = 0; gi < g.ngh; ++gi)
    for (int part = 0; part < 3; ++part) {
      float* dst = Wg + (size_t)(gi * 3 + part) * 4 * g.wgst;
      const float* Wp = a.W_g + (size_t)part * R * (R + Dx);
      load_rows4(dst, g.wgst, 0, Wp, R + Dx, (cta + gi * SCAN_G) * 4, R, 0, R, g.sR, tid);
      load_rows4(dst, g.wgst, g.sR, Wp, R + Dx, (cta + gi * SCAN_G) * 4, R, R, Dx, g.sDx, tid);
    }
  for (int gi = 0; gi < g.ngr; ++gi)
    load_rows4(Wr1 + (size_t)gi * 4 * g.sR, g.sR, 0, a.W_r1, a.ld_wr1, (cta + gi * SCAN_G) * 4, Dr, 0, R, g.sR, tid);
  if (sampler)
    for (int e = tid; e < D * Dr; e += SCAN_NT) {
      const int d = e / Dr, k = e - d * Dr;
      W2[d * g.w2st + k] = a.W_r2[((size_t)g.unit_g * D + d) * Dr + k];
    }
  for (int k = tid; k < R; k += SCAN_NT) H0[k] = a.h0[k];
  for (int k = tid; k < Dx; k += SCAN_NT) { LNXG[k] = a.lnx_g[k]; LNXB[k] = a.lnx_b[k]; }
  for (int k = tid; k < Dr; k += SCAN_NT) { LNRG[k] = a.lnr_g[k]; LNRB[k] = a.lnr_b[k]; }
  for (int c = tid; c < SCAN_G; c += SCAN_NT) nctab[c] = owned_cols(R, c);
  for (int gi = 0; gi < g.ngx; ++gi)
    load_rows4(Win + (size_t)gi * 4 * g.kin, g.kin, 0, a.W_in, Z + A, (cta + gi * SCAN_G) * 4, Dx, 0, Z + A, g.kin, tid);
  if (wid == 0) {  // class index of the learned initial posterior (one-hot `z0`)
    for (int gq = 0; gq < S; ++gq) {
      int best = 0;
      for (int d = lane; d < D; d += 32)
        if (a.z0[gq * D + d] > 0.5f) best = d;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) best = max(best, __shfl_xor_sync(0xffffffffu, best, o));
      if (lane == 0) z0idx[gq] = best;
    }
  }
  __syncthreads();
  for (int cj = tid; cj < g.ngx * 4; cj += SCAN_NT) {   // x_pre of z0 (used wherever is_first is set), owned columns
    float acc = 0.f;
    for (int gq = 0; gq < S; ++gq) acc += Win[(size_t)cj * g.kin + gq * D + z0idx[gq]];
    X0[cj] = acc;
  }
  // z_in of step 0 (z_{-1} = 0): f * z0, written by the sampling units for their (rows, group) block
  if (sampler)
    for (int e = tid; e < g.unit_nr * D; e += SCAN_NT) {
      const int b = g.unit_r0 + e / D, d = e % D;
      a.z_in[(size_t)b * Z + g.unit_g * D + d] = a.first[b] * ((z0idx[g.unit_g] == d) ? 1.f : 0.f);
    }
  // fixed element assignments (no index arithmetic inside the time loop)
  const int nh4 = g.ngh * 4, nh12 = g.ngh * 12, nr4 = g.ngr * 4, nx4 = g.ngx * 4;
  const Slot sH = make_slot(tid, nh4, B, cta, R);           // gate / h element
  const Slot sX = make_slot(tid, nx4, B, cta, Dx);          // x element (save of x_act)
  const Slot sR_ = make_slot(tid, nr4, B, cta, Dr);         // rp element
  // g_pre element: c = (group, part, j) inside the row of 12*ngh products
  const int pb = nh12 > 0 ? tid / nh12 : 0, pc = tid - pb * nh12;
  const int pcol = (cta + (pc / 12) * SCAN_G) * 4 + (pc & 3), ppart = (pc % 12) >> 2;
  const bool pok = nh12 > 0 && pb < B && pcol < R;
  const int ncol3 = 3 * owned_cols(R, cta);                // values per row in this CTA's share of the GRU LayerNorm
  const float bias2 = (sampler && lane < D) ? a.b_r2[g.unit_g * D + lane] : 0.f;
  float first_next = (tid < B) ? a.first[tid] : 0.f;        // is_first flags of the step about to run (threads < MAXB)
  __syncthreads();
  prof_mark(prof, 0, tlast, prof_on);

  for (int t = 0; t < T; ++t) {
    const size_t row0 = (size_t)t * B;
    const int par = t & 1;
    const unsigned tag = (unsigned)t + 1u;
    if (tid < MAXB) misc[tid] = first_next;                 // loaded during the previous step
    if (tid < MAXB) first_next = (tid < B && t + 1 < T) ? a.first[row0 + B + tid] : 0.f;
    // prefetches that do not depend on the chain
    const float pe_pref = sR_.ok ? a.pe[(row0 + sR_.b) * Dr + sR_.col] : 0.f;
    float noise_pref = 1.f, fnext = 0.f;
    if (sampler && wid < g.unit_nr) {
      if (lane < D) noise_pref = a.noise[(row0 + g.unit_r0 + wid) * Z + (size_t)g.unit_g * D + lane];
      if (t + 1 < T) fnext = a.first[row0 + B + g.unit_r0 + wid];
    }
    __syncthreads();
    const float* fl = misc;

    // ============ A (first: its hand-off is in flight while B1 runs): x_pre = W_in [z_in, a_in] for the owned columns, every row; z_in one-hot -> gather from the slice.
    // Warp b builds row b: lane = (column cj = lane / 8, part = lane % 8): 8 lanes sum S/8 gathered weights each, then a
    // fixed 3-level shuffle tree.
    if (t > 0)
      for (int e = tid; e < B * S; e += SCAN_NT) {
        const int b = e / S, gq = e - b * S;
        zall[b * 64 + gq] = (int)__float_as_uint(ll_wait(ws.ll + L.z + ((size_t)(par ^ 1) * MAXB + b) * S + gq, (unsigned)t, sp));
      }
    __syncthreads();
    prof_mark(prof, 2, tlast, prof_on);
    for (int b = wid; b < B; b += SCAN_NW) {
      const float f = fl[b];
      for (int c0 = 0; c0 < nx4; c0 += 4) {            // 4 columns x 8 parts per pass
        const int cj = c0 + (lane >> 3), part = lane & 7;
        const int col = (cta + (cj >> 2) * SCAN_G) * 4 + (cj & 3);
        const bool okc = cj < nx4 && col < Dx;
        float acc = 0.f;
        if (okc && t > 0 && f != 1.f) {
          const float* wrow = Win + (size_t)cj * g.kin;
          const int gper = (S + 7) >> 3, g_lo = part * gper, g_hi = imin(S, g_lo + gper);
          for (int gq = g_lo; gq < g_hi; ++gq) acc += wrow[gq * D + zall[b * 64 + gq]];
        }
        acc += __shfl_xor_sync(0xffffffffu, acc, 4);
        acc += __shfl_xor_sync(0xffffffffu, acc, 2);
        acc += __shfl_xor_sync(0xffffffffu, acc, 1);
        if (okc && part == 0) {
          float aa = 0.f;
          for (int qq = 0; qq < A; ++qq) aa = fmaf(a.actions[(row0 + b) * A + qq], Win[(size_t)cj * g.kin + Z + qq], aa);
          const float xv = (1.f - f) * (acc + aa) + f * X0[cj];
          ll_store(ws.ll + L.x + ((size_t)par * MAXB + b) * Dx + col, xv, tag);
          a.x_pre[(row0 + b) * Dx + col] = xv;
        }
      }
    }
    if (cta == (t % SCAN_G))
      for (int e = tid; e < B * A; e += SCAN_NT) a.a_in[row0 * A + e] = (1.f - fl[e / A]) * a.actions[row0 * A + e];
    prof_mark(prof, 3, tlast, prof_on);

    // ============ B1: h_in = (1-f) h_{t-1} + f h0 (agent.py:428), rows with f != 0 only; h-part of the GRU product
    for (int b = 0; b < B; ++b) {
      const float f = fl[b];
      if (f != 0.f || t == 0)
        for (int k = tid; k < R; k += SCAN_NT) Xh[b * g.sR + k] = (1.f - f) * ((t > 0) ? Xh[b * g.sR + k] : 0.f) + f * H0[k];
    }
    __syncthreads();
    prof_mark(prof, 12, tlast, prof_on);
    const int ksh = product(Xh, g.sR, Wg, g.wgst, g.ngh * 3, R, B, PART, ldp, 0, tid);
    prof_mark(prof, 1, tlast, prof_on);
    __syncthreads();
    const float acch = pok ? part_sum(PART, ldp, ksh, pb, pc) : 0.f;
    const float hin = sH.ok ? Xh[sH.b * g.sR + sH.col] : 0.f;
    prof_mark(prof, 13, tlast, prof_on);

    // ============ B2: x = SiLU(LN(x_pre)), x-part of the GRU product; g_pre columns; partial LayerNorm statistics
    ll_recv<8>(Xx, xxs, ws.ll + L.x + (size_t)par * MAXB * Dx, Dx, B, Dx, tag, tid, sp);
    __syncthreads();
    for (int b = wid; b < B; b += SCAN_NW) {   // warp b normalises row b in place: centred two passes, fixed order
      float* xr = Xx + b * xxs;
      float s = 0.f;
      for (int k = lane; k < Dx; k += 32) s += xr[k];
      const float mean = warp_sum(s) / (float)Dx;
      float m2 = 0.f;
      for (int k = lane; k < Dx; k += 32) { const float d = xr[k] - mean; m2 = fmaf(d, d, m2); }
      const float rstd = rsqrtf(warp_sum(m2) / (float)Dx + a.eps);
      for (int k = lane; k < Dx; k += 32) xr[k] = fsilu((xr[k] - mean) * rstd * LNXG[k] + LNXB[k]);
      if (lane == 0 && cta == ((t + 1) % SCAN_G)) {
        ws.ln_stats[((size_t)0 * NB + row0 + b) * 2] = mean;
        ws.ln_stats[((size_t)0 * NB + row0 + b) * 2 + 1] = rstd;
      }
    }
    __syncthreads();
    if (sX.ok) a.x_act[(row0 + sX.b) * Dx + sX.col] = Xx[sX.b * xxs + sX.col];
    prof_mark(prof, 4, tlast, prof_on);
    const int ksx = product(Xx, xxs, Wg + g.sR, g.wgst, g.ngh * 3, Dx, B, PART, ldp, 0, tid);
    __syncthreads();
    float gpre = 0.f;
    if (pok) {
      gpre = acch + part_sum(PART, ldp, ksx, pb, pc);
      ACC[pb * ldp + pc] = gpre;
    }
    __syncthreads();
    for (int b = wid; b < B; b += SCAN_NW) {   // per-row partial statistics (mean, M2) over the owned valid columns
      float s = 0.f;
      for (int c = lane; c < nh12; c += 32)
        if ((cta + (c / 12) * SCAN_G) * 4 + (c & 3) < R) s += ACC[b * ldp + c];
      s = warp_sum(s);
      const float mean = ncol3 > 0 ? s / (float)ncol3 : 0.f;
      float m2 = 0.f;
      for (int c = lane; c < nh12; c += 32)
        if ((cta + (c / 12) * SCAN_G) * 4 + (c & 3) < R) { const float d = ACC[b * ldp + c] - mean; m2 = fmaf(d, d, m2); }
      m2 = warp_sum(m2);
      if (lane == 0) ll_store2(ws.ll + L.s + (((size_t)par * MAXB + b) * SCAN_G + cta) * 2, mean, m2, tag);
    }
    if (pok) a.g_pre[(row0 + pb) * 3 * R + ppart * R + pcol] = gpre;      // save after the hand-off
    prof_mark(prof, 5, tlast, prof_on);

    // ============ C: merge statistics (Chan), LayerNorm, GRU gate -> h_t for the owned columns.  The element's LayerNorm
    // parameters are loaded here, in flight during the wait (kept in registers across the whole step, they were spilled)
    float lg_g[3] = {0.f, 0.f, 0.f}, lg_b[3] = {0.f, 0.f, 0.f};
    if (sH.ok)
#pragma unroll
      for (int part = 0; part < 3; ++part) { lg_g[part] = a.lng_g[part * R + sH.col]; lg_b[part] = a.lng_b[part * R + sH.col]; }
    for (int b0 = wid; b0 < B; b0 += 2 * SCAN_NW) {          // a warp merges up to two rows, all their loads in flight
      u64 x[2][SCAN_G / 32], y[2][SCAN_G / 32];
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        const int b = b0 + rr * SCAN_NW;
        if (b < B)
#pragma unroll
          for (int i = 0; i < SCAN_G / 32; ++i)
            ll_load2(ws.ll + L.s + (((size_t)par * MAXB + b) * SCAN_G + lane + 32 * i) * 2, x[rr][i], y[rr][i]);
      }
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        const int b = b0 + rr * SCAN_NW;
        if (b >= B) continue;
        float pm[SCAN_G / 32], pq[SCAN_G / 32];
        for (;;) {                                 // stale partials are re-polled together
          bool stale = false;
#pragma unroll
          for (int i = 0; i < SCAN_G / 32; ++i)
            if ((unsigned)(x[rr][i] >> 32) != tag || (unsigned)(y[rr][i] >> 32) != tag) stale = true;
          if (!stale || sp.fail()) break;
#pragma unroll
          for (int i = 0; i < SCAN_G / 32; ++i)
            if ((unsigned)(x[rr][i] >> 32) != tag || (unsigned)(y[rr][i] >> 32) != tag)
              ll_load2(ws.ll + L.s + (((size_t)par * MAXB + b) * SCAN_G + lane + 32 * i) * 2, x[rr][i], y[rr][i]);
        }
#pragma unroll
        for (int i = 0; i < SCAN_G / 32; ++i) {
          pm[i] = __uint_as_float((unsigned)x[rr][i]);
          pq[i] = __uint_as_float((unsigned)y[rr][i]);
        }
        float sm_ = 0.f;
#pragma unroll
        for (int i = 0; i < SCAN_G / 32; ++i) sm_ += (float)(3 * nctab[lane + 32 * i]) * pm[i];
        const float mean = warp_sum(sm_) / (float)(3 * R);
        float m2 = 0.f;
#pragma unroll
        for (int i = 0; i < SCAN_G / 32; ++i) {
          const float d = pm[i] - mean;
          m2 += pq[i] + (float)(3 * nctab[lane + 32 * i]) * d * d;
        }
        m2 = warp_sum(m2);
        if (lane == 0) {
          const float rstd = rsqrtf(m2 / (float)(3 * R) + a.eps);
          misc[16 + b] = mean;
          misc[32 + b] = rstd;
          if (cta == ((t + 2) % SCAN_G)) {
            ws.ln_stats[((size_t)1 * NB + row0 + b) * 2] = mean;
            ws.ln_stats[((size_t)1 * NB + row0 + b) * 2 + 1] = rstd;
          }
        }
      }
    }
    __syncthreads();
    prof_mark(prof, 6, tlast, prof_on);
    if (sH.ok) {
      const int b = sH.b, gi = sH.cj >> 2, j = sH.cj & 3;
      const float mu = misc[16 + b], rstd = misc[32 + b];
      float gl[3];
#pragma unroll
      for (int part = 0; part < 3; ++part)
        gl[part] = (ACC[b * ldp + gi * 12 + part * 4 + j] - mu) * rstd * lg_g[part] + lg_b[part];
      const float r = sigmoidf_(gl[0]);
      const float c = tanhf(r * gl[1]);
      const float u = sigmoidf_(gl[2] - 1.f);
      const float h = u * c + (1.f - u) * hin;
      ll_store(ws.ll + L.h + ((size_t)par * MAXB + b) * R + sH.col, h, tag);      // hand-off first, saves after
      a.latent[(row0 + b) * a.ld_lat + Z + sH.col] = h;
#pragma unroll
      for (int part = 0; part < 3; ++part) a.g_ln[(row0 + b) * 3 * R + part * R + sH.col] = gl[part];
      a.h_in[(row0 + b) * R + sH.col] = hin;
    }
    prof_mark(prof, 7, tlast, prof_on);

    // ============ D: rp_pre = h W_r1[:, :R]^T + pe for the owned columns (h rows stay in Xh for the next step)
    ll_recv<8>(Xh, g.sR, ws.ll + L.h + (size_t)par * MAXB * R, R, B, R, tag, tid, sp);   // (own h_in was read above, into `hin`)
    __syncthreads();
    prof_mark(prof, 8, tlast, prof_on);
    const int ksr = product(Xh, g.sR, Wr1, g.sR, g.ngr, R, B, PART, ldp, 0, tid);
    __syncthreads();
    if (sR_.ok) {
      const float v = part_sum(PART, ldp, ksr, sR_.b, sR_.cj) + pe_pref;
      ll_store(ws.ll + L.r + ((size_t)par * MAXB + sR_.b) * Dr + sR_.col, v, tag);
      a.rp_pre[(row0 + sR_.b) * Dr + sR_.col] = v;
    }
    prof_mark(prof, 9, tlast, prof_on);

    // ============ E (sampling unit): LN + SiLU of the unit's rows, logits of its group, unimix, sample
    if (sampler) {
      const int gq = g.unit_g, nr = g.unit_nr, rb = g.unit_r0;
      __syncthreads();                       // PART / Xx free
      ll_recv<8>(Xx, xxs, ws.ll + L.r + ((size_t)par * MAXB + rb) * Dr, Dr, nr, Dr, tag, tid, sp);
      __syncthreads();
      prof_mark(prof, 10, tlast, prof_on);
      {
        // LayerNorm + SiLU with all warps: wpr warps share a row (nrp = rows rounded up to a power of two)
        const int nrp = nr <= 1 ? 1 : (nr <= 2 ? 2 : (nr <= 4 ? 4 : 8));
        const int wpr = SCAN_NW / nrp, bb = wid / wpr, wi = wid - bb * wpr;
        float* xr = Xx + bb * xxs;
        // one pass, one barrier: sum and sum of squares together (rp_pre is O(1): the E[x^2] - mean^2 form costs ~1e-7
        // relative here, far inside the tolerance; the two-barrier centred form cost 1 k cycles of the critical path)
        float s = 0.f, q2 = 0.f;
        if (bb < nr)
          for (int k = wi * 32 + lane; k < Dr; k += wpr * 32) { const float xv = xr[k]; s += xv; q2 = fmaf(xv, xv, q2); }
        s = warp_sum(s);
        q2 = warp_sum(q2);
        if (lane == 0) { misc[48 + wid] = s; misc[80 + wid] = q2; }
        __syncthreads();
        float mu = 0.f, var = 0.f;
        for (int i = 0; i < wpr; ++i) { mu += misc[48 + bb * wpr + i]; var += misc[80 + bb * wpr + i]; }
        mu /= (float)Dr;
        var = fmaxf(var / (float)Dr - mu * mu, 0.f);
        const float rstd = rsqrtf(var + a.eps);
        if (bb < nr) {
          for (int k = wi * 32 + lane; k < Dr; k += wpr * 32) {
            const float o = fsilu((xr[k] - mu) * rstd * LNRG[k] + LNRB[k]);
            xr[k] = o;
            if (gq == 0) a.rp_act[(row0 + rb + bb) * Dr + k] = o;
          }
          if (gq == 0 && wi == 0 && lane == 0) {
            ws.ln_stats[((size_t)2 * NB + row0 + rb + bb) * 2] = mu;
            ws.ln_stats[((size_t)2 * NB + row0 + rb + bb) * 2 + 1] = rstd;
          }
        }
      }
      __syncthreads();
      prof_mark(prof, 14, tlast, prof_on);
      // logits: lane = class, warp = (K slice, row phase)
      class_product(Xx, xxs, W2, g.w2st, D, g.sDr, nr, PART, tid);
      __syncthreads();
      prof_mark(prof, 15, tlast, prof_on);
      // one warp per row: the D classes of the group live on the lanes (D <= 32)
      if (wid < nr) {
        const int bb = wid, b = rb + bb;
        const bool on = lane < D;
        float lg = 0.f;
        for (int s2 = 0; s2 < CLS_SLICES; ++s2) lg += PART[((size_t)s2 * MAXRPU + bb) * 32 + lane];
        const float raw = on ? lg + bias2 : -INFINITY;
        const float mx = warp_max(raw);
        const float ex = on ? expf(raw - mx) : 0.f;
        const float se = warp_sum(ex);
        // unimix (agent.py:437-449); Categorical(logits=l).probs is proportional to the clamped mixture pmc, so the draw
        // argmax(probs / q) (torch.multinomial) equals argmax(pmc / q): the normaliser is common to all classes
        float pmc = ex / se, l = raw;
        if (a.unimix > 0.f) {
          pmc = fminf(fmaxf((1.f - a.unimix) * pmc + a.unimix / (float)D, kFp32Eps), 1.f - kFp32Eps);
          l = logf(pmc);
        }
        float best = on ? pmc / noise_pref : -INFINITY;
        int besti = on ? lane : 0x7fffffff;
#pragma unroll
        for (int s2 = 16; s2 > 0; s2 >>= 1) {
          const float ob = __shfl_xor_sync(0xffffffffu, best, s2);
          const int oi = __shfl_xor_sync(0xffffffffu, besti, s2);
          if (ob > best || (ob == best && oi < besti)) { best = ob; besti = oi; }
        }
        if (lane == 0) ll_store(ws.ll + L.z + ((size_t)par * MAXB + b) * S + gq, __uint_as_float((unsigned)besti), tag);
        // saves after the hand-off
        const size_t o = (row0 + b) * Z + (size_t)gq * D + lane;
        if (lane == 0) ws.zidx[(row0 + b) * S + gq] = besti;
        if (on) {
          a.post_raw[o] = raw;
          a.post_mix[o] = l;
          const float zt = (lane == besti) ? 1.f : 0.f;
          a.latent[(row0 + b) * a.ld_lat + (size_t)gq * D + lane] = zt;
          if (t + 1 < T)     // z_in of the next step: (1-f) z_t + f z0 (agent.py:430), both one-hot
            a.z_in[(row0 + B + b) * Z + (size_t)gq * D + lane] = (1.f - fnext) * zt + fnext * ((z0idx[gq] == lane) ? 1.f : 0.f);
        }
      }
      prof_mark(prof, 11, tlast, prof_on);
    }
    __syncthreads();
    if (sp.dead) break;    // a hand-off timed out somewhere: bail out, never hang
  }
  if (prof_on)
    for (int i = 0; i < 32; ++i) ws.prof[cta * 32 + i] = sprof[i];
}

// =====================================================================================================
// backward (BPTT); consumes the activations, LayerNorm statistics and class indices saved by the forward kernel.
//
// Per step (t = T-1 .. 0) the gradient walks  z_t -> post logits -> rp -> h_t -> gates -> (h_{t-1}, x_t) -> z_{t-1}.
// LayerNorm backward  d_pre = rstd (dxh - mean(dxh) - xh mean(dxh xh))  is NOT a hand-off of its own: the producer
// sends dxh = d_act * act'(ln) * gamma for its columns together with its partial row sums, and the CONSUMER of d_pre
// (always a product d_pre W) applies the correction through linearity:
//     d_pre W = rstd (dxh W  -  S1 colsum(W)  -  S2 (xh W)),      xh W = rstd (pre W - mu colsum(W))
// where `pre W` does not depend on the backward chain: it is one batched tensor-core product per LayerNorm over all
// T*B rows, done before this kernel (q.q_r / q.q_g / q.q_x).  The d_pre rows themselves (operands of the deferred
// weight-gradient products) are produced afterwards by the batched LayerNorm-backward kernels from the d_act rows
// saved here.  That leaves four hand-offs per step: d_post_raw rows, dxh of the representation LayerNorm, dxh of the
// GRU LayerNorm, dxh of the x LayerNorm; the last one is consumed by the CTA that owns the (rows, categorical group)
// block, which immediately turns it into the next step's d_post_raw (straight-through + unimix + softmax backward).
// =====================================================================================================
struct GeoB {
  int ngh, ngx, ngr;            // owned 4-column groups of R (dh), Dx (d_x_act), Dr (d_rp_act)
  int sZ, sR, sDx, sDr, xw;     // padded widths; width of the row staging buffer
  int wgst, winst;              // smem row strides of the W_g^T slice (3 parts of sR) and the unit's W_in slice
  int nsplit, rpu, unit_g, unit_r0, unit_nr;
  int ldp;
  int oW2, oW1, oWg, oWin, oX, oPart, oAcc, oSt, oDhc, oDh0, oWs, oMisc, total;
};

__host__ __device__ inline GeoB make_geo_b(const Dims& a, int cta) {
  GeoB g;
  const int Z = a.S * a.D;
  g.ngh = owned_groups(a.R, cta);
  g.ngx = owned_groups(a.Dx, cta);
  g.ngr = owned_groups(a.Dr, cta);
  g.sZ = r4(Z); g.sR = r4(a.R); g.sDx = r4(a.Dx); g.sDr = r4(a.Dr);
  g.xw = imax(imax(g.sZ, 2 * g.sR), imax(g.sDx, g.sDr));
  g.wgst = 3 * g.sR;
  g.winst = g.sDx + 4;
  g.nsplit = imax(1, imin(a.B, SCAN_G / a.S));
  g.rpu = (a.B + g.nsplit - 1) / g.nsplit;
  g.unit_g = -1; g.unit_r0 = 0; g.unit_nr = 0;
  if (cta < a.S * g.nsplit) {
    const int sp = cta / a.S;
    g.unit_r0 = sp * g.rpu;
    g.unit_nr = imin(g.rpu, a.B - g.unit_r0);
    if (g.unit_nr > 0) g.unit_g = cta % a.S; else g.unit_nr = 0;
  }
  const int mh = owned_groups(a.R, 0), mx = owned_groups(a.Dx, 0), mr = owned_groups(a.Dr, 0);
  g.ldp = imax(imax((mh + mx) * 4, mr * 4), 4);
  int o = 0;
  g.oW2 = o;   o += mr * 4 * g.sZ;             // W_r2[:, c]  (own d_rp_act columns)
  g.oW1 = o;   o += mh * 4 * g.sDr;            // W_r1[:, j]  (own dh columns)
  g.oWg = o;   o += (mh + mx) * 4 * g.wgst;    // W_g[:, j] (h part) then W_g[:, R + c] (x part), 3 parts of sR each
  g.oWin = o;  o += a.D * g.winst;             // W_in[:, gq*D + d] of the unit's group
  g.oX = o;    o += MAXB * g.xw;
  g.oPart = o; o += imax(KS_MAX * MAXB * g.ldp, CLS_SLICES * MAXRPU * 32);
  g.oAcc = o;  o += MAXB * g.ldp;
  g.oSt = o;   o += 2 * MAXB * imax(imax(mh * 12, mx * 4), imax(mr * 4, 4));   // (dxh, dxh*xh) staging for the row sums
  g.oDhc = o;  o += MAXB * imax(mh * 4, 4);
  g.oDh0 = o;  o += imax(mh * 4, 4);
  g.oWs = o;   o += mh * 4 + (mh + mx) * 4 + 32;   // column sums of the weight slices
  g.oMisc = o; o += 16 * MAXB + 64;
  g.total = o;
  return g;
}

// per-row sums of the staged (dxh, dxh*xh) pairs of this CTA's columns -> LL partial for every row
__device__ __forceinline__ void send_row_sums(const float* ST, int ncols, int B, u64* base, int par, int cta, unsigned tag, int tid) {
  const int lane = tid & 31, wid = tid >> 5;
  for (int b = wid; b < B; b += SCAN_NW) {
    float s1 = 0.f, s2 = 0.f;
    for (int c = lane; c < ncols; c += 32) { s1 += ST[(b * ncols + c) * 2]; s2 += ST[(b * ncols + c) * 2 + 1]; }
    s1 = warp_sum(s1); s2 = warp_sum(s2);
    if (lane == 0) ll_store2(base + (((size_t)par * MAXB + b) * SCAN_G + cta) * 2, s1, s2, tag);
  }
}

template <bool FIX>
__global__ void __launch_bounds__(SCAN_NT, 1)
rssm_scan_bwd_kernel(const b200rl_rssm_scan_args a, const b200rl_rssm_scan_grads q) {
  extern __shared__ __align__(16) float sm[];
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int cta = blockIdx.x;
  const int T = a.T, B = a.B;
  const int S = FIX ? 32 : a.S, D = FIX ? 32 : a.D, Z = S * D, R = FIX ? 512 : a.R, Dx = FIX ? 512 : a.Dx, Dr = FIX ? 512 : a.Dr;
  const int KG = R + Dx, KIN = Z + a.A, NB = T * B;
  const GeoB g = make_geo_b(Dims{B, S, D, R, Dx, Dr, a.A}, cta);
  const Workspace ws = carve(a.workspace, T, B, S, D, Dx, R, Dr);
  const LLGeo L = make_ll(S, Dx, R, Dr, Z);
  const int mh = owned_groups(R, 0), mx = owned_groups(Dx, 0);
  float* W2T = sm + g.oW2;      // [ngr*4][sZ]
  float* W1T = sm + g.oW1;      // [ngh*4][sDr]
  float* WgT = sm + g.oWg;      // [(ngh+ngx)*4][3*sR]
  float* WinU = sm + g.oWin;    // [D][winst]
  float* X = sm + g.oX;         // [MAXB][xw]
  float* PART = sm + g.oPart;
  float* ACC = sm + g.oAcc;     // [MAXB][ldp]
  float* ST = sm + g.oSt;       // [(b, col)][2] staged (dxh, dxh*xh)
  float* DHC = sm + g.oDhc;     // [MAXB][nh4] dh carried to step t-1
  float* DH0 = sm + g.oDh0;     // [nh4] accumulated grad of tanh(initial_recurrent_state)
  float* WS1 = sm + g.oWs;      // [nh4] column sums of the W_r1 slice
  float* WSG = WS1 + mh * 4;    // [(ngh+ngx)*4] column sums of the W_g slice
  float* WSI = WSG + (mh + mx) * 4;   // [D] column sums of the unit's W_in slice
  float* misc = sm + g.oMisc;   // [0,16) first(t); [16,32) first(t+1); [32,48) S1; [48,64) S2; [64,..) per-row (mu, rstd) x3
  float* S1 = misc + 32;
  float* S2 = misc + 48;
  float* LNS = misc + 64;       // [3][MAXB][2]: x, g, rp LayerNorm statistics of step t
  float* LNX1 = misc + 64 + 6 * MAXB;   // [MAXB][2]: x LayerNorm statistics of step t+1 (units)
  const int xw = g.xw, ldp = g.ldp;
  const int nh4 = g.ngh * 4, nx4 = g.ngx * 4, nr4 = g.ngr * 4;
  const bool unit = g.unit_g >= 0;
  __shared__ long long sprof[32];
  const bool prof_on = (cta < 2) && tid == 0;
  long long* prof = sprof;
  if (tid < 32) sprof[tid] = 0;
  long long tlast = prof_on ? clock64() : 0;
  Spin sp;
  sp.init(ws.error);

  // ---------------- prologue: zero everything, then transposed weight slices -> shared memory, column sums
  for (int e = tid; e < g.total; e += SCAN_NT) sm[e] = 0.f;
  __syncthreads();
  for (int gi = 0; gi < g.ngr; ++gi)
    load_cols4(W2T + (size_t)gi * 4 * g.sZ, g.sZ, a.W_r2, Dr, (cta + gi * SCAN_G) * 4, Dr, Z, 0, tid);
  for (int gi = 0; gi < g.ngh; ++gi) {
    const int c0 = (cta + gi * SCAN_G) * 4;
    load_cols4(W1T + (size_t)gi * 4 * g.sDr, g.sDr, a.W_r1, a.ld_wr1, c0, R, Dr, 0, tid);
    for (int part = 0; part < 3; ++part)
      load_cols4(WgT + (size_t)gi * 4 * g.wgst, g.wgst, a.W_g + (size_t)part * R * KG, KG, c0, R, R, part * g.sR, tid);
  }
  for (int gi = 0; gi < g.ngx; ++gi)
    for (int part = 0; part < 3; ++part)
      load_cols4(WgT + (size_t)(g.ngh + gi) * 4 * g.wgst, g.wgst, a.W_g + (size_t)part * R * KG + R, KG,
                 (cta + gi * SCAN_G) * 4, Dx, R, part * g.sR, tid);
  if (unit)
    for (int e = tid; e < D * Dx; e += SCAN_NT) {
      const int c = e / D, d = e - c * D;
      WinU[d * g.winst + c] = a.W_in[(size_t)c * KIN + g.unit_g * D + d];
    }
  __syncthreads();
  for (int j = wid; j < nh4; j += SCAN_NW) {
    float s = 0.f;
    for (int k = lane; k < g.sDr; k += 32) s += W1T[(size_t)j * g.sDr + k];
    s = warp_sum(s);
    if (lane == 0) WS1[j] = s;
  }
  for (int j = wid; j < nh4 + nx4; j += SCAN_NW) {
    float s = 0.f;
    for (int k = lane; k < g.wgst; k += 32) s += WgT[(size_t)j * g.wgst + k];
    s = warp_sum(s);
    if (lane == 0) WSG[j] = s;
  }
  if (unit)
    for (int d = wid; d < D; d += SCAN_NW) {
      float s = 0.f;
      for (int k = lane; k < g.sDx; k += 32) s += WinU[(size_t)d * g.winst + k];
      s = warp_sum(s);
      if (lane == 0) WSI[d] = s;
    }
  __syncthreads();
  // fixed element assignments and per-element parameters (no index arithmetic / parameter loads inside the time loop)
  const Slot sR_ = make_slot(tid, nr4, B, cta, Dr);          // d_rp_act element
  const Slot sH = make_slot(tid, nh4, B, cta, R);            // dh element
  const Slot sX = make_slot(tid, nx4, B, cta, Dx);           // d_x_act element
  const float gam_r = sR_.ok ? a.lnr_g[sR_.col] : 0.f, bet_r = sR_.ok ? a.lnr_b[sR_.col] : 0.f;
  const float gam_x = sX.ok ? a.lnx_g[sX.col] : 0.f, bet_x = sX.ok ? a.lnx_b[sX.col] : 0.f;
  float gam_g[3] = {0.f, 0.f, 0.f};
  if (sH.ok)
#pragma unroll
    for (int part = 0; part < 3; ++part) gam_g[part] = a.lng_g[part * R + sH.col];
  const float ws1 = sH.ok ? WS1[sH.cj] : 0.f, wsgh = sH.ok ? WSG[sH.cj] : 0.f, wsgx = sX.ok ? WSG[nh4 + sX.cj] : 0.f;
  const float wsi = (unit && lane < D) ? WSI[lane] : 0.f;
  float dh0_acc = 0.f;                                        // (threads tid < nh4) accumulated over rows in fixed order
  prof_mark(prof, 16, tlast, prof_on);

  for (int t = T - 1; t >= 0; --t) {
    const size_t row0 = (size_t)t * B;
    const int bt = T - 1 - t, par = bt & 1;
    const unsigned tag = (unsigned)bt + 1u;
    const bool last = (t == T - 1);

    // ---------------- step-start prefetch of chain-independent inputs (registers of the element's thread)
    if (tid < MAXB) {
      misc[tid] = (tid < B) ? a.first[row0 + tid] : 0.f;
      misc[16 + tid] = (tid < B && !last) ? a.first[row0 + B + tid] : 0.f;
    }
    for (int e = tid; e < 3 * B * 2; e += SCAN_NT) {
      const int which = e / (B * 2), r_ = e - which * (B * 2);
      LNS[which * MAXB * 2 + r_] = ws.ln_stats[((size_t)which * NB + row0) * 2 + r_];
    }
    if (!last)
      for (int e = tid; e < B * 2; e += SCAN_NT) LNX1[e] = ws.ln_stats[((size_t)0 * NB + row0 + B) * 2 + e];
    const float p_rp = sR_.ok ? a.rp_pre[(row0 + sR_.b) * Dr + sR_.col] : 0.f;
    float p_hin = 0.f, p_dlh = 0.f, p_qr = 0.f, p_qgh = 0.f, p_gl[3] = {0.f, 0.f, 0.f}, p_gp[3] = {0.f, 0.f, 0.f};
    if (sH.ok) {
      p_hin = a.h_in[(row0 + sH.b) * R + sH.col];
      p_dlh = q.d_latent[(row0 + sH.b) * a.ld_lat + Z + sH.col];
      p_qr = q.q_r[(row0 + sH.b) * R + sH.col];
      p_qgh = q.q_g[(row0 + sH.b) * KG + sH.col];
#pragma unroll
      for (int part = 0; part < 3; ++part) {
        p_gl[part] = a.g_ln[(row0 + sH.b) * 3 * R + part * R + sH.col];
        p_gp[part] = a.g_pre[(row0 + sH.b) * 3 * R + part * R + sH.col];
      }
    }
    const float p_xp = sX.ok ? a.x_pre[(row0 + sX.b) * Dx + sX.col] : 0.f;
    const float p_qgx = sX.ok ? q.q_g[(row0 + sX.b) * KG + R + sX.col] : 0.f;
    // (unit) per-row inputs of the group: one warp per row
    float u_dl = 0.f, u_dmix = 0.f, u_raw = -INFINITY, u_qx = 0.f;
    if (unit && wid < g.unit_nr && lane < D) {
      const size_t o = (row0 + g.unit_r0 + wid) * Z + (size_t)g.unit_g * D + lane;
      u_dl = q.d_latent[(row0 + g.unit_r0 + wid) * a.ld_lat + (size_t)g.unit_g * D + lane];
      u_dmix = q.d_post_mix[o];
      u_raw = a.post_raw[o];
      if (!last) u_qx = q.q_x[(row0 + B + g.unit_r0 + wid) * Z + (size_t)g.unit_g * D + lane];
    }
    __syncthreads();
    const float* fl = misc;

    // ============ P (unit): dz carried from step t+1 through W_in, then the raw-logit gradients of the group
    if (unit) {
      const int gq = g.unit_g, nr = g.unit_nr, rb = g.unit_r0;
      if (!last) {
        ll_recv<4>(X, xw, ws.ll + L.d + ((size_t)(par ^ 1) * MAXB + rb) * Dx, Dx, nr, Dx, (unsigned)bt, tid, sp,
                   ws.ll + L.sd + (size_t)(par ^ 1) * MAXB * SCAN_G * 2, rb, 1.f / (float)Dx, S1, S2);
        __syncthreads();
        prof_mark(prof, 17, tlast, prof_on);
        class_product(X, xw, WinU, g.winst, D, g.sDx, nr, PART, tid);
        __syncthreads();
      }
      if (wid < nr) {
        const int bb = wid, b = rb + bb;
        const bool on = lane < D;
        float dz = u_dl;
        if (!last) {
          float p1 = 0.f;
          for (int s2 = 0; s2 < CLS_SLICES; ++s2) p1 += PART[((size_t)s2 * MAXRPU + bb) * 32 + lane];
          if (on) {
            const float mu = LNX1[b * 2], rstd = LNX1[b * 2 + 1];
            const float p2 = rstd * (u_qx - mu * wsi);
            dz += (1.f - fl[16 + b]) * rstd * (p1 - S1[b] * wsi - S2[b] * p2);
          }
        }
        const float mx_ = warp_max(u_raw);
        const float ex = on ? expf(u_raw - mx_) : 0.f;
        const float sft = ex / warp_sum(ex);
        float gg = u_dmix;
        if (a.unimix > 0.f) {
          const float pmx = (1.f - a.unimix) * sft + a.unimix / (float)D;
          const float pmc = on ? fminf(fmaxf(pmx, kFp32Eps), 1.f - kFp32Eps) : 0.f;
          const float p = pmc / warp_sum(pmc);          // Categorical(logits = log pmc).probs
          const float pdz = warp_sum(p * dz);
          gg += p * (dz - pdz);                          // straight-through sample: d/dlogits of probs . dz
          const bool inside = on && pmx >= kFp32Eps && pmx <= 1.f - kFp32Eps;
          const float ds = inside ? gg * (1.f - a.unimix) / pmx : 0.f;
          const float sds = warp_sum(sft * ds);
          gg = sft * (ds - sds);
        } else {
          const float pdz = warp_sum(sft * dz);
          gg += sft * (dz - pdz);
        }
        if (on) {
          ll_store(ws.ll + L.a + ((size_t)par * MAXB + b) * Z + (size_t)gq * D + lane, gg, tag);
          q.d_post_raw[(row0 + b) * Z + (size_t)gq * D + lane] = gg;
        }
      }
      prof_mark(prof, 18, tlast, prof_on);
    }

    // ============ Q: d_rp_act = d_post_raw W_r2 for the owned columns; dxh of the representation LayerNorm
    __syncthreads();
    ll_recv<4>(X, xw, ws.ll + L.a + (size_t)par * MAXB * Z, Z, B, Z, tag, tid, sp);
    __syncthreads();
    prof_mark(prof, 19, tlast, prof_on);
    const int ks2 = product(X, xw, W2T, g.sZ, g.ngr, Z, B, PART, ldp, 0, tid);
    __syncthreads();
    float dact_r = 0.f;
    if (sR_.ok) {
      dact_r = part_sum(PART, ldp, ks2, sR_.b, sR_.cj);
      const float xh = (p_rp - LNS[(2 * MAXB + sR_.b) * 2]) * LNS[(2 * MAXB + sR_.b) * 2 + 1];
      const float ln = xh * gam_r + bet_r;
      const float sg = sigmoidf_(ln);
      const float dxh = dact_r * sg * (1.f + ln * (1.f - sg)) * gam_r;
      ll_store(ws.ll + L.b + ((size_t)par * MAXB + sR_.b) * Dr + sR_.col, dxh, tag);
      ST[(sR_.b * nr4 + sR_.cj) * 2] = dxh;
      ST[(sR_.b * nr4 + sR_.cj) * 2 + 1] = dxh * xh;
    } else if (tid < B * nr4) {
      ST[tid * 2] = 0.f; ST[tid * 2 + 1] = 0.f;
    }
    __syncthreads();
    send_row_sums(ST, nr4, B, ws.ll + L.sb, par, cta, tag, tid);
    if (sR_.ok) q.d_rp_act[(row0 + sR_.b) * Dr + sR_.col] = dact_r;
    prof_mark(prof, 20, tlast, prof_on);

    // ============ R: dh = d_latent_h + carry + d_rp_pre W_r1h ; GRU gate backward ; dxh of the GRU LayerNorm
    __syncthreads();
    ll_recv<4>(X, xw, ws.ll + L.b + (size_t)par * MAXB * Dr, Dr, B, Dr, tag, tid, sp,
               ws.ll + L.sb + (size_t)par * MAXB * SCAN_G * 2, 0, 1.f / (float)Dr, S1, S2);
    __syncthreads();
    prof_mark(prof, 21, tlast, prof_on);
    const int ks1 = product(X, xw, W1T, g.sDr, g.ngh, Dr, B, PART, ldp, 0, tid);
    __syncthreads();
    float dhin_gate = 0.f, dgl[3] = {0.f, 0.f, 0.f};
    if (sH.ok) {
      const int b = sH.b;
      const float mur = LNS[(2 * MAXB + b) * 2], rstdr = LNS[(2 * MAXB + b) * 2 + 1];
      const float mug = LNS[(1 * MAXB + b) * 2], rstdg = LNS[(1 * MAXB + b) * 2 + 1];
      const float p1 = part_sum(PART, ldp, ks1, b, sH.cj);
      const float p2 = rstdr * (p_qr - mur * ws1);
      float dh = p_dlh + rstdr * (p1 - S1[b] * ws1 - S2[b] * p2);
      if (!last) dh += DHC[b * nh4 + sH.cj];
      const float r = sigmoidf_(p_gl[0]), cnd = tanhf(r * p_gl[1]), u = sigmoidf_(p_gl[2] - 1.f);
      const float du = dh * (cnd - p_hin);
      const float drc = dh * u * (1.f - cnd * cnd);
      dgl[0] = drc * p_gl[1] * r * (1.f - r);
      dgl[1] = drc * r;
      dgl[2] = du * u * (1.f - u);
      dhin_gate = dh * (1.f - u);
#pragma unroll
      for (int part = 0; part < 3; ++part) {
        const float xh = (p_gp[part] - mug) * rstdg;
        const float dxh = dgl[part] * gam_g[part];
        ll_store(ws.ll + L.c + ((size_t)par * MAXB + b) * 3 * R + (size_t)part * R + sH.col, dxh, tag);
        ST[(b * (3 * nh4) + part * nh4 + sH.cj) * 2] = dxh;
        ST[(b * (3 * nh4) + part * nh4 + sH.cj) * 2 + 1] = dxh * xh;
      }
    } else if (tid < B * nh4) {
      const int b = tid / imax(nh4, 1), cj = tid - b * nh4;
#pragma unroll
      for (int part = 0; part < 3; ++part) {
        ST[(b * (3 * nh4) + part * nh4 + cj) * 2] = 0.f;
        ST[(b * (3 * nh4) + part * nh4 + cj) * 2 + 1] = 0.f;
      }
    }
    __syncthreads();
    send_row_sums(ST, 3 * nh4, B, ws.ll + L.sc, par, cta, tag, tid);
    if (sH.ok)
#pragma unroll
      for (int part = 0; part < 3; ++part) q.d_g_ln[(row0 + sH.b) * 3 * R + part * R + sH.col] = dgl[part];
    prof_mark(prof, 22, tlast, prof_on);

    // ============ S: [dh_in, d_x_act] = d_g_pre W_g for the owned columns (K = 3R: parts r,c together, then u)
    __syncthreads();
    for (int part = 0; part < 2; ++part)
      ll_recv<4>(X + part * g.sR, xw, ws.ll + L.c + (size_t)par * MAXB * 3 * R + (size_t)part * R, 3 * R, B, R, tag, tid, sp);
    __syncthreads();
    const int ksa = product(X, xw, WgT, g.wgst, g.ngh + g.ngx, 2 * g.sR, B, PART, ldp, 0, tid);
    __syncthreads();
    float acc_h = sH.ok ? part_sum(PART, ldp, ksa, sH.b, sH.cj) : 0.f;
    float acc_x = sX.ok ? part_sum(PART, ldp, ksa, sX.b, nh4 + sX.cj) : 0.f;
    __syncthreads();
    ll_recv<4>(X, xw, ws.ll + L.c + (size_t)par * MAXB * 3 * R + (size_t)2 * R, 3 * R, B, R, tag, tid, sp,
               ws.ll + L.sc + (size_t)par * MAXB * SCAN_G * 2, 0, 1.f / (float)(3 * R), S1, S2);
    __syncthreads();
    const int ksb = product(X, xw, WgT + 2 * g.sR, g.wgst, g.ngh + g.ngx, R, B, PART, ldp, 0, tid);
    __syncthreads();
    prof_mark(prof, 23, tlast, prof_on);
    float dact_x = 0.f;
    if (sX.ok) {
      const int b = sX.b;
      acc_x += part_sum(PART, ldp, ksb, b, nh4 + sX.cj);
      const float mug = LNS[(1 * MAXB + b) * 2], rstdg = LNS[(1 * MAXB + b) * 2 + 1];
      const float mux = LNS[(0 * MAXB + b) * 2], rstdx = LNS[(0 * MAXB + b) * 2 + 1];
      const float p2 = rstdg * (p_qgx - mug * wsgx);
      dact_x = rstdg * (acc_x - S1[b] * wsgx - S2[b] * p2);
      const float xh = (p_xp - mux) * rstdx;
      const float ln = xh * gam_x + bet_x;
      const float sg = sigmoidf_(ln);
      const float dxh = dact_x * sg * (1.f + ln * (1.f - sg)) * gam_x;
      ll_store(ws.ll + L.d + ((size_t)par * MAXB + b) * Dx + sX.col, dxh, tag);
      ST[(b * nx4 + sX.cj) * 2] = dxh;
      ST[(b * nx4 + sX.cj) * 2 + 1] = dxh * xh;
    } else if (tid < B * nx4) {
      ST[tid * 2] = 0.f; ST[tid * 2 + 1] = 0.f;
    }
    float dhin_f = 0.f;
    if (sH.ok) {
      const int b = sH.b;
      acc_h += part_sum(PART, ldp, ksb, b, sH.cj);
      const float mug = LNS[(1 * MAXB + b) * 2], rstdg = LNS[(1 * MAXB + b) * 2 + 1];
      const float p2 = rstdg * (p_qgh - mug * wsgh);
      const float dhin = dhin_gate + rstdg * (acc_h - S1[b] * wsgh - S2[b] * p2);
      DHC[b * nh4 + sH.cj] = (1.f - fl[b]) * dhin;          // carried to step t-1 (agent.py:428 mask)
      dhin_f = fl[b] * dhin;                                // grad of tanh(initial_recurrent_state)
    }
    __syncthreads();
    send_row_sums(ST, nx4, B, ws.ll + L.sd, par, cta, tag, tid);
    if (sX.ok) q.d_x_act[(row0 + sX.b) * Dx + sX.col] = dact_x;
    // d_h0: sum over the rows with is_first set, fixed row order (bit-reproducible): stage through ACC
    if (sH.ok) ACC[sH.b * ldp + sH.cj] = dhin_f;
    __syncthreads();
    if (tid < nh4)
      for (int b = 0; b < B; ++b)
        if (fl[b] != 0.f) dh0_acc += ACC[b * ldp + tid];
    prof_mark(prof, 24, tlast, prof_on);
    __syncthreads();
    if (sp.dead) break;    // a hand-off timed out somewhere: bail out, never hang
  }
  if (tid < nh4) {
    const int col = (cta + (tid >> 2) * SCAN_G) * 4 + (tid & 3);
    if (col < R) q.d_h0[col] = dh0_acc;
  }
  (void)DH0;
  if (prof_on)
    for (int i = 0; i < 32; ++i) ws.prof[cta * 32 + i] = sprof[i];
}

// the BASELINE S model runs the instantiation with compile-time widths
bool fixed_dims(const b200rl_rssm_scan_args& a) { return a.S == 32 && a.D == 32 && a.R == 512 && a.Dx == 512 && a.Dr == 512; }

size_t scan_smem(const b200rl_rssm_scan_args& a, bool backward) {
  const Dims d{a.B, a.S, a.D, a.R, a.Dx, a.Dr, a.A};
  return sizeof(float) * (size_t)(backward ? make_geo_b(d, 0).total : make_geo_f(d, 0).total);
}

// the envelope of one direction: dims and the shared-memory budget (the backward needs more of it than the forward)
int scan_check(const b200rl_rssm_scan_args& a, bool backward) {
  RL_CHECK_ARG(a.B >= 1 && a.B <= MAXB, "persistent scan supports batch <= 16 rows per rank");
  RL_CHECK_ARG(a.D >= 1 && a.D <= 32, "persistent scan supports <= 32 classes per categorical");
  RL_CHECK_ARG(a.T >= 1 && a.S >= 1 && a.S <= 64, "persistent scan supports T >= 1 and 1 <= S <= 64 categoricals");
  RL_CHECK_ARG(a.Dx % 2 == 0 && a.R % 2 == 0 && a.Dr % 2 == 0 && (a.S * a.D) % 2 == 0, "persistent scan supports even layer widths");
  // at most two 4-column groups of x_pre per CTA: the widest owned share the tests run (Dx = 1024)
  RL_CHECK_ARG(a.Dx <= 1024, "persistent scan supports recurrent dense_units <= 1024");
  // one element of every per-step epilogue per thread (fixed assignments, rssm_scan.cu `Slot`)
  RL_CHECK_ARG(MAXB * owned_groups(a.R, 0) * 12 <= SCAN_NT, "persistent scan supports recurrent_state_size <= 1024");
  RL_CHECK_ARG(MAXB * owned_groups(a.Dr, 0) * 4 <= SCAN_NT, "persistent scan supports representation hidden_size <= 4096");
  RL_CHECK_ARG(scan_smem(a, backward) <= 227 * 1024, "weight slices do not fit in shared memory for this model size");
  return B200RL_OK;
}

int workspace_check(const b200rl_rssm_scan_args& a) {
  RL_CHECK_ARG(a.workspace && a.workspace_bytes >= (long long)ws_bytes(a.T, a.B, a.S, a.D, a.Dx, a.R, a.Dr), "workspace too small");
  return B200RL_OK;
}

// =====================================================================================================
// GRU-only scan (decoupled RSSM, agent.py:501-593 / dreamer_v3.py:115-129).  The posterior is a function of the embedding
// alone there, so z of every step, x = SiLU(LN(W_in [z, a])) and x's share of the gate pre-activation are batched products
// over all T*B rows outside these kernels; what stays on the recurrence is
//   forward   h_in = (1-f) h_{t-1} + f h0 --W_g[:, :R]--> (+ x share) g_pre --LN over 3R--> gates --> h_t
//   backward  dh_t --gates--> d_g_ln --LN--> d_g_pre --W_g[:, :R]--> dh_in --(1-f) / f--> dh_{t-1}, d_h0
// Same construction as the kernels above and on their helpers.  A CTA owns the r, c, u columns of the SAME h columns, so
// the gate is local and its W_g[:, :R] slice stays in shared memory for all T steps.  Two hand-offs per forward step (the
// LayerNorm partial statistics; the h rows — the statistics do not ride with the values: every CTA would then have to
// read all 3R pre-activations of every row instead of 128 partials) and one per backward step (the LayerNorm-backward
// inputs dxh of all 3R columns together with their row sums; the correction is applied by the consumer through
// q_g = g_pre W_g[:, :R], one batched product in front of the kernel).
// =====================================================================================================
struct GruLL { size_t s, h, c, sc, total; };      // offsets (u64 elements), double-buffered by step parity
__host__ __device__ inline GruLL make_gru_ll(int R) {
  GruLL g;
  size_t o = 0;
  g.s = o;  o += 2 * (size_t)MAXB * SCAN_G * 2;   // forward: partial statistics of the GRU LayerNorm
  g.h = o;  o += 2 * (size_t)MAXB * R;            //          h rows
  g.c = o;  o += 2 * (size_t)MAXB * 3 * R;        // backward: dxh of the GRU LayerNorm
  g.sc = o; o += 2 * (size_t)MAXB * SCAN_G * 2;   //           per-CTA row sums (sum dxh, sum dxh*xh)
  g.total = o;
  return g;
}
// workspace: [header 256 B (error word at +64, as above) | LL region (zeroed at every launch) | (mean, rstd) of every row]
__host__ __device__ inline size_t gru_ws_bytes(int T, int B, int R) {
  return WS_HEADER + make_gru_ll(R).total * sizeof(u64) + sizeof(float) * 2 * (size_t)T * B + 256;
}

struct GeoG {
  int ngh, sR, ldp;
  int pw;                        // backward: LayerNorm parts (of 3) staged per product pass — all three where they fit
  int oW, oX, oPart, oAcc, oSt, oDhc, oPar, oLn, oMisc, oTab, total;
};
__host__ __device__ inline GeoG make_geo_g(int R, int cta, bool backward) {
  GeoG g;
  g.ngh = owned_groups(R, cta);
  g.sR = r4(R);
  const int mh = owned_groups(R, 0);
  g.ldp = backward ? mh * 4 : mh * 12;
  for (g.pw = backward ? 3 : 1;; g.pw = 1) {
    int o = 0;
    g.oW = o;    o += mh * 12 * g.sR;            // fwd [ngh*12][sR] rows of W_g[:, :R]; bwd [ngh*4][3*sR] its columns
    g.oX = o;    o += MAXB * g.pw * g.sR;        // fwd h rows; bwd dxh rows
    g.oPart = o; o += KS_MAX * MAXB * g.ldp;
    g.oAcc = o;  o += MAXB * g.ldp;
    g.oSt = o;   o += backward ? 2 * MAXB * mh * 12 : 0;
    g.oDhc = o;  o += backward ? MAXB * mh * 4 : 0;
    g.oPar = o;  o += backward ? mh * 4 : g.sR;  // fwd h0; bwd column sums of the weight slice
    g.oLn = o;   o += mh * 24;                   // LayerNorm weight, bias of the owned columns: [part][gamma, beta][col]
    g.oMisc = o; o += 96;
    g.oTab = o;  o += SCAN_G;
    g.total = o;
    if (g.pw == 1 || sizeof(float) * (size_t)o <= 227 * 1024) break;
  }
  return g;
}

// Merges the per-CTA (mean, M2) partials of one row's LayerNorm statistics (Chan); the whole warp works on the row.
// `cnt[c]`: values CTA c contributed, `n` their total.
__device__ __forceinline__ void merge_row_stats(const u64* base, unsigned tag, const int* cnt, float n, float eps, int lane,
                                                Spin& sp, float& mean, float& rstd) {
  u64 x[SCAN_G / 32], y[SCAN_G / 32];
#pragma unroll
  for (int i = 0; i < SCAN_G / 32; ++i) ll_load2(base + (lane + 32 * i) * 2, x[i], y[i]);
  for (;;) {                                     // stale partials are re-polled together
    bool stale = false;
#pragma unroll
    for (int i = 0; i < SCAN_G / 32; ++i)
      if ((unsigned)(x[i] >> 32) != tag || (unsigned)(y[i] >> 32) != tag) stale = true;
    if (!stale || sp.fail()) break;
#pragma unroll
    for (int i = 0; i < SCAN_G / 32; ++i)
      if ((unsigned)(x[i] >> 32) != tag || (unsigned)(y[i] >> 32) != tag) ll_load2(base + (lane + 32 * i) * 2, x[i], y[i]);
  }
  float sm_ = 0.f;
#pragma unroll
  for (int i = 0; i < SCAN_G / 32; ++i) sm_ += (float)cnt[lane + 32 * i] * __uint_as_float((unsigned)x[i]);
  mean = warp_sum(sm_) / n;
  float m2 = 0.f;
#pragma unroll
  for (int i = 0; i < SCAN_G / 32; ++i) {
    const float d = __uint_as_float((unsigned)x[i]) - mean;
    m2 += __uint_as_float((unsigned)y[i]) + (float)cnt[lane + 32 * i] * d * d;
  }
  rstd = rsqrtf(warp_sum(m2) / n + eps);
}

__global__ void __launch_bounds__(SCAN_NT, 1) gru_scan_fwd_kernel(const b200rl_gru_scan_args a) {
  extern __shared__ __align__(16) float sm[];
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int cta = blockIdx.x;
  const int T = a.T, B = a.B, R = a.R;
  const GeoG g = make_geo_g(R, cta, false);
  const GruLL L = make_gru_ll(R);
  int* error = (int*)((char*)a.workspace + 64);
  u64* ll = (u64*)((char*)a.workspace + WS_HEADER);
  float* ln_stats = (float*)(ll + L.total);
  float* Wg = sm + g.oW;        // [ngh*12][sR]  rows: (group, part r/c/u, col-in-group)
  float* Xh = sm + g.oX;        // [MAXB][sR]  h rows (carried from one step to the next)
  float* PART = sm + g.oPart;
  float* ACC = sm + g.oAcc;     // [MAXB][ldp] finished g_pre columns (for the row statistics)
  float* H0 = sm + g.oPar;      // [R] tanh(initial_recurrent_state)
  float* LNP = sm + g.oLn;      // [3][2][nh4] (read from shared memory at the gate: values kept in registers across the
                                // product / receive calls were spilled)
  float* misc = sm + g.oMisc;   // [0,16) first flags; [16,32) mean; [32,48) rstd
  int* nctab = (int*)(sm + g.oTab);   // LayerNorm values per CTA
  const int ldp = g.ldp;
  Spin sp;
  sp.init(error);

  // ---------------- prologue: the weight slice and h0 -> shared memory (read from HBM once per scan)
  for (int e = tid; e < g.total; e += SCAN_NT) sm[e] = 0.f;
  __syncthreads();
  for (int gi = 0; gi < g.ngh; ++gi)
    for (int part = 0; part < 3; ++part)
      load_rows4(Wg + (size_t)(gi * 3 + part) * 4 * g.sR, g.sR, 0, a.W_g + (size_t)part * R * a.ld_wg, a.ld_wg,
                 (cta + gi * SCAN_G) * 4, R, 0, R, g.sR, tid);
  for (int k = tid; k < R; k += SCAN_NT) H0[k] = a.h0[k];
  for (int c = tid; c < SCAN_G; c += SCAN_NT) nctab[c] = 3 * owned_cols(R, c);
  // fixed element assignments (no index arithmetic inside the time loop)
  const int nh4 = g.ngh * 4, nh12 = g.ngh * 12;
  const Slot sH = make_slot(tid, nh4, B, cta, R);           // gate / h element
  const int pb = nh12 > 0 ? tid / nh12 : 0, pc = tid - pb * nh12;   // g_pre element: (group, part, j) of the 12*ngh products
  const int pcol = (cta + (pc / 12) * SCAN_G) * 4 + (pc & 3), ppart = (pc % 12) >> 2;
  const bool pok = nh12 > 0 && pb < B && pcol < R;
  for (int e = tid; e < 3 * nh4; e += SCAN_NT) {
    const int part = e / nh4, cj = e - part * nh4, col = (cta + (cj >> 2) * SCAN_G) * 4 + (cj & 3);
    LNP[(part * 2) * nh4 + cj] = col < R ? a.lng_g[part * R + col] : 0.f;
    LNP[(part * 2 + 1) * nh4 + cj] = col < R ? a.lng_b[part * R + col] : 0.f;
  }
  const int ncol3 = 3 * owned_cols(R, cta);
  float first_next = (tid < B) ? a.first[tid] : 0.f;        // is_first flags of the step about to run (threads < MAXB)
  __syncthreads();

  for (int t = 0; t < T; ++t) {
    const size_t row0 = (size_t)t * B;
    const int par = t & 1;
    const unsigned tag = (unsigned)t + 1u;
    // operands that do not depend on the chain, before the wait: flags, x's share of the pre-activation
    if (tid < MAXB) misc[tid] = first_next;
    if (tid < MAXB) first_next = (tid < B && t + 1 < T) ? a.first[row0 + B + tid] : 0.f;
    const float gx = pok ? a.g_pre[(row0 + pb) * 3 * R + (size_t)ppart * R + pcol] : 0.f;
    if (t > 0) ll_recv<8>(Xh, g.sR, ll + L.h + (size_t)(par ^ 1) * MAXB * R, R, B, R, (unsigned)t, tid, sp);
    __syncthreads();
    const float* fl = misc;
    // h_in = (1-f) h_{t-1} + f h0 (agent.py:574), rows with f != 0 only
    for (int b = 0; b < B; ++b) {
      const float f = fl[b];
      if (f != 0.f || t == 0)
        for (int k = tid; k < R; k += SCAN_NT) Xh[b * g.sR + k] = (1.f - f) * ((t > 0) ? Xh[b * g.sR + k] : 0.f) + f * H0[k];
    }
    __syncthreads();
    const int ksh = product(Xh, g.sR, Wg, g.sR, g.ngh * 3, R, B, PART, ldp, 0, tid);
    __syncthreads();
    float gpre = 0.f;
    if (pok) {
      gpre = gx + part_sum(PART, ldp, ksh, pb, pc);
      ACC[pb * ldp + pc] = gpre;
    }
    const float hin = sH.ok ? Xh[sH.b * g.sR + sH.col] : 0.f;
    __syncthreads();
    for (int b = wid; b < B; b += SCAN_NW) {   // per-row partial statistics (mean, M2) over the owned valid columns
      float s = 0.f;
      for (int c = lane; c < nh12; c += 32)
        if ((cta + (c / 12) * SCAN_G) * 4 + (c & 3) < R) s += ACC[b * ldp + c];
      s = warp_sum(s);
      const float mean = ncol3 > 0 ? s / (float)ncol3 : 0.f;
      float m2 = 0.f;
      for (int c = lane; c < nh12; c += 32)
        if ((cta + (c / 12) * SCAN_G) * 4 + (c & 3) < R) { const float d = ACC[b * ldp + c] - mean; m2 = fmaf(d, d, m2); }
      m2 = warp_sum(m2);
      if (lane == 0) ll_store2(ll + L.s + (((size_t)par * MAXB + b) * SCAN_G + cta) * 2, mean, m2, tag);
    }
    if (pok) a.g_pre[(row0 + pb) * 3 * R + (size_t)ppart * R + pcol] = gpre;      // save after the hand-off
    for (int b = wid; b < B; b += SCAN_NW) {
      float mean, rstd;
      merge_row_stats(ll + L.s + ((size_t)par * MAXB + b) * SCAN_G * 2, tag, nctab, (float)(3 * R), a.eps, lane, sp, mean, rstd);
      if (lane == 0) {
        misc[16 + b] = mean;
        misc[32 + b] = rstd;
        if (cta == (t % SCAN_G)) { ln_stats[(row0 + b) * 2] = mean; ln_stats[(row0 + b) * 2 + 1] = rstd; }
      }
    }
    __syncthreads();
    if (sH.ok) {                               // LayerNorm, GRU gate (models.py:396-403) -> h_t for the owned columns
      const int b = sH.b, gi = sH.cj >> 2, j = sH.cj & 3;
      const float mu = misc[16 + b], rstd = misc[32 + b];
      float gl[3];
#pragma unroll
      for (int part = 0; part < 3; ++part)
        gl[part] = (ACC[b * ldp + gi * 12 + part * 4 + j] - mu) * rstd * LNP[(part * 2) * nh4 + sH.cj] + LNP[(part * 2 + 1) * nh4 + sH.cj];
      const float r = sigmoidf_(gl[0]);
      const float c = tanhf(r * gl[1]);
      const float u = sigmoidf_(gl[2] - 1.f);
      const float h = u * c + (1.f - u) * hin;
      ll_store(ll + L.h + ((size_t)par * MAXB + b) * R + sH.col, h, tag);         // hand-off first, saves after
      a.latent[(row0 + b) * a.ld_lat + a.lat_off + sH.col] = h;
#pragma unroll
      for (int part = 0; part < 3; ++part) a.g_ln[(row0 + b) * 3 * R + (size_t)part * R + sH.col] = gl[part];
      a.h_in[(row0 + b) * R + sH.col] = hin;
    }
    __syncthreads();
    if (sp.dead) break;    // a hand-off timed out somewhere: bail out, never hang
  }
}

__global__ void __launch_bounds__(SCAN_NT, 1)
gru_scan_bwd_kernel(const b200rl_gru_scan_args a, const b200rl_gru_scan_grads q) {
  extern __shared__ __align__(16) float sm[];
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int cta = blockIdx.x;
  const int T = a.T, B = a.B, R = a.R;
  const GeoG g = make_geo_g(R, cta, true);
  const GruLL L = make_gru_ll(R);
  int* error = (int*)((char*)a.workspace + 64);
  u64* ll = (u64*)((char*)a.workspace + WS_HEADER);
  const float* ln_stats = (const float*)(ll + L.total);
  float* WgT = sm + g.oW;       // [ngh*4][3*sR] columns of W_g[:, :R] (3 parts of sR)
  float* X = sm + g.oX;         // [MAXB][pw*sR]
  float* PART = sm + g.oPart;
  float* ACC = sm + g.oAcc;     // [MAXB][ldp]
  float* ST = sm + g.oSt;       // [(b, col)][2] staged (dxh, dxh*xh)
  float* DHC = sm + g.oDhc;     // [MAXB][nh4] dh carried to step t-1
  float* WSG = sm + g.oPar;     // [nh4] column sums of the weight slice
  float* LNP = sm + g.oLn;      // [3][nh4] LayerNorm weight of the owned columns
  float* misc = sm + g.oMisc;   // [0,16) first(t); [32,48) S1; [48,64) S2; [64,96) (mu, rstd) of step t
  float* S1 = misc + 32;
  float* S2 = misc + 48;
  float* LNS = misc + 64;
  const int ldp = g.ldp, wgst = 3 * g.sR, xw = g.pw * g.sR, nh4 = g.ngh * 4;
  Spin sp;
  sp.init(error);

  for (int e = tid; e < g.total; e += SCAN_NT) sm[e] = 0.f;
  __syncthreads();
  for (int gi = 0; gi < g.ngh; ++gi)
    for (int part = 0; part < 3; ++part)
      load_cols4(WgT + (size_t)gi * 4 * wgst, wgst, a.W_g + (size_t)part * R * a.ld_wg, a.ld_wg, (cta + gi * SCAN_G) * 4, R, R,
                 part * g.sR, tid);
  __syncthreads();
  for (int j = wid; j < nh4; j += SCAN_NW) {
    float s = 0.f;
    for (int k = lane; k < wgst; k += 32) s += WgT[(size_t)j * wgst + k];
    s = warp_sum(s);
    if (lane == 0) WSG[j] = s;
  }
  __syncthreads();
  const Slot sH = make_slot(tid, nh4, B, cta, R);            // dh element
  for (int e = tid; e < 3 * nh4; e += SCAN_NT) {
    const int part = e / nh4, cj = e - part * nh4, col = (cta + (cj >> 2) * SCAN_G) * 4 + (cj & 3);
    LNP[part * nh4 + cj] = col < R ? a.lng_g[part * R + col] : 0.f;
  }
  float dh0_acc = 0.f;                                        // (threads tid < nh4) accumulated over rows in fixed order

  for (int t = T - 1; t >= 0; --t) {
    const size_t row0 = (size_t)t * B;
    const int bt = T - 1 - t, par = bt & 1;
    const unsigned tag = (unsigned)bt + 1u;
    const bool last = (t == T - 1);
    // ---------------- step-start prefetch of chain-independent inputs (registers of the element's thread)
    if (tid < MAXB) misc[tid] = (tid < B) ? a.first[row0 + tid] : 0.f;
    for (int e = tid; e < B * 2; e += SCAN_NT) LNS[e] = ln_stats[row0 * 2 + e];
    float p_hin = 0.f, p_dlh = 0.f, p_qg = 0.f, p_gl[3] = {0.f, 0.f, 0.f}, p_gp[3] = {0.f, 0.f, 0.f};
    if (sH.ok) {
      p_hin = a.h_in[(row0 + sH.b) * R + sH.col];
      p_dlh = q.d_latent[(row0 + sH.b) * a.ld_lat + a.lat_off + sH.col];
      p_qg = q.q_g[(row0 + sH.b) * R + sH.col];
#pragma unroll
      for (int part = 0; part < 3; ++part) {
        p_gl[part] = a.g_ln[(row0 + sH.b) * 3 * R + (size_t)part * R + sH.col];
        p_gp[part] = a.g_pre[(row0 + sH.b) * 3 * R + (size_t)part * R + sH.col];
      }
    }
    __syncthreads();
    const float* fl = misc;

    // ============ dh = d_latent_h + carry ; GRU gate backward ; dxh of the GRU LayerNorm and its row sums
    float dhin_gate = 0.f, dgl[3] = {0.f, 0.f, 0.f};
    if (sH.ok) {
      const int b = sH.b;
      const float mug = LNS[b * 2], rstdg = LNS[b * 2 + 1];
      float dh = p_dlh;
      if (!last) dh += DHC[b * nh4 + sH.cj];
      const float r = sigmoidf_(p_gl[0]), cnd = tanhf(r * p_gl[1]), u = sigmoidf_(p_gl[2] - 1.f);
      const float du = dh * (cnd - p_hin);
      const float drc = dh * u * (1.f - cnd * cnd);
      dgl[0] = drc * p_gl[1] * r * (1.f - r);
      dgl[1] = drc * r;
      dgl[2] = du * u * (1.f - u);
      dhin_gate = dh * (1.f - u);
#pragma unroll
      for (int part = 0; part < 3; ++part) {
        const float xh = (p_gp[part] - mug) * rstdg;
        const float dxh = dgl[part] * LNP[part * nh4 + sH.cj];
        ll_store(ll + L.c + ((size_t)par * MAXB + b) * 3 * R + (size_t)part * R + sH.col, dxh, tag);
        ST[(b * (3 * nh4) + part * nh4 + sH.cj) * 2] = dxh;
        ST[(b * (3 * nh4) + part * nh4 + sH.cj) * 2 + 1] = dxh * xh;
      }
    } else if (tid < B * nh4) {
      const int b = tid / imax(nh4, 1), cj = tid - b * nh4;
#pragma unroll
      for (int part = 0; part < 3; ++part) {
        ST[(b * (3 * nh4) + part * nh4 + cj) * 2] = 0.f;
        ST[(b * (3 * nh4) + part * nh4 + cj) * 2 + 1] = 0.f;
      }
    }
    __syncthreads();
    send_row_sums(ST, 3 * nh4, B, ll + L.sc, par, cta, tag, tid);
    if (sH.ok)
#pragma unroll
      for (int part = 0; part < 3; ++part) q.d_g_ln[(row0 + sH.b) * 3 * R + (size_t)part * R + sH.col] = dgl[part];

    // ============ dh_in = d_g_pre W_g[:, :R] for the owned columns (K = 3R, in 3 / pw passes)
    float acc_h = 0.f;
    for (int p0 = 0; p0 < 3; p0 += g.pw) {
      for (int part = p0; part < p0 + g.pw; ++part) {
        const u64* src = ll + L.c + (size_t)par * MAXB * 3 * R + (size_t)part * R;
        if (part == g.pw - 1)        // the row sums ride with the last part of the first pass
          ll_recv<4>(X + (part - p0) * g.sR, xw, src, 3 * R, B, R, tag, tid, sp, ll + L.sc + (size_t)par * MAXB * SCAN_G * 2, 0,
                     1.f / (float)(3 * R), S1, S2);
        else
          ll_recv<4>(X + (part - p0) * g.sR, xw, src, 3 * R, B, R, tag, tid, sp);
      }
      __syncthreads();
      const int ks = product(X, xw, WgT + p0 * g.sR, wgst, g.ngh, g.pw * g.sR, B, PART, ldp, 0, tid);
      __syncthreads();
      if (sH.ok) acc_h += part_sum(PART, ldp, ks, sH.b, sH.cj);
      __syncthreads();
    }
    float dhin_f = 0.f;
    if (sH.ok) {
      const int b = sH.b;
      const float mug = LNS[b * 2], rstdg = LNS[b * 2 + 1];
      const float wsgh = WSG[sH.cj];
      const float p2 = rstdg * (p_qg - mug * wsgh);
      const float dhin = dhin_gate + rstdg * (acc_h - S1[b] * wsgh - S2[b] * p2);
      DHC[b * nh4 + sH.cj] = (1.f - fl[b]) * dhin;          // carried to step t-1 (agent.py:574 mask)
      dhin_f = fl[b] * dhin;                                // grad of tanh(initial_recurrent_state)
    }
    // d_h0: sum over the rows with is_first set, fixed row order (bit-reproducible): stage through ACC
    if (sH.ok) ACC[sH.b * ldp + sH.cj] = dhin_f;
    __syncthreads();
    if (tid < nh4)
      for (int b = 0; b < B; ++b)
        if (fl[b] != 0.f) dh0_acc += ACC[b * ldp + tid];
    __syncthreads();
    if (sp.dead) break;    // a hand-off timed out somewhere: bail out, never hang
  }
  if (tid < nh4) {
    const int col = (cta + (tid >> 2) * SCAN_G) * 4 + (tid & 3);
    if (col < R) q.d_h0[col] = dh0_acc;
  }
}

int gru_check(const b200rl_gru_scan_args& a, bool backward) {
  RL_CHECK_ARG(a.T >= 1 && a.B >= 1 && a.B <= MAXB, "GRU scan supports T >= 1 and batch <= 16 rows per rank");
  RL_CHECK_ARG(a.R >= 2 && a.R % 2 == 0, "GRU scan supports even recurrent_state_size");
  // one element of every per-step epilogue per thread (fixed assignments, `Slot`)
  RL_CHECK_ARG(MAXB * owned_groups(a.R, 0) * 12 <= SCAN_NT, "GRU scan supports recurrent_state_size <= 1024");
  RL_CHECK_ARG(a.ld_wg >= a.R && a.lat_off >= 0 && a.ld_lat >= a.lat_off + a.R, "GRU scan: leading dimensions too small");
  RL_CHECK_ARG(sizeof(float) * (size_t)make_geo_g(a.R, 0, backward).total <= 227 * 1024,
               "weight slice does not fit in shared memory for this model size");
  return B200RL_OK;
}

int gru_launch(void* fn, const b200rl_gru_scan_args& a, void** kargs, bool backward, cudaStream_t st) {
  if (int rc = gru_check(a, backward)) return rc;
  RL_CHECK_ARG(a.workspace && a.workspace_bytes >= (long long)gru_ws_bytes(a.T, a.B, a.R), "workspace too small");
  const size_t smem = sizeof(float) * (size_t)make_geo_g(a.R, 0, backward).total;
  RL_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  // header + LL region are reset; the forward's LayerNorm statistics behind them stay for the backward
  RL_CUDA(cudaMemsetAsync(a.workspace, 0, WS_HEADER + make_gru_ll(a.R).total * sizeof(u64), st));
  RL_CUDA(cudaLaunchCooperativeKernel(fn, dim3(SCAN_G), dim3(SCAN_NT), kargs, smem, st));
  return B200RL_OK;
}

}  // namespace

extern "C" long long b200rl_rssm_scan_workspace_bytes(int T, int B, int S, int D, int Dx, int R, int Dr) {
  return (long long)ws_bytes(T, B, S, D, Dx, R, Dr);
}

extern "C" int b200rl_rssm_scan_fwd(const b200rl_rssm_scan_args* args, cudaStream_t st) {
  RL_CHECK_ARG(args, "null args");
  const b200rl_rssm_scan_args& a = *args;
  if (int rc = scan_check(a, false)) return rc;
  if (int rc = workspace_check(a)) return rc;
  const size_t smem = scan_smem(a, false);
  const bool fix = fixed_dims(a);
  void* fn = fix ? (void*)rssm_scan_fwd_kernel<true> : (void*)rssm_scan_fwd_kernel<false>;
  RL_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  RL_CUDA(cudaMemsetAsync(a.workspace, 0, WS_HEADER + WS_PROF + ws_ll_bytes(a.S, a.D, a.Dx, a.R, a.Dr), st));
  void* kargs[] = {(void*)args};
  RL_CUDA(cudaLaunchCooperativeKernel(fn, dim3(SCAN_G), dim3(SCAN_NT), kargs, smem, st));
  return B200RL_OK;
}

extern "C" int b200rl_rssm_scan_check(const b200rl_rssm_scan_args* args, int backward) {
  RL_CHECK_ARG(args, "null args");
  return scan_check(*args, backward != 0);
}

extern "C" int b200rl_rssm_scan_bwd(const b200rl_rssm_scan_args* args, const b200rl_rssm_scan_grads* grads,
                                    cudaStream_t st) {
  RL_CHECK_ARG(args && grads, "null args");
  const b200rl_rssm_scan_args& a = *args;
  if (int rc = scan_check(a, true)) return rc;
  if (int rc = workspace_check(a)) return rc;
  RL_CHECK_ARG(grads->q_r && grads->q_g && grads->q_x, "q_r / q_g / q_x (pre-activation x weight products) are required");
  const size_t smem = scan_smem(a, true);
  const bool fix = fixed_dims(a);
  void* fn = fix ? (void*)rssm_scan_bwd_kernel<true> : (void*)rssm_scan_bwd_kernel<false>;
  RL_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  // header + LL region are reset; the forward's saves (class indices, LayerNorm statistics) behind them stay
  RL_CUDA(cudaMemsetAsync(a.workspace, 0, WS_HEADER + WS_PROF + ws_ll_bytes(a.S, a.D, a.Dx, a.R, a.Dr), st));
  void* kargs[] = {(void*)args, (void*)grads};
  RL_CUDA(cudaLaunchCooperativeKernel(fn, dim3(SCAN_G), dim3(SCAN_NT), kargs, smem, st));
  return B200RL_OK;
}

extern "C" int b200rl_rssm_scan_error(const void* workspace, cudaStream_t st) {
  int flag = 0;
  RL_CUDA(cudaMemcpyAsync(&flag, (const char*)workspace + 64, sizeof(int), cudaMemcpyDeviceToHost, st));
  RL_CUDA(cudaStreamSynchronize(st));
  return flag;
}

// cycle counters of CTA 0 / CTA 1 (32 slots each) accumulated by the last launch on this workspace
extern "C" int b200rl_rssm_scan_profile(const void* workspace, long long* out64, cudaStream_t st) {
  RL_CUDA(cudaMemcpyAsync(out64, (const char*)workspace + WS_HEADER, WS_PROF, cudaMemcpyDeviceToHost, st));
  RL_CUDA(cudaStreamSynchronize(st));
  return B200RL_OK;
}

extern "C" long long b200rl_gru_scan_workspace_bytes(int T, int B, int R) { return (long long)gru_ws_bytes(T, B, R); }

extern "C" int b200rl_gru_scan_check(const b200rl_gru_scan_args* args, int backward) {
  RL_CHECK_ARG(args, "null args");
  return gru_check(*args, backward != 0);
}

extern "C" int b200rl_gru_scan_fwd(const b200rl_gru_scan_args* args, cudaStream_t st) {
  RL_CHECK_ARG(args, "null args");
  void* kargs[] = {(void*)args};
  return gru_launch((void*)gru_scan_fwd_kernel, *args, kargs, false, st);
}

extern "C" int b200rl_gru_scan_bwd(const b200rl_gru_scan_args* args, const b200rl_gru_scan_grads* grads, cudaStream_t st) {
  RL_CHECK_ARG(args && grads, "null args");
  RL_CHECK_ARG(grads->q_g, "q_g (g_pre W_g[:, :R] over all rows) is required");
  void* kargs[] = {(void*)args, (void*)grads};
  return gru_launch((void*)gru_scan_bwd_kernel, *args, kargs, true, st);
}
