// Tensor-core GEMM for sm_90a: C[M,N] = A[M,K] * B[N,K]^T (+bias) (+C), fp32 in / fp32 out, computed as 3xTF32 on the
// Hopper tensor cores (wgmma.mma_async kind tf32, operands staged in shared memory by TMA with the 128-byte swizzle,
// stages handed over with mbarriers).
//
// Why 3xTF32: the parity bar for this path is 1e-4 against an fp32 CPU oracle through chains of ~100 dependent
// layers (SURVEY.md §0 F7).  Each fp32 operand x is split in-kernel into hi = x with the 13 low mantissa bits
// cleared (exactly what the TF32 datapath keeps) and lo = x - hi (exact in fp32); the product is accumulated
// as hi*hi + hi*lo + lo*hi in fp32 (the dropped lo*lo term is ~2^-22 relative).  Effective rate is 1/3 of the
// TF32 peak.
//
// Pipeline (per 128 x BN output tile, K step 32 = one 128-byte swizzle atom), 384 threads = three warpgroups:
//   warp 0    : TMA producer   -- cp.async.bulk.tensor loads of the raw fp32 A / B tiles, mbarrier complete_tx
//   warps 1-3 : B splitters    -- write hi = trunc_tf32(x) and lo = x - hi of each landed B tile to two K-major
//                                 128B-swizzled buffers (wgmma reads tf32 B only K-major from shared memory, so an
//                                 MN-major B tile is transposed on the way), fence.proxy.async, arrive
//   warpgroups 1, 2: consumers -- rows [0, 64) / [64, 128) of the tile: load their A fragment straight from the raw
//                                 swizzled tile into registers (any layout, split in registers), issue 4 k-steps x 3
//                                 wgmma per stage, and every CH stages add the finished chunk accumulator into fp32
//                                 registers with RN adds; finally +bias / +C and store
// Replaces: every large nn.Linear forward / input-gradient product of the Dreamer-V3 step
// (sheeprl/models/models.py MLP; agent.py heads, RSSM imagination, actor, critic).
//
// The same pipeline runs the stride-2 k4 p1 convolutions as IMPLICIT GEMMs (no im2col buffer): the A tile of a
// k-block (one filter tap x 32 input channels) is a 4-D TMA box over the channel-last image
// [N][H][W][C] -- box {32 ch, bw, bh, bn} with element strides {1,2,2,1} for the strided gather of Conv2d
// forward ("down"), {1,1,1,1} for the 2x2 sub-pixel taps of ConvTranspose2d forward ("up") -- and TMA's
// out-of-bounds zero fill supplies the padding.  Replaces CNNEncoder / CNNDecoder convolutions
// (sheeprl/algos/dreamer_v3/agent.py:78-91, :199-222) and their input-gradient passes.
#include <cuda.h>
#include <cudaTypedefs.h>

#include <mutex>
#include <unordered_map>

#include "common.cuh"

namespace {

constexpr int BM = 128, BK = 32;
constexpr int NTHREADS = 384;
constexpr int NSPLIT_THREADS = 96;                  // warps 1-3
constexpr int NCONS_WARPS = 8;                      // warpgroups 1 and 2
// register budget per thread after setmaxnreg: the producer warpgroup gives its registers to the consumers, which hold
// the chunk accumulator, the running fp32 sum and the A fragments of a stage (128 x BN tile: up to 64 + 64 + 32)
constexpr int PRODUCER_REGS = 56, CONSUMER_REGS = 224;
// Operand stages that fit the 227 KB of shared memory (less the 1024-byte alignment slack and the barriers).  A raw-B
// stage holds raw A, raw B, B hi and B lo; a pre-split stage holds raw A and the B planes TMA loads straight into the
// wgmma operand buffers (hi and lo; hi only in a single-pass product).
template <int PASSES, bool PRESPLIT> __host__ __device__ constexpr int b_buffers() { return PRESPLIT ? (PASSES == 3 ? 2 : 1) : 3; }
template <int BN, int PASSES, bool PRESPLIT> constexpr int stages_for() {
  return (227 * 1024 - 1024 - 256) / ((BM + b_buffers<PASSES, PRESPLIT>() * BN) * BK * (int)sizeof(float));
}

// ---------------------------------------------------------------- PTX wrappers
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t"
      "}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a protocol bug must abort the kernel (trap -> launch failure), never hang the device.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > 2000000000LL) asm volatile("trap;");
  }
}
// one lane of a converged warp (warp-uniform choice: the same lane every time)
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "elect.sync _|p, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t"
      "}"
      : "=r"(pred));
  return pred != 0;
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
          smem_u32(smem_dst)),
      "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2,
                                            int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];" ::"r"(
          smem_u32(smem_dst)),
      "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}

// D[64 x N] (+)= A[64 x 8] (registers, tf32) * B[N x 8]^T (shared memory descriptor, K-major); scale_d = 0 overwrites D
__device__ __forceinline__ void wgmma_tf32(float (&d)[32], const uint32_t (&a)[4], uint64_t desc_b, int scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\twgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc_b), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_tf32(float (&d)[64], const uint32_t (&a)[4], uint64_t desc_b, int scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %69, 0;\n\twgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, {%64, %65, %66, %67}, %68, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc_b), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// Pins registers an in-flight wgmma reads or writes: the compiler may neither move their uses across this point nor
// reuse them before it.
template <int N>
__device__ __forceinline__ void fence_regs(float (&r)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(r[i])::"memory");
}
template <int N, int W>
__device__ __forceinline__ void fence_regs(uint32_t (&r)[N][W]) {
#pragma unroll
  for (int i = 0; i < N; ++i)
#pragma unroll
    for (int j = 0; j < W; ++j) asm volatile("" : "+r"(r[i][j])::"memory");
}

// K-major operand tile [rows][32 fp32] with the 128B swizzle: 8-row groups are 1024 B apart (SBO); a k-step of 8 tf32
// advances the start address by 32 B inside the swizzle row.  Layout type 1 = SWIZZLE_128B (bits 62-63).
__device__ __forceinline__ uint64_t make_desc(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);       // start address, bits [0,14)
  d |= (uint64_t)1 << 16;                            // leading byte offset (unused: a k-step stays inside one atom)
  d |= (uint64_t)(1024 >> 4) << 32;                  // stride byte offset between 8-row groups
  d |= (uint64_t)1 << 62;                            // SWIZZLE_128B
  return d;
}

// Byte offsets of element (r, k) in the two raw tile layouts TMA writes with the 128-byte swizzle (16-byte chunk index
// XOR-ed with the 128-byte line index):
//   K-major  [rows][32 k]              : line = row
//   MN-major [rows / 32][32 k][32 rows]: 4 KB per 32-row block (one TMA box), line = k
__device__ __forceinline__ uint32_t kmajor_off(int r, int k) {
  return (uint32_t)(r * 128 + ((((k >> 2) ^ r) & 7) << 4) + (k & 3) * 4);
}
__device__ __forceinline__ uint32_t mnmajor_off(int r, int k) {
  return (uint32_t)((r >> 5) * 4096 + k * 128 + (((((r & 31) >> 2) ^ k) & 7) << 4) + (r & 3) * 4);
}

template <int BN, int PASSES, bool PRESPLIT>
struct Smem;
template <int BN, int PASSES>
struct Smem<BN, PASSES, false> {
  static constexpr int STAGES = stages_for<BN, PASSES, false>();
  // every operand buffer is a whole number of 1024-byte swizzle groups
  float a[STAGES][BM * BK];      // raw A tiles (the consumers split them in registers)
  float b[STAGES][BN * BK];      // raw B tiles
  float b_hi[STAGES][BN * BK];   // K-major hi / lo halves of B, the wgmma operands
  float b_lo[STAGES][BN * BK];
  uint64_t full[STAGES], split[STAGES], empty[STAGES];
};
// B given as its K-major TF32 hi / lo planes: TMA fills the wgmma operand buffers directly (no b_lo at PASSES == 1)
template <int BN, int PASSES>
struct Smem<BN, PASSES, true> {
  static constexpr int STAGES = stages_for<BN, PASSES, true>();
  float a[STAGES][BM * BK];
  float b_hi[STAGES][BN * BK];
  float b_lo[PASSES == 3 ? STAGES : 1][PASSES == 3 ? BN * BK : 256];
  uint64_t full[STAGES], empty[STAGES];
};

// Two-level accumulation.  The tensor core adds each k-step into its fp32 accumulator with truncation
// (round-toward-zero), a bias of ~2^-24 |acc| per add that grows linearly with K.  So the wgmma accumulator only ever
// holds a CHUNK of CH k-blocks (CH*4 k-steps); each finished chunk is added into the running fp32 sum with
// round-to-nearest FADDs.
constexpr int CH = 4;

constexpr int MODE_GEMM = 0, MODE_DOWN = 1, MODE_UP = 2;
// MODE_UP4: ConvTranspose2d forward with all four output parity classes in ONE 128-column tile (Cout == 32): the K loop walks
// the 9 shifted input windows (dy, dx in {-1, 0, 1}) instead of 4 parities x 4 taps, so every input tile is fetched from L2
// 9 times instead of 16, the B tile is the parity-major weight [4 * Cout][9 * Cin] with zeros where a (parity, shift) pair
// does not exist, and the epilogue scatters column group p to output pixel (2y + py, 2x + px).
constexpr int MODE_UP4 = 3;
constexpr int GROUP_M = 16;
struct TileGeo {
  int mode;
  int h, w, NB;            // small-image grid (conv modes)
  int bw, bh, bn;          // output tile = bn images x bh rows x bw cols of the small grid (bw*bh*bn == 128)
  int tiles_x, tiles_y;    // tiles per image
  int chunks;              // input channels / 32
  int Cout;                // output channels
  int ksplits;             // GEMM mode: number of K splits (gridDim.z); > 1 => partial tiles go through `part`
  float* part;             // split-K workspace: [ksplits][mpad][ldw] partial sums (fixed-order reduction, no atomics)
  int mpad, ldw;           // split-K workspace geometry (rows per split, row stride)
  int force_part;          // write the partial tile to the workspace even with a single split (fused reduce + LayerNorm tail)
  int passes;              // 3: x = hi + lo split, three TF32 products per k-step (fp32-accurate); 1: one TF32 product
                           // (torch's float32_matmul_precision "high", the reference's default on GPUs)
  int a_mn, b_mn;          // GEMM mode: operand stored [K][M] / [K][N] (MN-major) instead of [M][K] / [N][K]
  int mtiles;              // number of M tiles
  int ntiles;              // number of N tiles.  A CTA walks the flattened (m, n) tile list blockIdx.y, blockIdx.y +
                           // gridDim.y, ... (persistent); consecutive ids cover GROUP_M m-tiles x all n-tiles column by
                           // column, so the tiles in flight share few operand panels in L2
  int wg;                  // GEMM mode, conv weight gradient: A rows = (tap, big channel), K = small-grid pixels gathered
                           // from the channel-last big image by 4-D TMA boxes of 32 pixels (Cout = big channels)
};

// PRESPLIT: B arrives as K-major TF32 hi / lo planes (mapB / mapBlo, [N][K]) that TMA loads into the wgmma operand
// buffers; warps 1-3 idle and the consumers wait on `full` alone.  Otherwise mapB is raw B (K- or MN-major, per geo.b_mn)
// and the splitters write its halves (mapBlo unused).
template <int BN, int PASSES, bool PRESPLIT>
__global__ void __launch_bounds__(NTHREADS, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapB,
               const __grid_constant__ CUtensorMap mapBlo, float* __restrict__ C, const float* __restrict__ bias, int M,
               int N, int K, int ldc, int accumulate, const TileGeo geo) {
  using S = Smem<BN, PASSES, PRESPLIT>;
  constexpr int STAGES = S::STAGES;
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  // Align by offsetting the shared array itself (not by integer arithmetic on its generic address), so that the compiler
  // still knows every access through `s` is to shared memory: the consumers' A-fragment loads and the splitters' B
  // loads / stores become 32-bit-addressed LDS / STS instead of generic 64-bit LD / ST.
  S& s = *reinterpret_cast<S*>(smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u));
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int mtiles = geo.mtiles * geo.ntiles, tstride = gridDim.y;   // flattened tile count
  auto tile_mn = [&](int id, int& tm, int& tn) {
    if (geo.ntiles == 1) { tm = id; tn = 0; return; }
    const int per = GROUP_M * geo.ntiles, grp = id / per, first = grp * GROUP_M;
    const int gsz = min(GROUP_M, geo.mtiles - first), r = id - grp * per;
    tn = r / gsz;
    tm = first + (r - tn * gsz);
  };
  // split-K (GEMM mode): blockIdx.z owns k-blocks [kb_base, kb_base + nkb); its partial tile goes to the workspace and
  // a reduce kernel sums all partials in split order (bit-reproducible, no atomics on C)
  int kb_base = 0, nkb = (K + BK - 1) / BK;
  if (geo.mode == MODE_GEMM && geo.ksplits > 1) {
    const int per = (nkb + geo.ksplits - 1) / geo.ksplits;
    kb_base = (int)blockIdx.z * per;
    nkb = min(per, nkb - kb_base);
  }
  // conv modes: a tile's origin on the small-image grid; blockIdx.z = output parity class (up)
  const int py = (int)blockIdx.z >> 1, px = (int)blockIdx.z & 1;
  auto tile_origin = [&](int id, int& tx0, int& ty0, int& tn0) {
    tx0 = (id % geo.tiles_x) * geo.bw;
    ty0 = ((id / geo.tiles_x) % geo.tiles_y) * geo.bh;
    tn0 = (id / (geo.tiles_x * geo.tiles_y)) * geo.bn;
  };

  if (threadIdx.x == 0) {
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&s.full[i], 1);
      if constexpr (!PRESPLIT) mbar_init(&s.split[i], NSPLIT_THREADS / 32);
      mbar_init(&s.empty[i], NCONS_WARPS);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp < 4) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(PRODUCER_REGS));
    if (warp == 0) {
      // ===== TMA producer.  The whole warp walks the loop with warp-uniform control flow; the elected lane issues.
      const bool leader = elect_one();
      constexpr uint32_t STAGE_TX = (uint32_t)((BM + (PRESPLIT ? b_buffers<PASSES, true>() : 1) * BN) * BK * sizeof(float));
      // the stage's K-major B tile(s) at (k, n): raw B, or the hi (and lo) planes
      auto load_b_kmajor = [&](int st, int k, int n) {
        if constexpr (PRESPLIT) {
          tma_load_2d(s.b_hi[st], &mapB, &s.full[st], k, n);
          if (PASSES == 3) tma_load_2d(s.b_lo[st], &mapBlo, &s.full[st], k, n);
        } else {
          tma_load_2d(s.b[st], &mapB, &s.full[st], k, n);
        }
      };
      int it = 0;                                  // k-blocks issued so far, across tiles: stage / phase bookkeeping
      for (int tile = blockIdx.y; tile < mtiles; tile += tstride) {
        int tm, tn;
        tile_mn(tile, tm, tn);
        const int m0 = tm * BM, n0 = tn * BN;
        int tx0 = 0, ty0 = 0, tn0 = 0;
        if (geo.mode != MODE_GEMM) tile_origin(tm, tx0, ty0, tn0);
        for (int kb = 0; kb < nkb; ++kb, ++it) {
          const int st = it % STAGES;
          if (it >= STAGES) mbar_wait(&s.empty[st], ((it / STAGES) - 1) & 1);
          if (leader) {
            mbar_expect_tx(&s.full[st], STAGE_TX);
            if (geo.mode == MODE_GEMM) {
              const int k0 = (kb_base + kb) * BK;
              if (geo.wg) {
                // k0 = first of 32 raster-consecutive small pixels (one box bw x bh x bn); block j of the tile = rows of
                // one (tap, 32-channel chunk): the same strided gather as the forward conv, read MN-major
                const int x0 = k0 % geo.w, y0 = (k0 / geo.w) % geo.h, i0 = k0 / (geo.w * geo.h);
                for (int j = 0; j < BM / 32; ++j) {
                  const int r0 = m0 + 32 * j, tap = r0 / geo.Cout, ch = r0 - tap * geo.Cout;
                  tma_load_4d(s.a[st] + j * 1024, &mapA, &s.full[st], ch, 2 * x0 - 1 + (tap & 3), 2 * y0 - 1 + (tap >> 2), i0);
                }
              } else if (!geo.a_mn) tma_load_2d(s.a[st], &mapA, &s.full[st], k0, m0);
              else
                for (int j = 0; j < BM / 32; ++j) tma_load_2d(s.a[st] + j * 1024, &mapA, &s.full[st], m0 + 32 * j, k0);
              if (PRESPLIT || !geo.b_mn) load_b_kmajor(st, k0, n0);
              else if constexpr (!PRESPLIT)
                for (int j = 0; j < BN / 32; ++j) tma_load_2d(s.b[st] + j * 1024, &mapB, &s.full[st], n0 + 32 * j, k0);
            } else {
              const int tap = kb / geo.chunks, ch = (kb - tap * geo.chunks) * BK;
              int x, y;
              if (geo.mode == MODE_DOWN)     { x = 2 * tx0 - 1 + (tap & 3); y = 2 * ty0 - 1 + (tap >> 2); }
              else if (geo.mode == MODE_UP4) { x = tx0 + (tap % 3) - 1;     y = ty0 + (tap / 3) - 1; }      // tap = shift index
              else                           { x = tx0 + px - (tap & 1);    y = ty0 + py - (tap >> 1); }
              tma_load_4d(s.a[st], &mapA, &s.full[st], ch, x, y, tn0);
              load_b_kmajor(st, kb * BK, n0 + (geo.mode == MODE_UP ? (int)blockIdx.z * geo.Cout : 0));
            }
          }
          __syncwarp();
        }
      }
    } else if constexpr (!PRESPLIT) {
      // ===== B splitters: hi / lo halves of each landed B tile into the K-major swizzled operand buffers
      const int t = threadIdx.x - 32;
      int ntl = 0;
      for (int tile = blockIdx.y; tile < mtiles; tile += tstride) ++ntl;
      const int total_kb = ntl * nkb;
      const bool b_mn = geo.b_mn != 0;
      for (int kb = 0; kb < total_kb; ++kb) {
        const int st = kb % STAGES;
        mbar_wait(&s.full[st], (kb / STAGES) & 1);
        const char* raw = reinterpret_cast<const char*>(s.b[st]);
        char* bh = reinterpret_cast<char*>(s.b_hi[st]);
        char* bl = reinterpret_cast<char*>(s.b_lo[st]);
        // ~11 work items per thread: unrolled so that several items' loads are in flight before their stores
#pragma unroll 4
        for (int w = t; w < BN * BK / 4; w += NSPLIT_THREADS) {
          // work item = one 16-byte chunk (row n, k = 4kc .. 4kc+3) of the K-major target.  MN-major source: a warp
          // covers 32 consecutive n of one kc, so every gather load reads one 128-byte line (conflict-free)
          int n, kc;
          float4 v;
          if (!b_mn) {
            n = w >> 3; kc = w & 7;
            v = *reinterpret_cast<const float4*>(raw + kmajor_off(n, 4 * kc));
          } else {
            n = w % BN; kc = w / BN;
            v.x = *reinterpret_cast<const float*>(raw + mnmajor_off(n, 4 * kc));
            v.y = *reinterpret_cast<const float*>(raw + mnmajor_off(n, 4 * kc + 1));
            v.z = *reinterpret_cast<const float*>(raw + mnmajor_off(n, 4 * kc + 2));
            v.w = *reinterpret_cast<const float*>(raw + mnmajor_off(n, 4 * kc + 3));
          }
          float4 h;
          h.x = __uint_as_float(__float_as_uint(v.x) & 0xffffe000u);
          h.y = __uint_as_float(__float_as_uint(v.y) & 0xffffe000u);
          h.z = __uint_as_float(__float_as_uint(v.z) & 0xffffe000u);
          h.w = __uint_as_float(__float_as_uint(v.w) & 0xffffe000u);
          const uint32_t o = kmajor_off(n, 4 * kc);
          *reinterpret_cast<float4*>(bh + o) = h;
          if (PASSES == 3) *reinterpret_cast<float4*>(bl + o) = make_float4(v.x - h.x, v.y - h.y, v.z - h.z, v.w - h.w);
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy writes -> async proxy (wgmma)
        __syncwarp();
        if (lane == 0) mbar_arrive(&s.split[st]);
      }
    }
  } else {
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(CONSUMER_REGS));
    // ===== consumers.  Warpgroup cw owns tile rows [64 cw, 64 cw + 64); warp wq of it rows 16 wq + {g, g + 8}.
    constexpr int NACC = BN / 2;
    const int cw = (warp >> 2) - 1, wq = warp & 3, g = lane >> 2, tq = lane & 3;
    const int r0 = cw * 64 + wq * 16 + g;          // tile rows of this thread: r0 and r0 + 8
    const bool a_mn_tile = geo.a_mn != 0;          // GEMM with transposed A, or the conv weight gradient
    const uint64_t dbh_base = make_desc(smem_u32(s.b_hi[0])), dbl_base = make_desc(smem_u32(s.b_lo[0]));
    constexpr uint64_t STAGE_STEP = (uint64_t)(BN * BK * sizeof(float)) >> 4;
    int it = 0;
    for (int tile = blockIdx.y; tile < mtiles; tile += tstride) {
      int tm, tn;
      tile_mn(tile, tm, tn);
      const int m0 = tm * BM, n0 = tn * BN;
      int tx0 = 0, ty0 = 0, tn0 = 0;
      if (geo.mode != MODE_GEMM) tile_origin(tm, tx0, ty0, tn0);
      float acc[NACC], cacc[NACC];
#pragma unroll
      for (int j = 0; j < NACC; ++j) { acc[j] = 0.f; cacc[j] = 0.f; }
      for (int kb = 0; kb < nkb; ++kb, ++it) {
        const int st = it % STAGES;
        const uint32_t ph = (it / STAGES) & 1;
        mbar_wait(&s.full[st], ph);
        if constexpr (!PRESPLIT) mbar_wait(&s.split[st], ph);
        // A fragment of the 4 k-steps (tf32 m64k8 layout: a0 (g, t), a1 (g+8, t), a2 (g, t+4), a3 (g+8, t+4))
        const char* araw = reinterpret_cast<const char*>(s.a[st]);
        uint32_t ahi[4][4], alo[4][4];
#pragma unroll
        for (int ks = 0; ks < 4; ++ks)
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const int r = r0 + 8 * (e & 1), k = 8 * ks + tq + 4 * (e >> 1);
            const uint32_t x = *reinterpret_cast<const uint32_t*>(araw + (a_mn_tile ? mnmajor_off(r, k) : kmajor_off(r, k)));
            ahi[ks][e] = x & 0xffffe000u;
            if (PASSES == 3) alo[ks][e] = __float_as_uint(__uint_as_float(x) - __uint_as_float(x & 0xffffe000u));
          }
        const bool chunk_start = (kb % CH) == 0;
        const uint64_t dbh0 = dbh_base + (uint64_t)st * STAGE_STEP, dbl0 = dbl_base + (uint64_t)st * STAGE_STEP;
        fence_regs(cacc);
        fence_regs(ahi);
        if (PASSES == 3) fence_regs(alo);
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) {
          const uint64_t ob = (uint64_t)ks * 2;    // 32 B per k-step, in 16-byte units
          const int keep = !(chunk_start && ks == 0);
          if (PASSES == 3) {
            // small cross terms first, then the leading term
            wgmma_tf32(cacc, ahi[ks], dbl0 + ob, keep);
            wgmma_tf32(cacc, alo[ks], dbh0 + ob, 1);
            wgmma_tf32(cacc, ahi[ks], dbh0 + ob, 1);
          } else {
            wgmma_tf32(cacc, ahi[ks], dbh0 + ob, keep);
          }
        }
        wgmma_commit();
        wgmma_wait_all();
        fence_regs(cacc);
        fence_regs(ahi);
        if (PASSES == 3) fence_regs(alo);
        __syncwarp();
        if (lane == 0) mbar_arrive(&s.empty[st]);   // this warp is done with the stage's A and B
        if ((kb % CH) == CH - 1 || kb == nkb - 1) {
#pragma unroll
          for (int j = 0; j < NACC; ++j) acc[j] += cacc[j];
        }
      }
      // ---- epilogue.  acc[4j + 2h + e] = tile (row r0 + 8h, column 8j + 2tq + e)
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const int r = r0 + 8 * hh;
        const int row = m0 + r;
        bool row_ok = row < M;
        size_t row_off = (size_t)row * ldc;
        int wi = 0, hi = 0, ni = 0;
        if (geo.mode != MODE_GEMM) {
          wi = r % geo.bw; hi = (r / geo.bw) % geo.bh; ni = r / (geo.bw * geo.bh);
          const int n = tn0 + ni, y = ty0 + hi, x = tx0 + wi;
          row_ok = n < geo.NB;
          if (geo.mode == MODE_DOWN) row_off = (((size_t)n * geo.h + y) * geo.w + x) * (size_t)ldc;
          else row_off = (((size_t)n * (2 * geo.h) + (2 * y + py)) * (2 * geo.w) + (2 * x + px)) * (size_t)ldc;
        }
        if (geo.mode == MODE_UP4) {
          // columns [32p, 32p + 32) of the tile = the Cout = 32 channels of output pixel (2y + (p >> 1), 2x + (p & 1))
          if (!row_ok) continue;
          const size_t n = (size_t)(tn0 + ni);
          const int y = ty0 + hi, x = tx0 + wi;
#pragma unroll
          for (int j = 0; j < NACC / 4; ++j) {
            const int c = 8 * j + 2 * tq, p = c >> 5, ch = c & 31;
            float* dst = C + ((n * (2 * geo.h) + (2 * y + (p >> 1))) * (2 * geo.w) + (2 * x + (p & 1))) * (size_t)32 + ch;
            float2 o = make_float2(acc[4 * j + 2 * hh], acc[4 * j + 2 * hh + 1]);
            if (bias) { o.x += bias[ch]; o.y += bias[ch + 1]; }
            *reinterpret_cast<float2*>(dst) = o;
          }
          continue;
        }
        if (geo.mode == MODE_GEMM && (geo.ksplits > 1 || geo.force_part)) {
          // ---- deterministic split-K: this split's partial tile goes to the workspace; splitk_reduce_kernel (launched
          // right behind this kernel) sums the partials of every output element in split order
          float* prow = geo.part + ((size_t)blockIdx.z * geo.mpad + (size_t)row) * geo.ldw + n0;
#pragma unroll
          for (int j = 0; j < NACC / 4; ++j)
            *reinterpret_cast<float2*>(prow + 8 * j + 2 * tq) = make_float2(acc[4 * j + 2 * hh], acc[4 * j + 2 * hh + 1]);
          continue;
        }
        if (!row_ok) continue;
        float* crow = C + row_off;
#pragma unroll
        for (int j = 0; j < NACC / 4; ++j) {
          const int cb = n0 + 8 * j + 2 * tq;
          float v0 = acc[4 * j + 2 * hh], v1 = acc[4 * j + 2 * hh + 1];
          if (cb + 1 < N && ((reinterpret_cast<uintptr_t>(crow + cb) & 7) == 0)) {
            if (bias) { v0 += bias[cb]; v1 += bias[cb + 1]; }
            if (accumulate) { const float2 q = *reinterpret_cast<const float2*>(crow + cb); v0 += q.x; v1 += q.y; }
            *reinterpret_cast<float2*>(crow + cb) = make_float2(v0, v1);
          } else {
            if (cb < N) crow[cb] = v0 + (bias ? bias[cb] : 0.f) + (accumulate ? crow[cb] : 0.f);
            if (cb + 1 < N) crow[cb + 1] = v1 + (bias ? bias[cb + 1] : 0.f) + (accumulate ? crow[cb + 1] : 0.f);
          }
        }
      }
    }   // tile loop
  }
}

// ---------------------------------------------------------------- host side: tensor-map cache
struct MapKey {
  const void* ptr; int rows, cols, ld, box_rows;
  bool operator==(const MapKey& o) const { return ptr == o.ptr && rows == o.rows && cols == o.cols && ld == o.ld && box_rows == o.box_rows; }
};
struct MapHash {
  size_t operator()(const MapKey& k) const {
    size_t h = std::hash<const void*>()(k.ptr);
    h ^= std::hash<long long>()(((long long)k.rows << 32) ^ k.cols) + 0x9e3779b97f4a7c15ull + (h << 6) + (h >> 2);
    h ^= std::hash<long long>()(((long long)k.ld << 8) ^ k.box_rows) + 0x9e3779b97f4a7c15ull + (h << 6) + (h >> 2);
    return h;
  }
};
std::unordered_map<MapKey, CUtensorMap, MapHash> g_maps;
std::mutex g_maps_mu;

// cuTensorMapEncodeTiled is a driver-API symbol: resolve it through the runtime at first use so that the library
// has no link-time dependency on libcuda.so (it must load on a GPU-less build host).
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn encode_tiled() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

// [rows][cols] fp32, row stride ld; box = [box_rows][32], 128-byte swizzle, zero fill out of bounds
int get_map(const float* ptr, int rows, int cols, int ld, int box_rows, CUtensorMap* out) {
  MapKey key{ptr, rows, cols, ld, box_rows};
  std::lock_guard<std::mutex> lk(g_maps_mu);
  auto it = g_maps.find(key);
  if (it != g_maps.end()) { *out = it->second; return B200RL_OK; }
  CUtensorMap m;
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)ld * sizeof(float)};
  cuuint32_t box[2] = {(cuuint32_t)BK, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  EncodeTiledFn enc = encode_tiled();
  if (!enc) { b200rl_set_error("cuTensorMapEncodeTiled is not available from this driver"); return B200RL_ERR_CUDA; }
  CUresult r = enc(&m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(ptr), dims, strides, box,
                                      estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                      CU_TENSOR_MAP_SWIZZLE_128B,
                                      CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    b200rl_set_error("cuTensorMapEncodeTiled failed (%d) for [%d x %d] ld %d", (int)r, rows, cols, ld);
    return B200RL_ERR_CUDA;
  }
  if (g_maps.size() > 4096) g_maps.clear();
  g_maps.emplace(key, m);
  *out = m;
  return B200RL_OK;
}

struct Map4Key {
  const void* ptr; int C, W, H, N, bw, bh, bn, es;
  bool operator==(const Map4Key& o) const {
    return ptr == o.ptr && C == o.C && W == o.W && H == o.H && N == o.N && bw == o.bw && bh == o.bh && bn == o.bn && es == o.es;
  }
};
struct Map4Hash {
  size_t operator()(const Map4Key& k) const {
    size_t h = std::hash<const void*>()(k.ptr);
    const long long v[4] = {((long long)k.C << 32) ^ k.W, ((long long)k.H << 32) ^ k.N, ((long long)k.bw << 32) ^ k.bh,
                            ((long long)k.bn << 32) ^ k.es};
    for (long long x : v) h ^= std::hash<long long>()(x) + 0x9e3779b97f4a7c15ull + (h << 6) + (h >> 2);
    return h;
  }
};
std::unordered_map<Map4Key, CUtensorMap, Map4Hash> g_maps4;

// channel-last image [N][H][W][C]; box = {32 ch, bw px, bh px, bn images} sampled with element stride es in W and H
int get_map4(const float* ptr, int C, int W, int H, int N, int bw, int bh, int bn, int es, CUtensorMap* out) {
  Map4Key key{ptr, C, W, H, N, bw, bh, bn, es};
  std::lock_guard<std::mutex> lk(g_maps_mu);
  auto it = g_maps4.find(key);
  if (it != g_maps4.end()) { *out = it->second; return B200RL_OK; }
  CUtensorMap m;
  cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
  cuuint64_t strides[3] = {(cuuint64_t)C * 4, (cuuint64_t)C * W * 4, (cuuint64_t)C * W * H * 4};
  // with an element stride e the box spans (count-1)*e+1 source elements and loads `count` of them
  cuuint32_t box[4] = {(cuuint32_t)BK, (cuuint32_t)((bw - 1) * es + 1), (cuuint32_t)((bh - 1) * es + 1), (cuuint32_t)bn};
  cuuint32_t estr[4] = {1, (cuuint32_t)es, (cuuint32_t)es, 1};
  EncodeTiledFn enc = encode_tiled();
  if (!enc) { b200rl_set_error("cuTensorMapEncodeTiled is not available from this driver"); return B200RL_ERR_CUDA; }
  CUresult r = enc(&m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, const_cast<float*>(ptr), dims, strides, box,
                                      estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                      CU_TENSOR_MAP_SWIZZLE_128B,
                                      CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    b200rl_set_error("cuTensorMapEncodeTiled(4D) failed (%d) for image [%d,%d,%d,%d]", (int)r, N, H, W, C);
    return B200RL_ERR_CUDA;
  }
  if (g_maps4.size() > 1024) g_maps4.clear();
  g_maps4.emplace(key, m);
  *out = m;
  return B200RL_OK;
}

// tile shape on the small grid: as wide as possible, 128 pixels in total
bool conv_tile(int h, int w, int NB, int* bw, int* bh, int* bn) {
  if (w <= 0 || h <= 0 || (w & (w - 1)) || (h & (h - 1))) return false;
  *bw = w < 128 ? w : 128;
  int rest = 128 / *bw;
  *bh = h < rest ? h : rest;
  *bn = rest / *bh;
  return (w % *bw == 0) && (h % *bh == 0) && (*bw * *bh * *bn == 128) && (NB % *bn == 0);
}

// Persistent scheduling: with one CTA per SM (the operand stages fill shared memory) a launch of many short tiles pays
// barrier setup and pipeline fill per tile.  When there are more than two waves of tiles, launch about one CTA per SM
// and let each walk its M tiles (the producer already loads the next tile's stages during the epilogue of a tile).
static unsigned persistent_grid_y(int tiles, unsigned gz) {
  const long long total = (long long)tiles * gz;
  if (total <= 2LL * kNumSMs) return (unsigned)tiles;
  unsigned gy = kNumSMs / gz;
  if (gy < 1) gy = 1;
  return gy < (unsigned)tiles ? gy : (unsigned)tiles;
}

// The TF32 split the B splitters apply in-kernel: hi = x with the 13 low mantissa bits cleared, lo = x - hi (exact)
__device__ __forceinline__ float tf32_hi(float x) { return __uint_as_float(__float_as_uint(x) & 0xffffe000u); }
// P[i] = v, or with a lo plane L: P[i] = hi(v), L[i] = v - hi(v)
__device__ __forceinline__ void store_split(float* P, float* L, long long i, float v) {
  if (L) { const float h = tf32_hi(v); P[i] = h; L[i] = v - h; }
  else P[i] = v;
}

__global__ void tf32_split_kernel(const float* __restrict__ X, float* __restrict__ H, float* __restrict__ L, long long n) {
  const long long i = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * 4;
  if (i + 4 <= n && !((reinterpret_cast<uintptr_t>(X) | reinterpret_cast<uintptr_t>(H) | reinterpret_cast<uintptr_t>(L)) & 15)) {
    const float4 v = *reinterpret_cast<const float4*>(X + i);
    const float4 h = make_float4(tf32_hi(v.x), tf32_hi(v.y), tf32_hi(v.z), tf32_hi(v.w));
    *reinterpret_cast<float4*>(H + i) = h;
    *reinterpret_cast<float4*>(L + i) = make_float4(v.x - h.x, v.y - h.y, v.z - h.z, v.w - h.w);
  } else {
    for (long long j = i; j < i + 4 && j < n; ++j) store_split(H, L, j, X[j]);
  }
}

// H[c][r], L[c][r] = split(W[r][c]) for r < rows; columns [rows, ldt) of H and L are zero.  32 x 32 tiles through shared
// memory, both sides coalesced.
__global__ void tf32_split_t_kernel(const float* __restrict__ W, float* __restrict__ H, float* __restrict__ L, int rows,
                                    int cols, long long ldw, long long ldt) {
  __shared__ float t[32][33];
  const int c0 = blockIdx.x * 32, r0 = blockIdx.y * 32;
  for (int j = threadIdx.y; j < 32; j += blockDim.y) {
    const int r = r0 + j, c = c0 + threadIdx.x;
    t[j][threadIdx.x] = (r < rows && c < cols) ? W[(long long)r * ldw + c] : 0.f;
  }
  __syncthreads();
  for (int j = threadIdx.y; j < 32; j += blockDim.y) {
    const int c = c0 + j, r = r0 + threadIdx.x;
    if (c < cols && r < ldt) store_split(H, L, (long long)c * ldt + r, t[threadIdx.x][j]);
  }
}

__global__ void conv_pack_down_kernel(const float* __restrict__ W, float* __restrict__ P, float* __restrict__ L, int Cs,
                                      int Cb) {
  // P[cs][tap][cb] = W[cs][cb][tap]
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)Cs * Cb * 16) return;
  const int cb = (int)(idx % Cb);
  const int tap = (int)((idx / Cb) % 16);
  const int cs = (int)(idx / ((long long)Cb * 16));
  store_split(P, L, idx, W[((long long)cs * Cb + cb) * 16 + tap]);
}
__global__ void conv_pack_up_kernel(const float* __restrict__ W, float* __restrict__ P, float* __restrict__ L, int Cs,
                                    int Cb) {
  // P[parity][cb][t][cs] = W[cs][cb][ky][kx], ky = (1-py)+2j, kx = (1-px)+2i, t = 2j+i
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)Cs * Cb * 16) return;
  const int cs = (int)(idx % Cs);
  const int t = (int)((idx / Cs) % 4);
  const int cb = (int)((idx / ((long long)Cs * 4)) % Cb);
  const int par = (int)(idx / ((long long)Cs * 4 * Cb));
  const int py = par >> 1, px = par & 1;
  const int ky = (1 - py) + 2 * (t >> 1), kx = (1 - px) + 2 * (t & 1);
  store_split(P, L, idx, W[((long long)cs * Cb + cb) * 16 + ky * 4 + kx]);
}

__global__ void conv_pack_up4_kernel(const float* __restrict__ W, float* __restrict__ P, float* __restrict__ L, int Cs,
                                     int Cb) {
  // P[parity * Cb + cb][shift * Cs + cs] = W[cs][cb][ky][kx] when output parity (py, px) reads shift (dy, dx) (j = py - dy,
  // i = px - dx in {0, 1}; ky = (1 - py) + 2j, kx = (1 - px) + 2i), else 0.  shift = (dy + 1) * 3 + (dx + 1).
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= 36LL * Cs * Cb) return;
  const int cs = (int)(idx % Cs);
  const int shift = (int)((idx / Cs) % 9);
  const int cb = (int)((idx / (9LL * Cs)) % Cb);
  const int par = (int)(idx / (9LL * Cs * Cb));
  const int py = par >> 1, px = par & 1, dy = shift / 3 - 1, dx = shift % 3 - 1;
  const int j = py - dy, i = px - dx;
  float v = 0.f;
  if (j >= 0 && j <= 1 && i >= 0 && i <= 1) v = W[((long long)cs * Cb + cb) * 16 + ((1 - py) + 2 * j) * 4 + (1 - px) + 2 * i];
  store_split(P, L, idx, v);
}
static bool conv_up_merged(int Cb) { return Cb == 32; }

// Matmul precision of every tensor-core product of the library (process-wide, like torch.set_float32_matmul_precision):
// 3 = fp32-accurate 3xTF32 (default; what the 1e-4 parity tests run), 1 = single TF32 pass.
int g_passes = 3;

// Split-K workspace (partial tiles), one per device, grown on demand OUTSIDE stream capture (launches on one stream
// serialise, so consecutive products share it; a capture replays the size it was captured with).
struct SplitWs {
  float* part = nullptr;
  size_t floats = 0;
};
SplitWs g_split[16];
std::mutex g_split_mu;

int split_workspace(size_t need_floats, cudaStream_t st, float** part) {
  int dev = 0;
  RL_CUDA(cudaGetDevice(&dev));
  RL_CHECK_ARG(dev < 16, "split-K workspace: device index out of range");
  std::lock_guard<std::mutex> lk(g_split_mu);
  SplitWs& w = g_split[dev];
  if (need_floats > w.floats) {
    cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
    RL_CUDA(cudaStreamIsCapturing(st, &cs));
    if (cs != cudaStreamCaptureStatusNone) {
      b200rl_set_error("split-K workspace must grow during stream capture: run the step once eagerly first");
      return B200RL_ERR_CUDA;
    }
    RL_CUDA(cudaDeviceSynchronize());
    if (w.part) RL_CUDA(cudaFree(w.part));
    const size_t n = need_floats + need_floats / 2 > (size_t)16 << 20 ? need_floats + need_floats / 2 : (size_t)16 << 20;
    RL_CUDA(cudaMalloc(&w.part, n * sizeof(float)));
    w.floats = n;
  }
  *part = w.part;
  return B200RL_OK;
}

// C[m][n] (+)= bias[n] + sum_z part[z][m][n], z ascending: the fixed-order tail of a split-K product
__global__ void __launch_bounds__(256)
splitk_reduce_kernel(const float* __restrict__ part, float* __restrict__ C, const float* __restrict__ bias, int M, int N,
                     int ldc, int ks, int mpad, int ldw, int accumulate) {
  const int n4 = (N + 3) >> 2;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)M * n4) return;
  const int m = (int)(idx / n4), n = (int)(idx - (long long)m * n4) * 4;
  const float* p = part + (size_t)m * ldw + n;
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 4                                    // the splits' loads in flight together; the adds keep split order
  for (int z = 0; z < ks; ++z) {
    const float4 v = __ldcg(reinterpret_cast<const float4*>(p + (size_t)z * mpad * ldw));
    acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
  }
  float* c = C + (size_t)m * ldc + n;
  const float o[4] = {acc.x, acc.y, acc.z, acc.w};
  if (n + 4 <= N && ((reinterpret_cast<uintptr_t>(c) & 15) == 0)) {
    float4 r = acc;
    if (bias) { r.x += bias[n]; r.y += bias[n + 1]; r.z += bias[n + 2]; r.w += bias[n + 3]; }
    if (accumulate) { const float4 q = *reinterpret_cast<const float4*>(c); r.x += q.x; r.y += q.y; r.z += q.z; r.w += q.w; }
    *reinterpret_cast<float4*>(c) = r;
  } else {
    for (int j = 0; j < 4 && n + j < N; ++j) {
      float r = o[j];
      if (bias) r += bias[n + j];
      if (accumulate) r += c[j];
      c[j] = r;
    }
  }
}

// one launch site for the eight instantiations (tile width x TF32 passes x B source)
#define LAUNCH_GEMM_TC(BN_, PASSES_, PRE_, grid_, st_, ...)                                                          \
  do {                                                                                                               \
    static_assert(sizeof(Smem<BN_, PASSES_, PRE_>) + 1024 <= 227 * 1024, "operand stages exceed shared memory");     \
    const size_t smem__ = sizeof(Smem<BN_, PASSES_, PRE_>) + 1024;                                                   \
    RL_CUDA(cudaFuncSetAttribute(gemm_tc_kernel<BN_, PASSES_, PRE_>, cudaFuncAttributeMaxDynamicSharedMemorySize,     \
                                 (int)smem__));                                                                      \
    gemm_tc_kernel<BN_, PASSES_, PRE_><<<grid_, NTHREADS, smem__, st_>>>(__VA_ARGS__);                                \
  } while (0)
#define DISPATCH_GEMM_TC_PRE(BN_val, passes_val, PRE_, grid_, st_, ...)                        \
  do {                                                                                          \
    if ((BN_val) == 64) {                                                                       \
      if ((passes_val) == 3) LAUNCH_GEMM_TC(64, 3, PRE_, grid_, st_, __VA_ARGS__);              \
      else LAUNCH_GEMM_TC(64, 1, PRE_, grid_, st_, __VA_ARGS__);                                \
    } else {                                                                                    \
      if ((passes_val) == 3) LAUNCH_GEMM_TC(128, 3, PRE_, grid_, st_, __VA_ARGS__);             \
      else LAUNCH_GEMM_TC(128, 1, PRE_, grid_, st_, __VA_ARGS__);                               \
    }                                                                                           \
  } while (0)
// mb2: the lo plane's map when `presplit`, else ignored
#define DISPATCH_GEMM_TC(BN_val, passes_val, presplit_, grid_, st_, ma_, mb_, mb2_, ...)                    \
  do {                                                                                                       \
    if (presplit_) DISPATCH_GEMM_TC_PRE(BN_val, passes_val, true, grid_, st_, ma_, mb_, mb2_, __VA_ARGS__);  \
    else DISPATCH_GEMM_TC_PRE(BN_val, passes_val, false, grid_, st_, ma_, mb_, mb_, __VA_ARGS__);           \
  } while (0)

// Wp: the packed weight; Wlo: its TF32 lo plane when Wp holds the hi plane (pre-split B), else null
int launch_conv(int mode, const float* img, const float* Wp, const float* Wlo, float* out, const float* bias, int NB, int h,
                int w, int Cin, int Cout, cudaStream_t st) {
  TileGeo g = {};
  g.mode = mode; g.h = h; g.w = w; g.NB = NB; g.chunks = Cin / BK; g.Cout = Cout; g.ksplits = 1;
  g.passes = g_passes;
  RL_CHECK_ARG(conv_tile(h, w, NB, &g.bw, &g.bh, &g.bn), "image grid not tileable by 128 pixels");
  g.tiles_x = w / g.bw; g.tiles_y = h / g.bh;
  if (mode == MODE_UP && conv_up_merged(Cout)) mode = g.mode = MODE_UP4;
  const int taps = mode == MODE_DOWN ? 16 : (mode == MODE_UP4 ? 9 : 4);
  const int K = taps * Cin;
  CUtensorMap ma, mb;
  if (mode == MODE_DOWN) { if (int rc = get_map4(img, Cin, 2 * w, 2 * h, NB, g.bw, g.bh, g.bn, 2, &ma)) return rc; }
  else                   { if (int rc = get_map4(img, Cin, w, h, NB, g.bw, g.bh, g.bn, 1, &ma)) return rc; }
  const int BN = (mode == MODE_UP4) ? 128 : ((Cout <= 64) ? 64 : 128);
  const int brows = (mode == MODE_UP || mode == MODE_UP4) ? 4 * Cout : Cout;
  if (int rc = get_map(Wp, brows, K, K, BN, &mb)) return rc;
  CUtensorMap mb2 = mb;
  if (Wlo && g.passes == 3) { if (int rc = get_map(Wlo, brows, K, K, BN, &mb2)) return rc; }
  const int mtiles = g.tiles_x * g.tiles_y * (NB / g.bn);
  g.mtiles = mtiles;
  g.ntiles = (mode == MODE_UP4) ? 1 : (Cout + BN - 1) / BN;
  dim3 grid(1, 1, mode == MODE_UP ? 4 : 1);
  grid.y = persistent_grid_y(mtiles * g.ntiles, grid.z);
  const int M = NB * h * w;  // unused by conv addressing; row validity comes from geo
  DISPATCH_GEMM_TC(BN, g.passes, Wlo != nullptr, grid, st, ma, mb, mb2, out, bias, M, Cout, K, Cout, 0, g);
  RL_CHECK_LAUNCH();
  return B200RL_OK;
}

}  // namespace

extern "C" int b200rl_set_matmul_precision(int tf32_passes) {
  RL_CHECK_ARG(tf32_passes == 1 || tf32_passes == 3, "tf32_passes must be 3 (fp32-accurate 3xTF32) or 1 (single TF32 pass)");
  g_passes = tf32_passes;
  return B200RL_OK;
}
extern "C" int b200rl_get_matmul_precision(void) { return g_passes; }

// ---- convolution entry points (tensor-core implicit GEMM).  Wpacked: caller workspace of b200rl_conv_pack_floats() floats
// (16*Cs*Cb; 36*Cs*Cb for the merged-parity ConvTranspose2d layout used when Cb == 32).
extern "C" long long b200rl_conv_pack_floats(int mode_up, int Cs, int Cb) {
  return (mode_up && conv_up_merged(Cb) ? 36LL : 16LL) * Cs * Cb;
}
extern "C" int b200rl_conv_tc_supported(int mode_up, int NB, int h, int w, int Cs, int Cb) {
  int bw, bh, bn;
  if (!conv_tile(h, w, NB, &bw, &bh, &bn)) return 0;
  const int Cin = mode_up ? Cs : Cb, Cout = mode_up ? Cb : Cs;
  if (Cin % BK != 0 || Cout < 16 || Cout % 4 != 0) return 0;
  return 1;
}
namespace {
int conv_pack_impl(const float* W, float* P, float* L, int mode_up, int Cs, int Cb, cudaStream_t st) {
  const long long n = (long long)Cs * Cb * 16;
  if (mode_up && conv_up_merged(Cb)) conv_pack_up4_kernel<<<ceil_div(36LL * Cs * Cb, 256), 256, 0, st>>>(W, P, L, Cs, Cb);
  else if (mode_up) conv_pack_up_kernel<<<ceil_div(n, 256), 256, 0, st>>>(W, P, L, Cs, Cb);
  else conv_pack_down_kernel<<<ceil_div(n, 256), 256, 0, st>>>(W, P, L, Cs, Cb);
  RL_CHECK_LAUNCH();
  return B200RL_OK;
}
}  // namespace
extern "C" int b200rl_conv_pack(const float* W, float* Wpacked, int mode_up, int Cs, int Cb, cudaStream_t st) {
  RL_CHECK_ARG(W && Wpacked, "null pointer");
  return conv_pack_impl(W, Wpacked, nullptr, mode_up, Cs, Cb, st);
}
extern "C" int b200rl_conv_pack_split(const float* W, float* Whi, float* Wlo, int mode_up, int Cs, int Cb, cudaStream_t st) {
  RL_CHECK_ARG(W && Whi && Wlo, "null pointer");
  return conv_pack_impl(W, Whi, Wlo, mode_up, Cs, Cb, st);
}
extern "C" int b200rl_conv_down_tc(const float* big, const float* Wpacked, float* small_, int NB, int h, int w, int Cs,
                                   int Cb, cudaStream_t st) {
  RL_CHECK_ARG(big && Wpacked && small_, "null pointer");
  RL_CHECK_ARG(b200rl_conv_tc_supported(0, NB, h, w, Cs, Cb), "shape not eligible for the tensor-core conv path");
  return launch_conv(MODE_DOWN, big, Wpacked, nullptr, small_, nullptr, NB, h, w, Cb, Cs, st);
}
extern "C" int b200rl_conv_up_tc(const float* small_, const float* Wpacked, float* big, const float* bias, int NB, int h,
                                 int w, int Cs, int Cb, cudaStream_t st) {
  RL_CHECK_ARG(big && Wpacked && small_, "null pointer");
  RL_CHECK_ARG(b200rl_conv_tc_supported(1, NB, h, w, Cs, Cb), "shape not eligible for the tensor-core conv path");
  return launch_conv(MODE_UP, small_, Wpacked, nullptr, big, bias, NB, h, w, Cs, Cb, st);
}
extern "C" int b200rl_conv_down_tc_presplit(const float* big, const float* Whi, const float* Wlo, float* small_, int NB,
                                            int h, int w, int Cs, int Cb, cudaStream_t st) {
  RL_CHECK_ARG(big && Whi && Wlo && small_, "null pointer");
  RL_CHECK_ARG(b200rl_conv_tc_supported(0, NB, h, w, Cs, Cb), "shape not eligible for the tensor-core conv path");
  return launch_conv(MODE_DOWN, big, Whi, Wlo, small_, nullptr, NB, h, w, Cb, Cs, st);
}
extern "C" int b200rl_conv_up_tc_presplit(const float* small_, const float* Whi, const float* Wlo, float* big,
                                          const float* bias, int NB, int h, int w, int Cs, int Cb, cudaStream_t st) {
  RL_CHECK_ARG(big && Whi && Wlo && small_, "null pointer");
  RL_CHECK_ARG(b200rl_conv_tc_supported(1, NB, h, w, Cs, Cb), "shape not eligible for the tensor-core conv path");
  return launch_conv(MODE_UP, small_, Whi, Wlo, big, bias, NB, h, w, Cs, Cb, st);
}

extern "C" int b200rl_tf32_split(const float* X, float* Xhi, float* Xlo, long long n, cudaStream_t st) {
  RL_CHECK_ARG(X && Xhi && Xlo, "null pointer");
  RL_CHECK_ARG(n >= 0, "negative length");
  if (n == 0) return B200RL_OK;
  tf32_split_kernel<<<ceil_div((n + 3) / 4, 256), 256, 0, st>>>(X, Xhi, Xlo, n);
  RL_CHECK_LAUNCH();
  return B200RL_OK;
}
extern "C" int b200rl_tf32_split_t(const float* W, float* Thi, float* Tlo, int rows, int cols, long long ldw, long long ldt,
                                   cudaStream_t st) {
  RL_CHECK_ARG(W && Thi && Tlo, "null pointer");
  RL_CHECK_ARG(rows > 0 && cols > 0 && ldw >= cols && ldt >= rows, "bad transposed-split geometry");
  dim3 grid(ceil_div(cols, 32), ceil_div(ldt, 32));
  tf32_split_t_kernel<<<grid, dim3(32, 8), 0, st>>>(W, Thi, Tlo, rows, cols, ldw, ldt);
  RL_CHECK_LAUNCH();
  return B200RL_OK;
}

// Shapes the tensor-core path accepts: NT product, 16-byte aligned operands with row strides that are
// multiples of 16 bytes, and enough work to fill a tile.
extern "C" int b200rl_gemm_tc_supported(const float* A, const float* B, int M, int N, int K, int lda, int ldb,
                                        int transA, int transB) {
  (void)transA; (void)transB;      // all four layouts: a transposed operand is read MN-major, in place
  // M < 128 (the 64-row products of a per-step RSSM scan at the XL width) still runs here: TMA zero-fills the missing
  // rows of the 128-row box and the epilogue masks them; half of the tile is idle but these products are bound by
  // streaming the weight matrix, which the SIMT path does 5-10x slower
  if (M < 32 || N < 48 || K < 32) return 0;
  if ((lda & 3) || (ldb & 3)) return 0;
  if ((reinterpret_cast<uintptr_t>(A) & 15) || (reinterpret_cast<uintptr_t>(B) & 15)) return 0;
  return 1;
}

namespace {
// `fused`: when non-null the product always leaves its result as split-K partial tiles (one split is allowed) and the
// caller launches the reduction itself, fused with what follows (LayerNorm, activation, GRU gate): *fused receives the
// workspace geometry.
struct FusedTail { float* part; int ks, mpad, ldw; };

// Blo: non-null when B is given as its TF32 planes, B = hi plane and Blo = lo plane, both [N][K] (transB) with row
// stride ldb
int gemm_tc_impl(const float* A, const float* B, const float* Blo, float* C, const float* bias, int M, int N, int K,
                 int lda, int ldb, int ldc, int transA, int transB, int accumulate, cudaStream_t st, FusedTail* fused) {
  RL_CHECK_ARG(A && B && (C || fused), "null pointer");
  RL_CHECK_ARG(b200rl_gemm_tc_supported(A, B, M, N, K, lda, ldb, transA, transB), "shape not eligible for the tensor-core path");
  RL_CHECK_ARG(!Blo || (transB && !(reinterpret_cast<uintptr_t>(Blo) & 15)), "pre-split B must be 16-byte aligned [N][K] planes");
  const int BN = (N <= 64) ? 64 : 128;
  CUtensorMap ma, mb, mb2;
  // A: [M][K] (K-major) or, transposed, [K][M] (MN-major: boxes of 32 k-rows x 32 m);  B: [N][K] or [K][N]
  if (!transA) { if (int rc = get_map(A, M, K, lda, BM, &ma)) return rc; }
  else         { if (int rc = get_map(A, K, M, lda, 32, &ma)) return rc; }
  if (transB)  { if (int rc = get_map(B, N, K, ldb, BN, &mb)) return rc; }
  else         { if (int rc = get_map(B, K, N, ldb, 32, &mb)) return rc; }
  mb2 = mb;
  if (Blo && g_passes == 3) { if (int rc = get_map(Blo, N, K, ldb, BN, &mb2)) return rc; }
  dim3 grid((N + BN - 1) / BN, (M + BM - 1) / BM);
  TileGeo g = {};
  g.mode = MODE_GEMM;
  g.a_mn = transA ? 1 : 0;
  g.b_mn = transB ? 0 : 1;
  g.ksplits = 1;
  g.passes = g_passes;
  const int tiles = grid.x * grid.y, nkb = (K + BK - 1) / BK;
  if (tiles < 2 * kNumSMs && nkb >= 8) {
    // split-K for launches that cannot fill the SMs (the M = T*B = 1024 products of the imagination rollout, weight
    // gradients): pick the split count that minimises  waves x (k-blocks per CTA x t_kb + fixed cost)  with
    // t_kb ~ 0.8 us per 128x128x32 k-block, ~4 us of pipeline fill + epilogue per CTA, and for the fixed-order reduce
    // kernel behind a split product ~3 us + 0.3 us per split
    int best = 1;
    float best_t = 1e30f;
    const int max_sp = nkb / 4 < 32 ? nkb / 4 : 32;
    for (int sp = 1; sp <= (max_sp < 1 ? 1 : max_sp); ++sp) {
      const int per = (nkb + sp - 1) / sp, real = (nkb + per - 1) / per;
      const int waves = (tiles * real + kNumSMs - 1) / kNumSMs;
      const float t = waves * (per * 0.8f + 4.0f) + (real > 1 ? 3.0f + 0.3f * real : 0.0f);
      if (t < best_t - 1e-3f) { best_t = t; best = real; }
    }
    g.ksplits = best;
  }
  if (g.ksplits > 1 || fused) {
    grid.z = g.ksplits;
    g.mpad = (int)grid.y * BM;
    g.ldw = (int)grid.x * BN;
    if (int rc = split_workspace((size_t)g.ksplits * g.mpad * g.ldw, st, &g.part)) return rc;
    if (fused) { g.force_part = 1; *fused = FusedTail{g.part, g.ksplits, g.mpad, g.ldw}; }
  }
  g.mtiles = (int)grid.y;
  g.ntiles = (int)grid.x;
  grid.x = 1;
  grid.y = persistent_grid_y(g.mtiles * g.ntiles, grid.z);
  DISPATCH_GEMM_TC(BN, g.passes, Blo != nullptr, grid, st, ma, mb, mb2, C, bias, M, N, K, ldc, accumulate, g);
  RL_CHECK_LAUNCH();
  if (g.ksplits > 1 && !fused) {
    splitk_reduce_kernel<<<ceil_div((long long)M * ((N + 3) / 4), 256), 256, 0, st>>>(g.part, C, bias, M, N, ldc, g.ksplits, g.mpad,
                                                                                      g.ldw, accumulate);
    RL_CHECK_LAUNCH();
  }
  return B200RL_OK;
}

// Fixed-order sum of the split-K partial tiles of a row, fused with LayerNorm (+ activation) or LayerNorm + GRU gate.
// One warp per row, the row in registers (NV float4 per lane, N = 128 * NV or less).
//   mode 0: out = act(LN(pre));  mode 1 (N = 3R, R % 128 == 0): LayerNormGRUCell gate (models.py:396-403) on the
//   normalised (reset | cand | update) thirds with h_prev -> h_out (and h_out2).  `pre` / `ln_out` are optional saves.
template <int NV>
__global__ void __launch_bounds__(256)
splitk_ln_kernel(const float* __restrict__ part, int ks, int mpad, int ldw, int M, int N, const float* __restrict__ gamma,
                 const float* __restrict__ beta, float eps, int act, float* __restrict__ pre, long long ldpre,
                 float* __restrict__ ln_out, long long ldln, int mode, const float* __restrict__ h_prev, long long ldh,
                 float* __restrict__ h_out, long long ldho, float* __restrict__ h_out2, long long ldho2) {
  const int lane = threadIdx.x & 31;
  const long long row = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (row >= M) return;
  const int n4 = N >> 2;
  float4 v[NV];
#pragma unroll
  for (int i = 0; i < NV; ++i) v[i] = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 4                                    // the splits' loads in flight together; the adds keep split order
  for (int z = 0; z < ks; ++z) {
    const float4* p = reinterpret_cast<const float4*>(part + ((size_t)z * mpad + row) * ldw);
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int c = lane + 32 * i;
      if (c < n4) { const float4 t = __ldcg(p + c); v[i].x += t.x; v[i].y += t.y; v[i].z += t.z; v[i].w += t.w; }
    }
  }
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int c = lane + 32 * i;
    if (c < n4) {
      if (pre) reinterpret_cast<float4*>(pre + row * ldpre)[c] = v[i];
      s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
    }
  }
  const float mu = warp_sum(s) / (float)N;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int c = lane + 32 * i;
    if (c < n4) {
      const float dx = v[i].x - mu, dy = v[i].y - mu, dz = v[i].z - mu, dw = v[i].w - mu;
      q += (dx * dx + dy * dy) + (dz * dz + dw * dw);
    }
  }
  const float rstd = rsqrtf(warp_sum(q) / (float)N + eps);
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int c = lane + 32 * i;
    if (c < n4) {
      const float4 g = reinterpret_cast<const float4*>(gamma)[c], b = reinterpret_cast<const float4*>(beta)[c];
      v[i].x = (v[i].x - mu) * rstd * g.x + b.x; v[i].y = (v[i].y - mu) * rstd * g.y + b.y;
      v[i].z = (v[i].z - mu) * rstd * g.z + b.z; v[i].w = (v[i].w - mu) * rstd * g.w + b.w;
      if (mode == 0 && act == 1) {   // SiLU
        v[i].x = v[i].x / (1.f + expf(-v[i].x)); v[i].y = v[i].y / (1.f + expf(-v[i].y));
        v[i].z = v[i].z / (1.f + expf(-v[i].z)); v[i].w = v[i].w / (1.f + expf(-v[i].w));
      }
      if (ln_out) reinterpret_cast<float4*>(ln_out + row * ldln)[c] = v[i];
    }
  }
  if (mode == 1) {
    constexpr int NR = NV / 3;      // float4 per lane of one third (R = 128 * NR)
#pragma unroll
    for (int i = 0; i < NR; ++i) {
      const int c = lane + 32 * i;
      const float4 hp = reinterpret_cast<const float4*>(h_prev + row * ldh)[c];
      const float4 gr = v[i], gc = v[i + NR], gu = v[i + 2 * NR];
      float4 h;
      auto gate = [](float r_, float c_, float u_, float hprev) {
        const float r = 1.f / (1.f + expf(-r_));
        const float cand = tanhf(r * c_);
        const float u = 1.f / (1.f + expf(-(u_ - 1.f)));
        return u * cand + (1.f - u) * hprev;
      };
      h.x = gate(gr.x, gc.x, gu.x, hp.x); h.y = gate(gr.y, gc.y, gu.y, hp.y);
      h.z = gate(gr.z, gc.z, gu.z, hp.z); h.w = gate(gr.w, gc.w, gu.w, hp.w);
      reinterpret_cast<float4*>(h_out + row * ldho)[c] = h;
      if (h_out2) reinterpret_cast<float4*>(h_out2 + row * ldho2)[c] = h;
    }
  }
}
}  // namespace

extern "C" int b200rl_gemm_tc(const float* A, const float* B, float* C, const float* bias, int M, int N, int K, int lda,
                              int ldb, int ldc, int transA, int transB, int accumulate, cudaStream_t st) {
  return gemm_tc_impl(A, B, nullptr, C, bias, M, N, K, lda, ldb, ldc, transA, transB, accumulate, st, nullptr);
}

extern "C" int b200rl_gemm_tc_presplit_supported(const float* A, const float* Bhi, const float* Blo, int M, int N, int K,
                                                 int lda, int ldb) {
  return b200rl_gemm_tc_supported(A, Bhi, M, N, K, lda, ldb, 0, 1) && !(reinterpret_cast<uintptr_t>(Blo) & 15);
}
extern "C" int b200rl_gemm_tc_presplit(const float* A, const float* Bhi, const float* Blo, float* C, const float* bias, int M,
                                       int N, int K, int lda, int ldb, int ldc, int accumulate, cudaStream_t st) {
  RL_CHECK_ARG(Blo, "null pointer");
  return gemm_tc_impl(A, Bhi, Blo, C, bias, M, N, K, lda, ldb, ldc, 0, 1, accumulate, st, nullptr);
}

extern "C" int b200rl_gemm_ln_supported(const float* A, const float* B, int M, int N, int K, int lda, int ldb, int mode) {
  if (!b200rl_gemm_tc_supported(A, B, M, N, K, lda, ldb, 0, 1)) return 0;
  if (N % 4 || N > 1536) return 0;
  if (mode == 1 && (N % 384 != 0)) return 0;      // three thirds of R = 128 * k columns each
  return 1;
}

namespace {
// Wlo: non-null when W is the TF32 hi plane of the weight and Wlo its lo plane
int gemm_ln_impl(const float* A, const float* W, const float* Wlo, int M, int N, int K, int lda, int ldw_, const float* gamma,
                 const float* beta, float eps, int act, float* pre, long long ldpre, float* out, long long ldout, int mode,
                 const float* h_prev, long long ldh, float* h_out, long long ldho, float* h_out2, long long ldho2,
                 cudaStream_t st) {
  RL_CHECK_ARG(A && W && gamma && beta, "null pointer");
  RL_CHECK_ARG(b200rl_gemm_ln_supported(A, W, M, N, K, lda, ldw_, mode), "shape not eligible for the fused product + LayerNorm");
  RL_CHECK_ARG(mode == 0 ? out != nullptr : (h_prev && h_out), "missing output");
  RL_CHECK_ARG(((reinterpret_cast<uintptr_t>(gamma) | reinterpret_cast<uintptr_t>(beta) | reinterpret_cast<uintptr_t>(pre) |
                 reinterpret_cast<uintptr_t>(out) | reinterpret_cast<uintptr_t>(h_prev) | reinterpret_cast<uintptr_t>(h_out) |
                 reinterpret_cast<uintptr_t>(h_out2)) & 15) == 0 &&
                   ((ldpre | ldout | ldh | ldho | ldho2) & 3) == 0,
               "fused product + LayerNorm needs 16-byte aligned rows");
  FusedTail ft;
  if (int rc = gemm_tc_impl(A, W, Wlo, nullptr, nullptr, M, N, K, lda, ldw_, N, 0, 1, 0, st, &ft)) return rc;
  const int blocks = ceil_div((long long)M * 32, 256);
#define LAUNCH_SPLITK_LN(NV_)                                                                                              \
  splitk_ln_kernel<NV_><<<blocks, 256, 0, st>>>(ft.part, ft.ks, ft.mpad, ft.ldw, M, N, gamma, beta, eps, act, pre, ldpre, out, \
                                                ldout, mode, h_prev, ldh, h_out, ldho, h_out2, ldho2)
  if (mode == 1) {
    if (N == 384) LAUNCH_SPLITK_LN(3); else if (N == 768) LAUNCH_SPLITK_LN(6); else if (N == 1152) LAUNCH_SPLITK_LN(9);
    else LAUNCH_SPLITK_LN(12);
  } else if (N <= 128) LAUNCH_SPLITK_LN(1);
  else if (N <= 256) LAUNCH_SPLITK_LN(2);
  else if (N <= 512) LAUNCH_SPLITK_LN(4);
  else if (N <= 1024) LAUNCH_SPLITK_LN(8);
  else LAUNCH_SPLITK_LN(12);
#undef LAUNCH_SPLITK_LN
  RL_CHECK_LAUNCH();
  return B200RL_OK;
}
}  // namespace

extern "C" int b200rl_gemm_ln(const float* A, const float* W, int M, int N, int K, int lda, int ldw_, const float* gamma,
                              const float* beta, float eps, int act, float* pre, long long ldpre, float* out, long long ldout,
                              int mode, const float* h_prev, long long ldh, float* h_out, long long ldho, float* h_out2,
                              long long ldho2, cudaStream_t st) {
  return gemm_ln_impl(A, W, nullptr, M, N, K, lda, ldw_, gamma, beta, eps, act, pre, ldpre, out, ldout, mode, h_prev, ldh,
                      h_out, ldho, h_out2, ldho2, st);
}
extern "C" int b200rl_gemm_ln_presplit_supported(const float* A, const float* Whi, const float* Wlo, int M, int N, int K,
                                                 int lda, int ldw, int mode) {
  return b200rl_gemm_ln_supported(A, Whi, M, N, K, lda, ldw, mode) && !(reinterpret_cast<uintptr_t>(Wlo) & 15);
}
extern "C" int b200rl_gemm_ln_presplit(const float* A, const float* Whi, const float* Wlo, int M, int N, int K, int lda,
                                       int ldw, const float* gamma, const float* beta, float eps, int act, float* pre,
                                       long long ldpre, float* out, long long ldout, int mode, const float* h_prev,
                                       long long ldh, float* h_out, long long ldho, float* h_out2, long long ldho2,
                                       cudaStream_t st) {
  RL_CHECK_ARG(Wlo, "null pointer");
  return gemm_ln_impl(A, Whi, Wlo, M, N, K, lda, ldw, gamma, beta, eps, act, pre, ldpre, out, ldout, mode, h_prev, ldh,
                      h_out, ldho, h_out2, ldho2, st);
}

// ---- convolution weight gradient on the tensor cores, operands read in place (no im2col, no transposes):
//   G[(tap, cb), cs] = sum over small pixels p of big[patch(p)][tap][cb] * small[p][cs]
// A = gathered big image, MN-major (rows (tap, cb), K = pixels); B = small [P][Cs], MN-major; split-K over pixels.
extern "C" int b200rl_conv_wgrad_mn_supported(int NB, int h, int w, int Cs, int Cb) {
  if (w <= 0 || h <= 0 || (w & (w - 1)) || (h & (h - 1))) return 0;
  const long long P = (long long)NB * h * w;
  if (Cb % 32 || Cs < 48 || Cs % 4 || P % 32 || P < 1024 || P > 2000000000LL) return 0;
  // the 32 pixels of a k-block must be one box: part of a row, whole rows of one image, or whole images
  const int bw = w < 32 ? w : 32, bh = (32 / bw) < h ? (32 / bw) : h, bn = 32 / (bw * bh);
  return (bw * bh * bn == 32) && (NB % bn == 0);
}

extern "C" int b200rl_conv_wgrad_mn(const float* small_, const float* big, float* G, int NB, int h, int w, int Cs, int Cb,
                                    cudaStream_t st) {
  RL_CHECK_ARG(small_ && big && G, "null pointer");
  RL_CHECK_ARG(b200rl_conv_wgrad_mn_supported(NB, h, w, Cs, Cb), "shape not eligible for the in-place wgrad path");
  const int P = NB * h * w, M = 16 * Cb, N = Cs;
  TileGeo g = {};
  g.mode = MODE_GEMM; g.a_mn = 1; g.b_mn = 1; g.wg = 1; g.passes = g_passes;
  g.h = h; g.w = w; g.NB = NB; g.Cout = Cb;
  g.bw = w < 32 ? w : 32; g.bh = (32 / g.bw) < h ? (32 / g.bw) : h; g.bn = 32 / (g.bw * g.bh);
  CUtensorMap ma, mb;
  if (int rc = get_map4(big, Cb, 2 * w, 2 * h, NB, g.bw, g.bh, g.bn, 2, &ma)) return rc;
  if (int rc = get_map(small_, P, Cs, Cs, 32, &mb)) return rc;
  const int BN = (N <= 64) ? 64 : 128;
  dim3 grid((N + BN - 1) / BN, M / BM);
  const int tiles = grid.x * grid.y, nkb = P / BK;
  int sp = (2 * kNumSMs + tiles - 1) / tiles;
  if (sp > nkb / 8) sp = nkb / 8;
  if (sp < 1) sp = 1;
  const int per = (nkb + sp - 1) / sp;
  g.ksplits = (nkb + per - 1) / per;
  grid.z = g.ksplits;
  g.mtiles = (int)grid.y;
  g.ntiles = (int)grid.x;
  if (g.ksplits > 1) {
    g.mpad = (int)grid.y * BM;
    g.ldw = (int)grid.x * BN;
    if (int rc = split_workspace((size_t)g.ksplits * g.mpad * g.ldw, st, &g.part)) return rc;
  }
  grid.x = 1;
  grid.y = (unsigned)(g.mtiles * g.ntiles);
  DISPATCH_GEMM_TC(BN, g.passes, false, grid, st, ma, mb, mb, G, nullptr, M, N, P, N, 0, g);
  RL_CHECK_LAUNCH();
  if (g.ksplits > 1) {
    splitk_reduce_kernel<<<ceil_div((long long)M * ((N + 3) / 4), 256), 256, 0, st>>>(g.part, G, nullptr, M, N, N, g.ksplits, g.mpad,
                                                                                      g.ldw, 0);
    RL_CHECK_LAUNCH();
  }
  return B200RL_OK;
}
