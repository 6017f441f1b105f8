// K2b — the headline kernel: moments  M = [X|Y|1]^T [X|Y|1]  for f32 frames on the Hopper tensor cores (wgmma + TMA).
//
// Replaces faer's matmul in get_xtx_with_lambda / build_xty (/root/reference/src/linear/lr/lr_solvers.rs:183-211,
// 262-278) and the column sums of faer_coordinate_descent (:483-484): one pass over the frame instead of three.
//
// Shape of the problem: X has p <= 64 columns and n ~ 1e8 rows, i.e. a GEMM with M = N = p and K = n — tiny output,
// enormous reduction.  At p = 32 the FP32 SIMT pipes cannot keep up with HBM (595 FMA per 132-byte row), so X'X goes
// to wgmma.mma_async .tf32 — and because one TF32 product loses 13 mantissa bits it is computed as the classic
// 3-term split  x = hi + lo  (hi = x with the low 13 mantissa bits cleared, lo = x - hi, exact in fp32):
//        X'X = HH + LH + LH^T (+ LL ~ 2^-22, dropped),     HH = hi^T hi,  LH = lo^T hi.
// Both products come out of ONE instruction stream by stacking hi and lo along the MMA's M dimension:
//        A  (registers, 64 rows x 8 per wgmma): hi and lo of the feature columns, loaded from the tile and split in place
//        B  (SMEM, N x 8, K-major, 128B swizzle): the feature rows of the TMA tile as they landed, N = p padded to 16
// The hi operand is the RAW data: the tensor core reads an fp32 operand as TF32 by ignoring the low 13 mantissa bits
// (tests/test_gpu_moments.py compares against exact-product f64-accumulated moments, and variant 0 — hi rows that clear
// those bits themselves — against the raw variant bit for bit), so B needs no conversion and the hi rows of A are a copy.
//
// Only the FEATURES go through the tensor core.  What the targets and the ones column contribute is O(p t) per row and
// runs on the CUDA cores of two side warps:  x . y_j, sum x, sum y, y_j . y_k and the masked row count.
//
// A-row layout.  An m64 block of A holds 32 features: warp q of the warpgroup has feature 8q + g (g = lane / 4) as hi in
// its fragment row g and as lo in row g + 8, so one shared-memory load gives a thread both of its A registers for that
// k (the row order of A only permutes the rows of D).  Up to 32 features (NB <= 2) one m64 wgmma carries everything and
// three consumer warpgroups take every third stage each.  From 33 to 64 features warpgroup 0 holds features 0..31 and
// warpgroup 1 features 32..63, and both work on every stage.
//
// Data flow per CTA (persistent, one CTA per SM, 128-row stages dealt round-robin):
//   warps 0 .. 4W-1    W consumer warpgroups (W = 3 up to 32 features, else 2): tile -> registers (hi / lo) -> 16 x wgmma
//                      (K = 8) per stage, fp32 accumulators in registers, added to f64 registers after every stage
//   warps 4W, 4W+1     side warps: warp k takes boxes 2k, 2k + 1 of every stage for the target / ones-column sums
//   warp 4W+2          TMA producer: cp.async.bulk.tensor, per 32-row box one {32 x p} load of X and one {32 x t} of Y
// A second tiny kernel sums the per-CTA partials in a fixed order (bit-reproducible) and applies the symmetrisation.
// Roofline: HBM-bound, algorithmic bytes = 4 (p + t) per row (+4 with a mask).
#include "../common.h"
#include "kernels.h"
#include "f32x2.h"
#include "mbarrier.h"
#include <cuda.h>

namespace pdsb {

namespace {

constexpr int BOX_ROWS = 32;            // K extent of one TMA box = 128 bytes of f32 = one swizzle row
constexpr int BPS = 4;                  // boxes per pipeline stage  (stage = 128 rows)
constexpr int STAGE_ROWS = BOX_ROWS * BPS;
constexpr int MAX_RING = 15;            // TMA landing ring (stages)
constexpr int PART_SLOTS = 3;           // partial slots per CTA: one per consumer warpgroup (at most three)
constexpr int NSIDE = 2;                // side warps (two boxes of every stage each)
constexpr int PART_ROWS = 128;          // partial rows per (CTA, slot): hi of feature c at row c, lo at row 64 + c
constexpr int Y_ROWS = 8;               // tile rows reserved for the targets (t <= 4; one 8-row swizzle group)
constexpr int MAX_T = 4;
constexpr uint32_t HI_MASK = 0xFFFFE000u;   // TF32 keeps 10 mantissa bits
constexpr int SIDE_SLOTS = NSIDE;       // partial slots per CTA for the side sums
constexpr int XSIDE_COLS = 64;          // doubles per (CTA, side warp, slot): slot j < T = x . y_j, slot T = sum x
constexpr int YSIDE_STRIDE = 32;        // doubles per (CTA, side warp): [3u+0] sum y_u, [3u+1] sum y_u^2, [2] count, [12 + 4j + k] y_j.y_k

template <int NB>
struct Shape {
  static constexpr int N = NB * 16;                                  // MMA N = feature rows of the tile, padded to 16
  static constexpr int MB = NB <= 2 ? 1 : 2;                         // m64 blocks of the A operand (hi and lo stacked)
  static constexpr int TILE_ROWS = N + Y_ROWS;                       // feature rows, then the target rows
  static constexpr uint32_t TILE_BYTES = TILE_ROWS * 128;            // one box-tile (a multiple of 1024 bytes)
  // ring depth: as many stages as fit in ~200 KB of the 227 KB a block may use (bytes in flight per SM are what
  // keeps HBM busy)
  // consumer warpgroups: three taking every third stage up to 32 features (15 warps = 480 threads: four warps on a
  // scheduler cap a thread at 128 registers, which these variants fit); two (features 0..31 / 32..63) on every stage
  // above
  static constexpr int NWG = NB <= 2 ? 3 : 2;
  static constexpr int NUM_THREADS = (4 * NWG + NSIDE + 1) * 32;
  static constexpr int RING = (NB == 1) ? 15 : (NB == 2 ? 9 : (NB == 3 ? 7 : 5));
  static constexpr size_t SMEM = (size_t)RING * BPS * TILE_BYTES;
  // consumer arrivals that free a ring slot: one per consumer warp that reads the stage
  static constexpr int CONSUMER_WARPS = MB == 2 ? 4 * NWG : 4;
  // a warpgroup waits on a slot's parity only if it also consumed the slot's previous phase
  static_assert(MB == 2 || RING % NWG == 0, "every ring slot must go to the same warpgroup");
};

// ---------------------------------------------------------------- PTX helpers ----------------------------
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2) : "memory");
}
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int K>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(K) : "memory"); }
// keeps the compiler from moving accumulator reads / writes across the asynchronous MMAs
template <int R>
__device__ __forceinline__ void fence_regs(float* d) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// wgmma shared-memory matrix descriptor (sm_90): K-major, 128-byte swizzle, 8-row groups 1024 bytes apart
__device__ __forceinline__ uint64_t make_b_desc(uint32_t saddr) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr & 0x3FFFF) >> 4);          // start address        bits [0,14)
  d |= (uint64_t)1 << 16;                           // leading byte offset  (unused for swizzled K-major)
  d |= (uint64_t)(1024 >> 4) << 32;                 // stride byte offset   bits [32,46)
  d |= (uint64_t)1 << 62;                           // layout: SWIZZLE_128B
  return d;
}

// D (m64 x N, f32, registers) (+)= A (m64 x k8, tf32, registers) * B (N x k8, tf32, shared memory)^T
template <int N> struct Wgmma;
template <> struct Wgmma<16> {
  static __device__ __forceinline__ void mma(float* d, const uint32_t* a, uint64_t b_desc, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %13, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n16k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7}, {%8, %9, %10, %11}, %12, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc), "r"(accumulate));
  }
};
template <> struct Wgmma<32> {
  static __device__ __forceinline__ void mma(float* d, const uint32_t* a, uint64_t b_desc, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %21, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, {%16, %17, %18, %19}, %20, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc), "r"(accumulate));
  }
};
template <> struct Wgmma<48> {
  static __device__ __forceinline__ void mma(float* d, const uint32_t* a, uint64_t b_desc, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %29, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n48k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23}, {%24, %25, %26, %27}, %28, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc), "r"(accumulate));
  }
};
template <> struct Wgmma<64> {
  static __device__ __forceinline__ void mma(float* d, const uint32_t* a, uint64_t b_desc, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc), "r"(accumulate));
  }
};

struct alignas(8) Barriers {
  uint64_t raw_full[MAX_RING], raw_empty[MAX_RING];   // TMA landed / tile free again (consumers and side warps done)
};

struct GramArgs {
  int64_t n, stages_total;
  int p, t;
  int xcol, ycol;        // row-blocked frame: first feature / target column of the frame
  int blocked;           // row-blocked frame (3-D tensor maps) or column-major matrices (2-D)
  int explicit_hi;       // cross-check: the hi rows clear the low 13 bits themselves
  int joined;            // Y follows X in memory and p is a multiple of 16: ONE box {32 x (p + t)} per load lands Y at tile row N
};

// A fragment of one 32-row box for this thread: 4 k-steps x {a0..a3}.  Fragment layout of wgmma .tf32 (per warp,
// 16 rows): a0 (row g, k c), a1 (row g + 8, k c), a2 (row g, k c + 4), a3 (row g + 8, k c + 4), g = lane / 4, c = lane % 4.
// Rows g and g + 8 are the hi and lo of the same feature (tile row at rowoff, swizzle sw), so one load per k gives both:
// hi keeps the raw value (or clears the low bits itself in the cross-check variant), lo subtracts the TF32 truncation.
__device__ __forceinline__ void load_a_box(const unsigned char* tile, int rowoff, uint32_t sw, bool explicit_hi, int c,
                                           uint32_t (*a)[4]) {
#pragma unroll
  for (int ks = 0; ks < BOX_ROWS / 8; ++ks) {
#pragma unroll
    for (int kh = 0; kh < 2; ++kh) {                                         // data row ks * 8 + 4 kh + c of the box
      const uint32_t chunk = (uint32_t)(ks * 2 + kh);
      const uint32_t v = *reinterpret_cast<const uint32_t*>(tile + rowoff + ((chunk ^ sw) << 4) + (c << 2));
      const uint32_t hb = v & HI_MASK;
      a[ks][2 * kh] = explicit_hi ? hb : v;
      // v - hb (round-to-nearest, exact) computed straight into a 32-bit integer register: a float result would be
      // moved into the operand register after wgmma.fence, and ptxas would inject a second fence before each MMA
      asm("sub.rn.f32 %0, %1, %2;" : "=r"(a[ks][2 * kh + 1]) : "r"(v), "r"(hb));
    }
  }
}

// T = targets the side lanes are compiled for (1, or 4 for t = 2..4)
template <int NB, int T>
__global__ void __launch_bounds__(Shape<NB>::NUM_THREADS, 1)
gram_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_x, const __grid_constant__ CUtensorMap tmap_y,
                  const float* __restrict__ mask, const GramArgs g, double* __restrict__ partials /* [grid][PART_SLOTS][128][N] */,
                  double* __restrict__ xside /* [grid][SIDE_SLOTS][T+1][64] */, double* __restrict__ yside /* [grid][SIDE_SLOTS][32] */  /* both zero-filled */) {
  using S = Shape<NB>;
  constexpr int N = S::N, MB = S::MB, RING = S::RING, NACC = N / 2;
  constexpr uint32_t TILE_BYTES = S::TILE_BYTES;
  constexpr int NWG = S::NWG, NUM_THREADS = S::NUM_THREADS;
  extern __shared__ unsigned char smem_dyn[];
  // 128-byte swizzled TMA tiles and the wgmma descriptors assume 1024-byte aligned tiles.  The base is smem_dyn plus an
  // offset (not a round trip through an integer address) so that the compiler keeps the shared state space: every tile
  // read below is then an LDS with a 32-bit address instead of a generic load.
  unsigned char* raw = smem_dyn + ((1024u - (smem_u32(smem_dyn) & 1023u)) & 1023u);
  Barriers* bars = reinterpret_cast<Barriers*>(raw + S::SMEM);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int p = g.p, t = g.t;
  // stages are dealt round-robin: at any moment the CTAs stream ADJACENT rows of every column (DRAM page locality)
  const uint32_t my_stages = g.stages_total > (int64_t)blockIdx.x
                                 ? (uint32_t)((g.stages_total - 1 - blockIdx.x) / gridDim.x + 1) : 0u;
  auto stage_row0 = [&](uint32_t it) { return ((int64_t)it * gridDim.x + blockIdx.x) * STAGE_ROWS; };

  if (threadIdx.x == 0) {
    for (int i = 0; i < RING; ++i) { mbar_init(&bars->raw_full[i], 1); mbar_init(&bars->raw_empty[i], S::CONSUMER_WARPS + NSIDE); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  // rows the TMA never writes (feature rows p .. N-1 feed accumulator columns nobody reads, target rows t .. 7 feed
  // side lanes whose results nobody reads): zero them once so that nothing uninitialised is ever multiplied
  for (int i = threadIdx.x; i < RING * BPS * (S::TILE_ROWS - p - t) * 8; i += NUM_THREADS) {
    const int per = (S::TILE_ROWS - p - t) * 8;
    const int tile = i / per, rem = i % per;
    int r = rem / 8;
    const int c = rem % 8;
    r = (r < N - p) ? p + r : N + t + (r - (N - p));
    *reinterpret_cast<uint4*>(raw + (size_t)tile * TILE_BYTES + (size_t)r * 128 + c * 16) = make_uint4(0, 0, 0, 0);
  }
  fence_async_smem();
  __syncthreads();

  if (warp < 4 * NWG) {
    // =============================== consumer warpgroups: tile -> hi / lo registers -> wgmma ===============
    const int wg = warp >> 2, wq = warp & 3;
    const int gq = lane >> 2, c = lane & 3;
    // this thread's feature: hi in A row 16 wq + gq of its warpgroup's m64 block, lo in row 16 wq + gq + 8
    const int f = (MB == 2 ? 32 * wg : 0) + 8 * wq + gq;
    const int frow = f < p ? f : 0;                            // padding rows read a real row (their results are not read)
    const int rowoff = frow * 128;
    const uint32_t sw = (uint32_t)(frow & 7);
    const bool explicit_hi = g.explicit_hi != 0;
    float acc[NACC];
    double dacc[NACC];
#pragma unroll
    for (int j = 0; j < NACC; ++j) { acc[j] = 0.0f; dacc[j] = 0.0; }
    const uint32_t raw_addr = smem_u32(raw);
    // up to 32 features the warpgroups take stages round-robin; above, both take every stage (features 0..31 / 32..63)
    const uint32_t first = MB == 2 ? 0u : (uint32_t)wg, step = MB == 2 ? 1u : (uint32_t)NWG;
    // A registers double-buffered over the boxes: the loads of box b + 1 run while the MMAs of box b execute, and box 0
    // of this warpgroup's next stage loads while the last box of this stage executes, before the drain
    uint32_t a[2][BOX_ROWS / 8][4];
    if (first < my_stages) {
      mbar_wait(&bars->raw_full[first % RING], (first / RING) & 1);
      load_a_box(raw + (size_t)(first % RING) * BPS * TILE_BYTES, rowoff, sw, explicit_hi, c, a[0]);
    }
    for (uint32_t it = first; it < my_stages; it += step) {
      const uint32_t rs = it % RING, nxt = it + step;
      const unsigned char* st = raw + (size_t)rs * BPS * TILE_BYTES;
      const uint32_t st_addr = raw_addr + rs * (BPS * TILE_BYTES);
#pragma unroll
      for (int b = 0; b < BPS; ++b) {
        wg_fence();
        fence_regs<NACC>(acc);
        const uint64_t bd = make_b_desc(st_addr + b * TILE_BYTES);
#pragma unroll
        for (int ks = 0; ks < BOX_ROWS / 8; ++ks)
          // descriptor start address advances in 16-byte units: +32 bytes per K = 8 step inside the swizzle row
          Wgmma<N>::mma(acc, a[b & 1][ks], bd + (uint64_t)((ks * 32) >> 4), (b == 0 && ks == 0) ? 0u : 1u);
        wg_commit();
        fence_regs<NACC>(acc);
        if (b + 1 < BPS) {
          wg_wait<1>();                                        // box b - 1 done: its A buffer is free
          load_a_box(st + (b + 1) * TILE_BYTES, rowoff, sw, explicit_hi, c, a[(b + 1) & 1]);
        } else if (nxt < my_stages) {
          mbar_wait(&bars->raw_full[nxt % RING], (nxt / RING) & 1);
          wg_wait<1>();                                        // box BPS - 2 done: a[0] is free
          load_a_box(raw + (size_t)(nxt % RING) * BPS * TILE_BYTES, rowoff, sw, explicit_hi, c, a[0]);
        }
      }
      wg_wait<0>();
      fence_regs<NACC>(acc);
      __syncwarp();
      if (lane == 0) mbar_arrive(&bars->raw_empty[rs]);        // this warp's reads of the tile are complete
      // 128 rows of fp32 accumulation inside the tensor core, then f64
#pragma unroll
      for (int j = 0; j < NACC; ++j) dacc[j] += (double)acc[j];
    }
    // accumulator layout (m64nN f32): element j -> row 16 wq + g + 8 ((j / 2) % 2), column 8 (j / 4) + 2 c + (j % 2);
    // row 16 wq + g is the hi of feature f (partial row f), row 16 wq + g + 8 its lo (partial row 64 + f)
    const int slot = MB == 2 ? 0 : wg;
    double* out = partials + ((size_t)blockIdx.x * PART_SLOTS + slot) * PART_ROWS * N;
#pragma unroll
    for (int j = 0; j < NACC; ++j) {
      const int prow = 64 * ((j >> 1) & 1) + f;
      out[(size_t)prow * N + 8 * (j >> 2) + 2 * c + (j & 1)] = dacc[j];
    }
  } else if (warp < 4 * NWG + NSIDE) {
    // =============================== side warps: warp k takes boxes 2k, 2k + 1 of EVERY stage, lane = feature ======
    // x . y_j and sum x over NATURAL register pairs (a 16-byte load gives rows (4c, 4c+1), (4c+2, 4c+3) of the column, the
    // broadcast load of y_j the same rows of the target: one pair FMA / add per two rows); above 32 features a lane also
    // takes feature lane + 32.  Lanes 8j + c hold chunk c of target j (sum y, y_j . y_k); lanes 0..7 count the rows of a
    // masked frame.  f32 partial sums (chains of at most 128 terms) go to the f64 totals every SIDE_FLUSH stages.
    constexpr int FH = NB > 2 ? 2 : 1;                         // features per lane
    constexpr uint32_t SIDE_FLUSH = 4;
    const int sw_id = warp - 4 * NWG;
    int frow[FH];
    uint32_t fsw[FH];
#pragma unroll
    for (int h = 0; h < FH; ++h) {
      const int f = lane + 32 * h;
      frow[h] = f < p ? f : 0;
      fsw[h] = (uint32_t)(frow[h] & 7);
    }
    float2 axy[FH][T][2], asx[FH][2];
#pragma unroll
    for (int h = 0; h < FH; ++h) {
#pragma unroll
      for (int j = 0; j < T; ++j) axy[h][j][0] = axy[h][j][1] = make_float2(0.0f, 0.0f);
      asx[h][0] = asx[h][1] = make_float2(0.0f, 0.0f);
    }
    double dxs[FH][T + 1];
#pragma unroll
    for (int h = 0; h < FH; ++h)
#pragma unroll
      for (int j = 0; j <= T; ++j) dxs[h][j] = 0.0;
    float sy = 0.0f, syy = 0.0f, sxy[3] = {0.0f, 0.0f, 0.0f};
    double dsy = 0.0, dsyy = 0.0, dcnt = 0.0, dxy[3] = {0.0, 0.0, 0.0};
    uint32_t rs = 0, rph = 0;
    for (uint32_t it = 0; it < my_stages; ++it) {
      mbar_wait(&bars->raw_full[rs], rph);
#pragma unroll 1
      for (int bb = 0; bb < BPS / NSIDE; ++bb) {
      const int b = sw_id * (BPS / NSIDE) + bb;
      const unsigned char* tile = raw + ((size_t)rs * BPS + b) * TILE_BYTES;
      // chunk by chunk (four rows), so that each target chunk is loaded once per box for all the lane's features
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        uint4 yv[T];
#pragma unroll
        for (int j = 0; j < T; ++j) yv[j] = *reinterpret_cast<const uint4*>(tile + (size_t)(N + j) * 128 + ((c ^ j) << 4));   // same address in every lane
#pragma unroll
        for (int h = 0; h < FH; ++h) {
          const uint4 xv = *reinterpret_cast<const uint4*>(tile + (size_t)frow[h] * 128 + ((c ^ fsw[h]) << 4));
#pragma unroll
          for (int j = 0; j < T; ++j) {
            axy[h][j][0] = ffma2(make_float2(__uint_as_float(xv.x), __uint_as_float(xv.y)),
                                 make_float2(__uint_as_float(yv[j].x), __uint_as_float(yv[j].y)), axy[h][j][0]);
            axy[h][j][1] = ffma2(make_float2(__uint_as_float(xv.z), __uint_as_float(xv.w)),
                                 make_float2(__uint_as_float(yv[j].z), __uint_as_float(yv[j].w)), axy[h][j][1]);
          }
          asx[h][0] = fadd2(asx[h][0], make_float2(__uint_as_float(xv.x), __uint_as_float(xv.y)));
          asx[h][1] = fadd2(asx[h][1], make_float2(__uint_as_float(xv.z), __uint_as_float(xv.w)));
        }
      }
      if (lane < 8 * t) {
        const int j = lane >> 3, c = lane & 7;
        const uint4 yv = *reinterpret_cast<const uint4*>(tile + (size_t)(N + j) * 128 + ((c ^ j) << 4));
        const float y0 = __uint_as_float(yv.x), y1 = __uint_as_float(yv.y), y2 = __uint_as_float(yv.z), y3 = __uint_as_float(yv.w);
        sy += (y0 + y1) + (y2 + y3);
        syy = fmaf(y0, y0, fmaf(y1, y1, fmaf(y2, y2, fmaf(y3, y3, syy))));
        if (T > 1) {
#pragma unroll
          for (int d = 1; d < 4; ++d)
            if (j + d < t) {
              const int kr = j + d;
              const uint4 kv = *reinterpret_cast<const uint4*>(tile + (size_t)(N + kr) * 128 + ((c ^ kr) << 4));
              sxy[d - 1] = fmaf(y0, __uint_as_float(kv.x), fmaf(y1, __uint_as_float(kv.y),
                           fmaf(y2, __uint_as_float(kv.z), fmaf(y3, __uint_as_float(kv.w), sxy[d - 1]))));
            }
        }
      }
      if (mask != nullptr && lane < 8) {
        // row count of a masked frame: the packer zeroes masked rows, so only the count needs the mask
        const int64_t r0 = stage_row0(it) + b * BOX_ROWS + lane * 4;
        float o = 0.0f;
#pragma unroll
        for (int e = 0; e < 4; ++e) if (r0 + e < g.n) o += __ldg(mask + r0 + e);
        dcnt += (double)o;
      }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&bars->raw_empty[rs]);
      if ((it % SIDE_FLUSH) == SIDE_FLUSH - 1 || it == my_stages - 1) {
#pragma unroll
        for (int h = 0; h < FH; ++h) {
#pragma unroll
          for (int j = 0; j < T; ++j) {
            const float2 a = fadd2(axy[h][j][0], axy[h][j][1]);
            dxs[h][j] += (double)(a.x + a.y);
            axy[h][j][0] = axy[h][j][1] = make_float2(0.0f, 0.0f);
          }
          const float2 a = fadd2(asx[h][0], asx[h][1]);
          dxs[h][T] += (double)(a.x + a.y);
          asx[h][0] = asx[h][1] = make_float2(0.0f, 0.0f);
        }
        dsy += (double)sy; dsyy += (double)syy; sy = 0.0f; syy = 0.0f;
        if (T > 1) {
#pragma unroll
          for (int d = 0; d < 3; ++d) { dxy[d] += (double)sxy[d]; sxy[d] = 0.0f; }
        }
      }
      if (++rs == RING) { rs = 0; rph ^= 1; }
    }
    double* xs = xside + ((size_t)blockIdx.x * SIDE_SLOTS + sw_id) * (T + 1) * XSIDE_COLS;
#pragma unroll
    for (int h = 0; h < FH; ++h)
      if (lane + 32 * h < p) {
#pragma unroll
        for (int j = 0; j <= T; ++j) xs[j * XSIDE_COLS + lane + 32 * h] = dxs[h][j];
      }
    double* ys = yside + ((size_t)blockIdx.x * SIDE_SLOTS + sw_id) * YSIDE_STRIDE;
    for (int off = 4; off; off >>= 1) {
      dsy += __shfl_down_sync(0xffffffffu, dsy, off, 8);
      dsyy += __shfl_down_sync(0xffffffffu, dsyy, off, 8);
      dcnt += __shfl_down_sync(0xffffffffu, dcnt, off, 8);
#pragma unroll
      for (int d = 0; d < 3; ++d) dxy[d] += __shfl_down_sync(0xffffffffu, dxy[d], off, 8);
    }
    if ((lane & 7) == 0 && (lane >> 3) < t) {
      const int j = lane >> 3;
      ys[j * 3 + 0] = dsy; ys[j * 3 + 1] = dsyy;
      for (int d = 1; d < 4; ++d) if (j + d < t) ys[12 + j * 4 + (j + d)] = dxy[d - 1];
    }
    if (lane == 0) ys[2] = dcnt;
  } else {
    // =============================== TMA producer (warp-uniform loop, one elected lane issues) ===============
    uint32_t rs = 0, ph = 0;
    for (uint32_t it = 0; it < my_stages; ++it) {
      mbar_wait(&bars->raw_empty[rs], ph ^ 1);
      if (elect_one()) {
        mbar_arrive_expect_tx(&bars->raw_full[rs], (uint32_t)(BPS * (p + t) * 128));
        const int64_t row0 = stage_row0(it);
#pragma unroll
        for (int b = 0; b < BPS; ++b) {
          unsigned char* dst = raw + ((size_t)rs * BPS + b) * TILE_BYTES;
          if (g.blocked) {
            tma_load_3d(dst, &tmap_x, &bars->raw_full[rs], b * BOX_ROWS, g.xcol, (int)(row0 / STAGE_ROWS));
            if (!g.joined) tma_load_3d(dst + N * 128, &tmap_y, &bars->raw_full[rs], b * BOX_ROWS, g.ycol, (int)(row0 / STAGE_ROWS));
          } else {
            tma_load_2d(dst, &tmap_x, &bars->raw_full[rs], (int)(row0 + b * BOX_ROWS), 0);
            if (!g.joined) tma_load_2d(dst + N * 128, &tmap_y, &bars->raw_full[rs], (int)(row0 + b * BOX_ROWS), 0);
          }
        }
      }
      __syncwarp();
      if (++rs == RING) { rs = 0; ph ^= 1; }
    }
  }
}

// Sum the per-CTA partials in a fixed order (bit-reproducible), X'X[a][b] = HH[a][b] + LH[a][b] + LH[b][a], and lay the
// moments out in the order [X | Y | 1].  One WARP per element of the upper triangle (mirrored -> exactly symmetric): lane
// l sums parts l, l + 32, ..., then a fixed-order xor tree.
__global__ void __launch_bounds__(256)
gram_finalize_kernel(const double* __restrict__ partials, const double* __restrict__ xside, const double* __restrict__ yside,
                     int nparts, int nslots, int N, int T, int p, int t, int64_t n, int masked, double* __restrict__ M) {
  const int q1 = p + t + 1;
  const int lane = threadIdx.x & 31;
  const int idx = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (idx >= q1 * q1) return;
  const int i = idx / q1, j = idx % q1;
  if (i > j) return;
  double r = 0.0;
  if (j < p) {                                     // X'X
    double hh = 0.0, hh_t = 0.0, lh_ij = 0.0, lh_ji = 0.0;
    for (int k = lane; k < nparts * nslots; k += 32) {
      const double* P = partials + ((size_t)(k % nparts) * PART_SLOTS + k / nparts) * PART_ROWS * N;
      hh += P[(size_t)i * N + j];
      hh_t += P[(size_t)j * N + i];
      lh_ij += P[(size_t)(64 + i) * N + j];
      lh_ji += P[(size_t)(64 + j) * N + i];
    }
    r = 0.5 * (hh + hh_t) + (lh_ij + lh_ji);      // per lane; the lanes are added below
  } else if (i < p) {                              // X'y_k (slot k) and the column sums (slot T) from the side sums
    const int slot = (j < p + t) ? j - p : T;
    for (int k = lane; k < nparts * SIDE_SLOTS; k += 32) r += xside[((size_t)k * (T + 1) + slot) * XSIDE_COLS + i];
  } else {
    // y / ones block from the side lanes: [3u+0] sum y_u, [3u+1] sum y_u^2, [2] count, [12 + 4a + b] y_a . y_b
    const int a = i - p, bb = j - p;
    int off;
    if (j == p + t) off = (i == p + t) ? 2 : a * 3 + 0;
    else off = (i == j) ? a * 3 + 1 : 12 + a * 4 + bb;
    if (!(j == p + t && i == p + t && !masked))
      for (int k = lane; k < nparts * SIDE_SLOTS; k += 32) r += yside[(size_t)k * YSIDE_STRIDE + off];
  }
  for (int off = 16; off; off >>= 1) r += __shfl_xor_sync(0xffffffffu, r, off);
  if (j == p + t && i == p + t && !masked) r = (double)n;
  if (lane == 0) {
    M[(size_t)i * q1 + j] = r;
    M[(size_t)j * q1 + i] = r;
  }
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) != cudaSuccess ||
        qres != cudaDriverEntryPointSuccess)
      p = nullptr;
    return reinterpret_cast<EncodeTiledFn>(p);
  }();
  return fn;
}

bool shape_ok(int p, int t) { return p >= 1 && p <= 64 && t >= 1 && t <= MAX_T; }

// 1 (default): raw hi operand;  0: the hi rows clear the low 13 bits themselves (proves the hardware truncation of A)
std::atomic<int> g_tc_mode{1};

template <int NB, int T>
int launch_one(const CUtensorMap& tx, const CUtensorMap& ty, const float* mask, const GramArgs& g, int grid,
               double* partials, double* xside, double* yside, cudaStream_t s) {
  const size_t smem = Shape<NB>::SMEM + 1024 /* alignment slack */ + sizeof(Barriers);
  auto k = gram_wgmma_kernel<NB, T>;
  PDSB_CUDA_OK(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  k<<<grid, Shape<NB>::NUM_THREADS, smem, s>>>(tx, ty, mask, g, partials, xside, yside);
  PDSB_LAUNCH_OK();
  count_launch();
  return 0;
}

// geometry of one call: where X and Y lie
struct Geometry {
  const float* xbase; const float* ybase;   // column-major: first feature / target column;  blocked: the frame (both)
  int64_t ldx, ldy;
  int ncols, xcol, ycol;                    // blocked frame
  bool blocked;
};

int encode_maps(const Geometry& g, int64_t n, int p, int t, bool joined, CUtensorMap* tx, CUtensorMap* ty) {
  EncodeTiledFn enc = get_encode_fn();
  if (!enc) return -1;
  CUresult cr = CUDA_SUCCESS;
  for (int which = 0; which < 2 && cr == CUDA_SUCCESS; ++which) {
    CUtensorMap* tm = which ? ty : tx;
    const int cols = which ? t : (joined ? p + t : p);
    if (g.blocked) {
      // row-blocked frame: [block][column][128 rows] -> every 128-row x ncols stage is ONE contiguous run in HBM
      cuuint64_t dims3[3] = {(cuuint64_t)STAGE_ROWS, (cuuint64_t)g.ncols, (cuuint64_t)ceil_div(n, (int64_t)STAGE_ROWS)};
      cuuint64_t strides3[2] = {(cuuint64_t)STAGE_ROWS * sizeof(float), (cuuint64_t)STAGE_ROWS * g.ncols * sizeof(float)};
      cuuint32_t box3[3] = {(cuuint32_t)BOX_ROWS, (cuuint32_t)cols, 1};
      cuuint32_t estr3[3] = {1, 1, 1};
      cr = enc(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<float*>(g.xbase), dims3, strides3, box3, estr3,
               CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    } else {
      const int64_t ld = which ? g.ldy : g.ldx;
      cuuint64_t dims[2] = {(cuuint64_t)n, (cuuint64_t)cols};      // joined: X's map also spans the t target columns behind it
      cuuint64_t strides[1] = {(cuuint64_t)ld * sizeof(float)};
      cuuint32_t box[2] = {(cuuint32_t)BOX_ROWS, (cuuint32_t)cols};
      cuuint32_t estr[2] = {1, 1};
      cr = enc(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(which ? g.ybase : g.xbase), dims, strides, box, estr,
               CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    }
  }
  if (cr != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled failed (%d)", (int)cr); return 1; }
  return 0;
}

int moments_wgmma_core(const Geometry& geo, const float* mask, int64_t n, int p, int t, double* M, cudaStream_t s) {
  // Y right behind X and N == p: one box per load carries both (half the TMA requests)
  const bool joined = (p % 16 == 0) && (geo.blocked ? geo.ycol == geo.xcol + p
                                                     : (geo.ybase == geo.xbase + (size_t)p * geo.ldx && geo.ldx == geo.ldy));
  CUtensorMap tx, ty;
  if (int rc = encode_maps(geo, n, p, t, joined, &tx, &ty)) return rc;
  GramArgs a;
  a.n = n; a.stages_total = ceil_div(n, (int64_t)STAGE_ROWS); a.p = p; a.t = t; a.xcol = geo.xcol; a.ycol = geo.ycol;
  a.blocked = geo.blocked ? 1 : 0; a.explicit_hi = (g_tc_mode.load() == 0) ? 1 : 0; a.joined = joined ? 1 : 0;
  const int NB = (p + 15) / 16, N = NB * 16, T = (t == 1) ? 1 : MAX_T;
  const int nslots = NB <= 2 ? Shape<1>::NWG : 1;            // partial slots the finalize sums (every slot it reads is written)
  int grid = sm_count();
  if (a.stages_total < grid) grid = (int)a.stages_total;
  const size_t n_part = (size_t)grid * PART_SLOTS * PART_ROWS * N, n_xs = (size_t)grid * SIDE_SLOTS * (T + 1) * XSIDE_COLS,
               n_ys = (size_t)grid * SIDE_SLOTS * YSIDE_STRIDE;
  double* partials = nullptr;
  if (dev_alloc((void**)&partials, (n_part + n_xs + n_ys) * sizeof(double), s)) return 1;
  double* xside = partials + n_part;
  double* yside = xside + n_xs;
  PDSB_CUDA_OK(cudaMemsetAsync(xside, 0, (n_xs + n_ys) * sizeof(double), s));     // not every slot has a writer
  int rc;
#define PDSB_GO(NBV) (t == 1 ? launch_one<NBV, 1>(tx, ty, mask, a, grid, partials, xside, yside, s) \
                             : launch_one<NBV, MAX_T>(tx, ty, mask, a, grid, partials, xside, yside, s))
  switch (NB) {
    case 1: rc = PDSB_GO(1); break;
    case 2: rc = PDSB_GO(2); break;
    case 3: rc = PDSB_GO(3); break;
    default: rc = PDSB_GO(4); break;
  }
#undef PDSB_GO
  if (!rc) {
    const int q1 = p + t + 1;
    gram_finalize_kernel<<<(q1 * q1 + 7) / 8, 256, 0, s>>>(partials, xside, yside, grid, nslots, N, T, p, t, n, mask ? 1 : 0, M);   // 8 warps = 8 elements per block
    cudaError_t e = cudaGetLastError();
    count_launch();
    if (e != cudaSuccess) { set_error("gram finalize launch failed: %s", cudaGetErrorString(e)); rc = 1; }
  }
  dev_free(partials, s);
  return rc;
}

}  // namespace

void set_tc_mode(int m) { g_tc_mode.store(m); }

// column-major matrices: X = p columns with leading dimension ldx, Y = t columns with ldy (anywhere in memory)
bool moments_wgmma_supported(const float* X, int64_t ldx, const float* Y, int64_t ldy, int64_t n, int p, int t) {
  if (n < 4096) return false;                 // latency-bound sizes stay on the SIMT kernel
  if (n >= (int64_t(1) << 31) - STAGE_ROWS) return false;   // the 2-D tensor maps are addressed with int32 row coordinates
  if (!get_encode_fn() || !shape_ok(p, t)) return false;
  if ((ldx % 4) != 0 || (ldy % 4) != 0) return false;       // global strides of a tensor map are multiples of 16 bytes
  return ((reinterpret_cast<uintptr_t>(X) | reinterpret_cast<uintptr_t>(Y)) & 15) == 0;
}

int moments_wgmma_f32(const float* X, int64_t ldx, const float* Y, int64_t ldy, const float* mask, int64_t n, int p,
                      int t, double* M, cudaStream_t s) {
  if (!moments_wgmma_supported(X, ldx, Y, ldy, n, p, t)) return -1;
  Geometry g{X, Y, ldx, ldy, 0, 0, 0, false};
  return moments_wgmma_core(g, mask, n, p, t, M, s);
}

// row-blocked frame: [block][column][FRAME_ROWS]; X = columns xcol .. xcol+p-1, Y = columns ycol .. ycol+t-1
bool moments_wgmma_frame_supported(int64_t n, int ncols, int xcol, int p, int ycol, int t) {
  if (!get_encode_fn()) return false;
  if (n < 4096 || !shape_ok(p, t)) return false;
  if (xcol < 0 || ycol < 0 || xcol + p > ncols || ycol + t > ncols) return false;
  return ceil_div(n, (int64_t)STAGE_ROWS) < (int64_t(1) << 31);     // int32 block coordinate of the 3-D tensor maps
}

int moments_wgmma_frame_f32(const float* frame, int64_t n, int ncols, int xcol, int p, int ycol, int t, const float* mask,
                            double* M, cudaStream_t s) {
  if (!moments_wgmma_frame_supported(n, ncols, xcol, p, ycol, t)) return -1;
  if (reinterpret_cast<uintptr_t>(frame) & 15) return -1;
  Geometry g{frame, frame, 0, 0, ncols, xcol, ycol, true};
  return moments_wgmma_core(g, mask, n, p, t, M, s);
}

}  // namespace pdsb
