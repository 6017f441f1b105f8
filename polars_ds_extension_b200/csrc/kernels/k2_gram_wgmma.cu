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
//        B  (SMEM, N x 8, K-major, 128B swizzle): every row of the TMA tile as it landed — the p feature rows (padded
//           to NF = 16 ceil(p / 16)), then the targets y_j, their TF32 remainders ylo_j and a row of ones
// The hi operand is the RAW data: the tensor core reads an fp32 operand as TF32 by ignoring the low 13 mantissa bits
// (tests/test_gpu_moments.py compares against exact-product f64-accumulated moments, and variant 0 — hi rows that clear
// those bits themselves — against the raw variant bit for bit), so B needs no conversion and the hi rows of A are a copy.
//
// x . y_j and sum x come out of the same MMAs as extra columns of D:
//        X'y_j = D[hi, y_j] + D[lo, y_j] + D[hi, ylo_j] + D[lo, ylo_j],      sum x = D[hi, 1] + D[lo, 1]
// (the same 3-term TF32 split as X'X, ~2^-22 relative).  The consumer thread that writes ylo_j of a stage row also adds
// sum y_j, sum y_j^2, y_j . y_k and the masked row count of that row into f64 registers.
//
// A-row layout.  An m64 block of A holds 32 features: warp q of the warpgroup has feature 8q + g (g = lane / 4) as hi in
// its fragment row g and as lo in row g + 8, so one shared-memory load gives a thread both of its A registers for that
// k (the row order of A only permutes the rows of D).  Up to 32 features (NB <= 2) one m64 wgmma carries everything and
// three consumer warpgroups take every third stage each.  From 33 to 64 features warpgroup 0 holds features 0..31 and
// warpgroup 1 features 32..63, and both work on every stage.
//
// Data flow per CTA (persistent, one CTA per SM, 128-row stages dealt round-robin):
//   warps 0 .. 4W-1    W consumer warpgroups (W = 3 up to 32 features, else 2): per stage, ylo rows + target sums, then
//                      tile -> registers (hi / lo) -> 16 x wgmma (K = 8), fp32 accumulators in registers, added to f64
//                      registers after every stage
//   warp 4W            TMA producer: cp.async.bulk.tensor, per 32-row box one {32 x p} load of X and one {32 x t} of Y
//                      (a whole warpgroup that hands registers to the consumers with setmaxnreg where they need more)
// A second tiny kernel sums the per-CTA partials in a fixed order (bit-reproducible) and applies the symmetrisation.
// Roofline: HBM-bound, algorithmic bytes = 4 (p + t) per row (+4 with a mask).
#include "../common.h"
#include "kernels.h"
#include "mbarrier.h"
#include <cuda.h>

namespace pdsb {

namespace {

constexpr int BOX_ROWS = 32;            // K extent of one TMA box = 128 bytes of f32 = one swizzle row
constexpr int BPS = 4;                  // boxes per pipeline stage  (stage = 128 rows)
constexpr int STAGE_ROWS = BOX_ROWS * BPS;
constexpr int MAX_RING = 15;            // TMA landing ring (stages)
constexpr int PART_SLOTS = 3;           // partial slots per CTA: one per consumer warpgroup (at most three)
constexpr int PART_ROWS = 128;          // partial rows per (CTA, slot): hi of feature c at row c, lo at row 64 + c
constexpr int MAX_T = 4;
constexpr uint32_t HI_MASK = 0xFFFFE000u;   // TF32 keeps 10 mantissa bits
constexpr int YSIDE_SLOTS = 4 * PART_SLOTS; // target-sum slots per CTA: one per consumer warp
constexpr int YSIDE_STRIDE = 16;        // doubles per (CTA, warp): [j] sum y_j, [4 + j] sum y_j^2, [8 + pair] y_j.y_k, [14] count

// Tile rows of one box, from the top: the feature rows (p of them, padded to NF = 16 NB), then the target block that
// the MMA's N also covers:  t = 1:  NF y_0, NF + 1 ylo_0, NF + 2 the constant 1, 5 zero rows (one 8-row group);
//                           t = 2..4:  NF + j y_j, NF + 4 + j ylo_j (j < 4), NF + 8 the constant 1, 7 zero rows (two).
// ylo_j = y_j - trunc_tf32(y_j) is written by the consumers on every stage; the 1 row once at kernel start.
template <int NB, int T>
struct Shape {
  static constexpr int NF = NB * 16;                                 // feature rows of the tile, padded to 16
  static constexpr int YLO = NF + (T == 1 ? 1 : 4);                  // first ylo row
  static constexpr int ONE = NF + (T == 1 ? 2 : 8);                  // the row of ones
  static constexpr int N = NF + (T == 1 ? 8 : 16);                   // MMA N = every row of the tile
  static constexpr int MB = NB <= 2 ? 1 : 2;                         // m64 blocks of the A operand (hi and lo stacked)
  static constexpr int TILE_ROWS = N;
  static constexpr uint32_t TILE_BYTES = TILE_ROWS * 128;            // one box-tile (a multiple of 1024 bytes)
  // consumer warpgroups: three taking every third stage up to 32 features (13 warps = 416 threads: four warps on a
  // scheduler cap a thread at 128 registers); two (features 0..31 / 32..63) on every stage above (9 warps, 168)
  static constexpr int NWG = NB <= 2 ? 3 : 2;
  // Above those caps (2..4 targets: 15 f64 target sums per thread and a 16-column target block; 64 features with one
  // target) the producer is a whole warpgroup that gives registers back with setmaxnreg, and the consumers take them.
  static constexpr bool MOVE_REGS = T > 1 || NB == 4;
  static constexpr int PRODUCER_REGS = NWG == 3 ? 24 : 40;
  static constexpr int CONSUMER_REGS = NWG == 3 ? 160 : 232;
  static_assert(128 * (NWG * CONSUMER_REGS + PRODUCER_REGS) <= 65536, "register file of an SM exceeded");
  static constexpr int NUM_THREADS = (4 * NWG + (MOVE_REGS ? 4 : 1)) * 32;
  // ring depth: as many stages as fit in ~200 KB of the 227 KB a block may use (bytes in flight per SM are what keeps
  // HBM busy), a multiple of three up to 32 features.  The 32-feature, 2..4-target tile (24 KB a stage) takes 9 = 216 KB
  // rather than 6.
  static constexpr int RING = T == 1 ? (NB == 1 ? 15 : NB == 2 ? 9 : NB == 3 ? 7 : 5)
                                     : (NB == 1 ? 12 : NB == 2 ? 9 : NB == 3 ? 6 : 5);
  static constexpr size_t SMEM = (size_t)RING * BPS * TILE_BYTES;
  // consumer arrivals that free a ring slot: one per consumer warp that reads the stage
  static constexpr int CONSUMER_WARPS = MB == 2 ? 4 * NWG : 4;
  // a warpgroup waits on a slot's parity only if it also consumed the slot's previous phase
  static_assert(MB == 2 || RING % NWG == 0, "every ring slot must go to the same warpgroup");
  static_assert(RING <= MAX_RING, "ring deeper than the barrier array");
  static_assert(SMEM + 1024 + 2 * MAX_RING * 8 <= 227 * 1024, "ring exceeds the shared memory of a block");
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
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

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

// D (m64 x N, f32, registers) (+)= A (m64 x k8, tf32, registers) * B (N x k8, tf32, shared memory)^T.  One macro writes
// the wrapper for every N the kernel uses (N = 24 .. 80 in steps of 8; N / 2 accumulators per thread).  Operands
// %0 .. %(N/2 - 1) are the accumulators, then the four A registers, the B descriptor and the accumulate flag.
#define PDSB_D12 "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11"
#define PDSB_D16 PDSB_D12 ", %12, %13, %14, %15"
#define PDSB_D20 PDSB_D16 ", %16, %17, %18, %19"
#define PDSB_D24 PDSB_D20 ", %20, %21, %22, %23"
#define PDSB_D28 PDSB_D24 ", %24, %25, %26, %27"
#define PDSB_D32 PDSB_D28 ", %28, %29, %30, %31"
#define PDSB_D36 PDSB_D32 ", %32, %33, %34, %35"
#define PDSB_D40 PDSB_D36 ", %36, %37, %38, %39"
#define PDSB_F4(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3])
#define PDSB_F12 PDSB_F4(0), PDSB_F4(4), PDSB_F4(8)
#define PDSB_F16 PDSB_F12, PDSB_F4(12)
#define PDSB_F20 PDSB_F16, PDSB_F4(16)
#define PDSB_F24 PDSB_F20, PDSB_F4(20)
#define PDSB_F28 PDSB_F24, PDSB_F4(24)
#define PDSB_F32 PDSB_F28, PDSB_F4(28)
#define PDSB_F36 PDSB_F32, PDSB_F4(32)
#define PDSB_F40 PDSB_F36, PDSB_F4(36)
// NV = N, K = N / 2 (first operand after the accumulators), K1 .. K5 = K + 1 .. K + 5
#define PDSB_WGMMA(NV, K, K1, K2, K3, K4, K5)                                                                          \
  template <> struct Wgmma<NV> {                                                                                      \
    static __device__ __forceinline__ void mma(float* d, const uint32_t* a, uint64_t b_desc, uint32_t accumulate) {   \
      asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %" #K5 ", 0;\n\t"                                            \
                   "wgmma.mma_async.sync.aligned.m64n" #NV "k8.f32.tf32.tf32 {" PDSB_D##K "}, "                       \
                   "{%" #K ", %" #K1 ", %" #K2 ", %" #K3 "}, %" #K4 ", p, 1, 1;\n\t}"                                 \
                   : PDSB_F##K                                                                                         \
                   : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc), "r"(accumulate));                     \
    }                                                                                                                  \
  };
template <int N> struct Wgmma;
PDSB_WGMMA(24, 12, 13, 14, 15, 16, 17)
PDSB_WGMMA(32, 16, 17, 18, 19, 20, 21)
PDSB_WGMMA(40, 20, 21, 22, 23, 24, 25)
PDSB_WGMMA(48, 24, 25, 26, 27, 28, 29)
PDSB_WGMMA(56, 28, 29, 30, 31, 32, 33)
PDSB_WGMMA(64, 32, 33, 34, 35, 36, 37)
PDSB_WGMMA(72, 36, 37, 38, 39, 40, 41)
PDSB_WGMMA(80, 40, 41, 42, 43, 44, 45)
#undef PDSB_WGMMA

struct alignas(8) Barriers {
  uint64_t raw_full[MAX_RING], raw_empty[MAX_RING];   // TMA landed / tile free again (every consumer warp done)
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

// T = target rows the tile is laid out for (1, or 4 for t = 2..4)
template <int NB, int T>
__global__ void __launch_bounds__(Shape<NB, T>::NUM_THREADS, 1)
gram_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_x, const __grid_constant__ CUtensorMap tmap_y,
                  const float* __restrict__ mask, const GramArgs g, double* __restrict__ partials /* [grid][PART_SLOTS][128][N] */,
                  double* __restrict__ yside /* [grid][YSIDE_SLOTS][YSIDE_STRIDE] */) {
  using S = Shape<NB, T>;
  constexpr int NF = S::NF, N = S::N, MB = S::MB, RING = S::RING, NACC = N / 2;
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
    for (int i = 0; i < RING; ++i) { mbar_init(&bars->raw_full[i], 1); mbar_init(&bars->raw_empty[i], S::CONSUMER_WARPS); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  // rows the TMA never writes: the row of ones gets 1.0f; the rest (feature rows p .. NF-1, target rows t .. , the
  // ylo rows before their first write, the padding rows) is zeroed once, so that nothing uninitialised is multiplied
  for (int i = threadIdx.x; i < RING * BPS * S::TILE_ROWS * 8; i += NUM_THREADS) {
    const int tile = i / (S::TILE_ROWS * 8), r = (i / 8) % S::TILE_ROWS, c = i % 8;
    if (r < p || (r >= NF && r < NF + t)) continue;
    const uint32_t v = r == S::ONE ? __float_as_uint(1.0f) : 0u;
    *reinterpret_cast<uint4*>(raw + (size_t)tile * TILE_BYTES + (size_t)r * 128 + c * 16) = make_uint4(v, v, v, v);
  }
  fence_async_smem();
  __syncthreads();

  if (warp < 4 * NWG) {
    // =============================== consumer warpgroups: tile -> hi / lo registers -> wgmma ===============
    if constexpr (S::MOVE_REGS) asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(S::CONSUMER_REGS));
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

    // ---- the target rows of a stage: one stage row per thread.  Up to 32 features the warpgroup that consumes the
    // stage takes all 128 rows; above, warpgroup w takes rows 64 w .. 64 w + 63 (its warps 0 and 1).  The thread writes
    // ylo_j of its row for the MMAs and adds sum y_j, sum y_j^2, y_j . y_k and the masked count straight into f64.
    const int yrow = MB == 2 ? 64 * wg + (threadIdx.x & 127) : (threadIdx.x & 127);
    const bool yact = MB == 1 || (threadIdx.x & 127) < 64;
    const uint32_t ybox = (uint32_t)(yrow >> 5) * TILE_BYTES, ych = (uint32_t)((yrow & 31) >> 2), yel = (uint32_t)(yrow & 3) * 4;
    constexpr int NPAIR = T * (T - 1) / 2;
    double dsy[T], dsyy[T], dyy[NPAIR > 0 ? NPAIR : 1], dcnt = 0.0;
#pragma unroll
    for (int j = 0; j < T; ++j) { dsy[j] = 0.0; dsyy[j] = 0.0; }
#pragma unroll
    for (int k = 0; k < NPAIR; ++k) dyy[k] = 0.0;
    // Called after the stage's full barrier and before any MMA of it.  The write after read against the MMAs of the
    // slot's previous phase is ordered: those MMAs completed before their warpgroup's wg_wait<0>, which precedes its
    // arrival on raw_empty; the producer refills the slot only after every arrival, and this thread waited on the refill.
    // fence.proxy.async makes the generic-proxy stores visible to the tensor core's async-proxy reads, and the named
    // barrier holds every MMA of the stage until all of its rows are written.
    auto prep_targets = [&](uint32_t it) {
      if (yact) {
        unsigned char* st = raw + (size_t)(it % RING) * BPS * TILE_BYTES + ybox;
        float y[T];
#pragma unroll
        for (int j = 0; j < T; ++j) {
          const uint32_t v = *reinterpret_cast<const uint32_t*>(st + (NF + j) * 128 + ((ych ^ ((NF + j) & 7)) << 4) + yel);
          uint32_t lo;
          asm("sub.rn.f32 %0, %1, %2;" : "=r"(lo) : "r"(v), "r"(v & HI_MASK));
          *reinterpret_cast<uint32_t*>(st + (S::YLO + j) * 128 + ((ych ^ ((S::YLO + j) & 7)) << 4) + yel) = lo;
          y[j] = __uint_as_float(v);
        }
        int k = 0;
#pragma unroll
        for (int j = 0; j < T; ++j) {
          const double yj = (double)y[j];
          dsy[j] += yj;
          dsyy[j] = fma(yj, yj, dsyy[j]);
#pragma unroll
          for (int l = j + 1; l < T; ++l, ++k) dyy[k] = fma(yj, (double)y[l], dyy[k]);
        }
        if (mask != nullptr) {
          // row count of a masked frame: the packer zeroes masked rows, so only the count needs the mask
          const int64_t r = stage_row0(it) + yrow;
          if (r < g.n) dcnt += (double)__ldg(mask + r);
        }
      }
      fence_async_smem();
      if (MB == 2) named_bar_sync(1, 256);
      else named_bar_sync(1 + wg, 128);
    };

    // A registers double-buffered over the boxes: the loads of box b + 1 run while the MMAs of box b execute, and box 0
    // of this warpgroup's next stage loads while the last box of this stage executes, before the drain
    uint32_t a[2][BOX_ROWS / 8][4];
    if (first < my_stages) {
      mbar_wait(&bars->raw_full[first % RING], (first / RING) & 1);
      prep_targets(first);
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
          prep_targets(nxt);                                   // another slot than the one the MMAs in flight read
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
    // target sums: a fixed-order tree over the warp, one slot per warp (every consumer warp writes its slot)
#pragma unroll
    for (int off = 16; off; off >>= 1) {
#pragma unroll
      for (int j = 0; j < T; ++j) {
        dsy[j] += __shfl_xor_sync(0xffffffffu, dsy[j], off);
        dsyy[j] += __shfl_xor_sync(0xffffffffu, dsyy[j], off);
      }
#pragma unroll
      for (int k = 0; k < NPAIR; ++k) dyy[k] += __shfl_xor_sync(0xffffffffu, dyy[k], off);
      dcnt += __shfl_xor_sync(0xffffffffu, dcnt, off);
    }
    if (lane == 0) {
      double* ys = yside + ((size_t)blockIdx.x * YSIDE_SLOTS + warp) * YSIDE_STRIDE;
#pragma unroll
      for (int j = 0; j < T; ++j) { ys[j] = dsy[j]; ys[4 + j] = dsyy[j]; }
#pragma unroll
      for (int k = 0; k < NPAIR; ++k) ys[8 + k] = dyy[k];
      ys[14] = dcnt;
    }
  } else {
    // =============================== TMA producer (warp-uniform loop, one elected lane issues) ===============
    if constexpr (S::MOVE_REGS) {
      asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(S::PRODUCER_REGS));
      if (warp != 4 * NWG) return;                             // one warp of the producer warpgroup issues
    }
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
            if (!g.joined) tma_load_3d(dst + NF * 128, &tmap_y, &bars->raw_full[rs], b * BOX_ROWS, g.ycol, (int)(row0 / STAGE_ROWS));
          } else {
            tma_load_2d(dst, &tmap_x, &bars->raw_full[rs], (int)(row0 + b * BOX_ROWS), 0);
            if (!g.joined) tma_load_2d(dst + NF * 128, &tmap_y, &bars->raw_full[rs], (int)(row0 + b * BOX_ROWS), 0);
          }
        }
      }
      __syncwarp();
      if (++rs == RING) { rs = 0; ph ^= 1; }
    }
  }
}

// Sum the per-CTA partials in a fixed order (bit-reproducible) and lay the moments out in the order [X | Y | 1].  Partial
// row c / 64 + c is the hi / lo of feature c; columns 0 .. p-1 are the features, yc + k target k, ylc + k its ylo and
// onec the row of ones:
//   X'X[a][b] = HH[a][b] + LH[a][b] + LH[b][a]        (symmetrised: 0.5 (HH[a][b] + HH[b][a]))
//   X'y_k[a]  = D[hi_a, y_k] + D[lo_a, y_k] + D[hi_a, ylo_k] + D[lo_a, ylo_k]
//   sum x_a   = D[hi_a, 1] + D[lo_a, 1]
// The target block comes from the per-warp target sums.  One WARP per element of the upper triangle (mirrored ->
// exactly symmetric): lane l sums parts l, l + 32, ..., then a fixed-order xor tree.
__global__ void __launch_bounds__(256)
gram_finalize_kernel(const double* __restrict__ partials, const double* __restrict__ yside, int nparts, int nslots,
                     int nyslots, int N, int yc, int ylc, int onec, int p, int t, int64_t n, int masked,
                     double* __restrict__ M) {
  const int q1 = p + t + 1;
  const int lane = threadIdx.x & 31;
  const int idx = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (idx >= q1 * q1) return;
  const int i = idx / q1, j = idx % q1;
  if (i > j) return;
  double r = 0.0;
  if (i < p) {
    double s0 = 0.0, s1 = 0.0, s2 = 0.0, s3 = 0.0;
    if (j < p) {                                   // X'X
      for (int k = lane; k < nparts * nslots; k += 32) {
        const double* P = partials + ((size_t)(k % nparts) * PART_SLOTS + k / nparts) * PART_ROWS * N;
        s0 += P[(size_t)i * N + j];
        s1 += P[(size_t)j * N + i];
        s2 += P[(size_t)(64 + i) * N + j];
        s3 += P[(size_t)(64 + j) * N + i];
      }
      r = 0.5 * (s0 + s1) + (s2 + s3);             // per lane; the lanes are added below
    } else if (j < p + t) {                        // X'y_k
      const int cy = yc + (j - p), cl = ylc + (j - p);
      for (int k = lane; k < nparts * nslots; k += 32) {
        const double* P = partials + ((size_t)(k % nparts) * PART_SLOTS + k / nparts) * PART_ROWS * N;
        s0 += P[(size_t)i * N + cy];
        s1 += P[(size_t)(64 + i) * N + cy];
        s2 += P[(size_t)i * N + cl];
        s3 += P[(size_t)(64 + i) * N + cl];
      }
      r = (s0 + s1) + (s2 + s3);
    } else {                                       // sum x
      for (int k = lane; k < nparts * nslots; k += 32) {
        const double* P = partials + ((size_t)(k % nparts) * PART_SLOTS + k / nparts) * PART_ROWS * N;
        s0 += P[(size_t)i * N + onec];
        s1 += P[(size_t)(64 + i) * N + onec];
      }
      r = s0 + s1;
    }
  } else {
    // target / ones block: [a] sum y_a, [4 + a] sum y_a^2, [8 + pair(a, b)] y_a . y_b, [14] count
    const int a = i - p, bb = j - p;
    int off;
    if (j == p + t) off = (i == p + t) ? 14 : a;
    else off = (a == bb) ? 4 + a : 8 + a * (7 - a) / 2 + (bb - a - 1);
    if (!(j == p + t && i == p + t && !masked))
      for (int k = lane; k < nparts * nyslots; k += 32)
        r += yside[((size_t)(k % nparts) * YSIDE_SLOTS + k / nparts) * YSIDE_STRIDE + off];
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
               double* partials, double* yside, double* M, cudaStream_t s) {
  using S = Shape<NB, T>;
  const size_t smem = S::SMEM + 1024 /* alignment slack */ + sizeof(Barriers);
  auto k = gram_wgmma_kernel<NB, T>;
  PDSB_CUDA_OK(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  k<<<grid, S::NUM_THREADS, smem, s>>>(tx, ty, mask, g, partials, yside);
  PDSB_LAUNCH_OK();
  count_launch();
  const int q1 = g.p + g.t + 1;
  // 8 warps = 8 elements per block; partial slots: one per warpgroup up to 32 features, one shared above
  gram_finalize_kernel<<<(q1 * q1 + 7) / 8, 256, 0, s>>>(partials, yside, grid, S::MB == 2 ? 1 : S::NWG, 4 * S::NWG,
                                                         S::N, S::NF, S::YLO, S::ONE, g.p, g.t, g.n, mask ? 1 : 0, M);
  cudaError_t e = cudaGetLastError();
  count_launch();
  if (e != cudaSuccess) { set_error("gram finalize launch failed: %s", cudaGetErrorString(e)); return 1; }
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
  // Y right behind X and NF == p: one box per load carries both (half the TMA requests)
  const bool joined = (p % 16 == 0) && (geo.blocked ? geo.ycol == geo.xcol + p
                                                     : (geo.ybase == geo.xbase + (size_t)p * geo.ldx && geo.ldx == geo.ldy));
  CUtensorMap tx, ty;
  if (int rc = encode_maps(geo, n, p, t, joined, &tx, &ty)) return rc;
  GramArgs a;
  a.n = n; a.stages_total = ceil_div(n, (int64_t)STAGE_ROWS); a.p = p; a.t = t; a.xcol = geo.xcol; a.ycol = geo.ycol;
  a.blocked = geo.blocked ? 1 : 0; a.explicit_hi = (g_tc_mode.load() == 0) ? 1 : 0; a.joined = joined ? 1 : 0;
  const int NB = (p + 15) / 16, N = NB * 16 + (t == 1 ? 8 : 16);
  int grid = sm_count();
  if (a.stages_total < grid) grid = (int)a.stages_total;
  // every slot the finalize reads has a writer: each CTA has at least one stage, and every consumer warp writes its
  // partial rows and its target-sum slot
  const size_t n_part = (size_t)grid * PART_SLOTS * PART_ROWS * N, n_ys = (size_t)grid * YSIDE_SLOTS * YSIDE_STRIDE;
  double* partials = nullptr;
  if (dev_alloc((void**)&partials, (n_part + n_ys) * sizeof(double), s)) return 1;
  double* yside = partials + n_part;
  int rc;
#define PDSB_GO(NBV) (t == 1 ? launch_one<NBV, 1>(tx, ty, mask, a, grid, partials, yside, M, s) \
                             : launch_one<NBV, MAX_T>(tx, ty, mask, a, grid, partials, yside, M, s))
  switch (NB) {
    case 1: rc = PDSB_GO(1); break;
    case 2: rc = PDSB_GO(2); break;
    case 3: rc = PDSB_GO(3); break;
    default: rc = PDSB_GO(4); break;
  }
#undef PDSB_GO
  dev_free(partials, s);
  return rc;
}

}  // namespace

void set_tc_mode(int m) { g_tc_mode.store(m); }

// column-major matrices (bstride == 0): X = p columns with leading dimension ldx, Y = t columns with ldy (anywhere in
// memory).  Row-blocked frame [block][column][FRAME_ROWS] (bstride = ncols * FRAME_ROWS): X and Y point at columns of
// one frame, which must start on a 16-byte boundary.
bool moments_wgmma_supported(const float* X, int64_t ldx, const float* Y, int64_t ldy, int64_t n, int p, int t,
                             int64_t bstride) {
  if (n < 4096) return false;                 // latency-bound sizes stay on the SIMT kernel
  if (!get_encode_fn() || !shape_ok(p, t)) return false;
  if (bstride)                                // int32 block coordinate of the 3-D tensor maps
    return ceil_div(n, (int64_t)STAGE_ROWS) < (int64_t(1) << 31) && (reinterpret_cast<uintptr_t>(std::min(X, Y)) & 15) == 0;
  if (n >= (int64_t(1) << 31) - STAGE_ROWS) return false;   // the 2-D tensor maps are addressed with int32 row coordinates
  if ((ldx % 4) != 0 || (ldy % 4) != 0) return false;       // global strides of a tensor map are multiples of 16 bytes
  return ((reinterpret_cast<uintptr_t>(X) | reinterpret_cast<uintptr_t>(Y)) & 15) == 0;
}

int moments_wgmma_f32(const float* X, int64_t ldx, const float* Y, int64_t ldy, const float* mask, int64_t n, int p,
                      int t, double* M, cudaStream_t s, int64_t bstride) {
  Geometry g{X, Y, ldx, ldy, 0, 0, 0, false};
  if (bstride) {   // the maps start at the first of the two column ranges; xcol / ycol count frame columns from there
    const float* base = std::min(X, Y);
    g = Geometry{base, base, 0, 0, (int)(bstride / FRAME_ROWS), (int)((X - base) / FRAME_ROWS),
                 (int)((Y - base) / FRAME_ROWS), true};
  }
  return moments_wgmma_core(g, mask, n, p, t, M, s);
}

}  // namespace pdsb
