// K6 / K7 — rolling_lin_reg and recursive_lin_reg without the sequential Woodbury chain.
//
// Reference: faer_rolling_lr / faer_rolling_skipping_lr / faer_recursive_lr + woodbury_step
// (src/linear/online_lr/lr_online_solvers.rs:148-332) and the output loops of pl_rolling_lr /
// pl_recursive_lr (src/num_ext/linear_regression.rs:1121-1283).  The reference walks the rows strictly one after
// another (2 rank-1 updates per row, ~6 small heap allocations per row, single thread).  What its tests pin is the
// mathematical definition — rolling == per-window OLS/ridge, recursive == prefix OLS/ridge
// (tests/test_linear_exprs.py:123-166, 718-854) — and that is what this kernel evaluates directly and in parallel:
//
//   row vector          e = (z_0..z_{D-1}, y, 1)  with z = (x_0..x_{p-1}[,1]);  all zero for a non-finite row
//                       (OnlineLR::update skips non-finite rows, lr_online_solvers.rs:85-89)
//   moments of a row    m = [ e_i e_j (i<=j<D), e_i y, 1*1 ]          NM = D(D+1)/2 + D + 1 numbers
//   pass A  chain sums  S_k = sum of m over chain k (1024 rows), f64
//   pass B  chain scan  C_k = sum_{j<k} S_j  (exclusive, f64)
//   pass C  per row     W_t = C_k + E(t) - [C_k' + H + L(t-w)]   (f64: the global-prefix difference loses
//                       ~1e-16 * (n/w) relative, harmless), then G = W_GG + lambda I, solved by an in-register
//                       Cholesky in the data dtype, pred_t = x_t . beta_t.
// Rolling = both sides, recursive = entering side only (w = infinity).  Every chain is independent after pass B.
//
// Work decomposition (passes A and C): ONE WARP PER CHAIN, and inside the warp two alternating roles per 32-row batch
//   * lane-per-row:       coalesced loads of the batch's entering (and leaving) rows, e-vectors written to shared
//                         memory as doubles; later the Cholesky solve of "its" row from the staged Gram, and the stores;
//   * lane-per-component: each lane owns <= 3 of the NM running moments in f64 registers and walks the 32 rows
//                         (one LDS.64 + one LDS.128 feed two DFMAs per row and side), dropping W_t (cast to the data
//                         dtype) into shared memory for the row's solver lane.
// Pass A has no per-row output and stays thread-per-row (NM register accumulators, one shuffle reduction per chain).
// This keeps the running state at 2-3 doubles per lane (the thread-per-row-chain version of this kernel carried all
// NM in registers: 254 registers, 8 warps per SM, low issue utilisation) and needs no
// intra-tile scan at all.
// Bytes per row (algorithmic): (p+1) s read, (p+bias) s + s + 1 written.
//
// Pass C has three kernels, chosen for each call by online_plan (which also says whether and in which precision passes
// A and B run) and launched by the one driver run_online:
//   packed           online_main_f32x2_kernel   f32 row pairs, up to 9 coefficients
//   lane-per-moment  online_main_kernel         the lane-per-row / lane-per-component kernel above, up to 12
//   generic          online_generic_kernel      up to 129 coefficients, moments in shared memory
// The rules every kernel shares are stated once: row_valid (which rows get a fit), rolling_head (the rows of the first
// window before the chain), component_pair (moment component -> pair of row entries) and row_finite (the row probe).
//
// Groups (recursive_lin_reg(...).over(key) and rolling over groups, grouped_online_lin_reg): every group is cut into
// chains from its own first row, so chain j of group g holds the rows a call on the group alone gives its chain j.
// Passes A and C take the group's rows, length and skip flag from the chain table (chain_pos) and keep row indices
// group-local; pass B scans each group's chains alone (group_scan_kernel).  A rolling head reads the prefix of its
// group's chain kl, at the global chain k - cp.k + kl.  Every value is then formed as in that call, and a group's outputs
// are its call's, bit for bit.  A rolling plan depends on skip (online_plan), so a call whose groups fall in both skip
// classes may run two plans, each over its own class (ChainTab::cls).  The single column is the one-group case of the
// same kernels: their ONE instantiations read no table.
#include "../common.h"
#include "../host/host.h"
#include "kernels.h"
#include "f32x2.h"
#include "segment_groups.h"
#include <cub/cub.cuh>
#include <type_traits>

namespace pdsb {

static thread_local int t_last_online_path = 0;   // 1 packed f32, 2 lane-per-moment, 3 generic (pdsb_last_online_path)
int last_online_path() { return t_last_online_path; }

namespace {

constexpr int WARPS = 5;                 // independent chains per CTA (no block-level synchronisation anywhere);
                                         // 3 CTAs x 5 warps fit the 8-feature + bias f32 case in shared memory and registers
constexpr int CTA_THREADS = WARPS * 32;
constexpr int BATCH = 32;                // rows per role switch
constexpr int CHAIN_ROWS = 1024;         // rows per warp = granularity of the prefix arrays

// A lane-per-component "task" (a, b) accumulates e_a*e_b and e_a*e_{b+1} (b even): one LDS.64 + one LDS.128 feed two
// DFMAs.  Row a of the upper triangle needs b = a&~1, .., <= D (the y column is entry D); one more task holds 1*1.
template <int D> constexpr int n_tasks() {
  int t = 0;
  for (int a = 0; a < D; ++a) for (int b = a & ~1; b <= D; b += 2) ++t;
  return t + 1;
}
constexpr int even_odd_half(int x) { int e = (x + 1) & ~1; return ((e / 2) & 1) ? e : e + 2; }   // even, half of it odd

template <int D> struct MomN {
  static constexpr int NG = D * (D + 1) / 2;
  static constexpr int NM = NG + D + 1;
  static constexpr int ES = even_odd_half(((D + 1) | 1) + 1);   // 16-byte pairs; <= 2-way conflicts when staging
  static constexpr int GS = (NM + 1) | 1;                  // odd stride; slot NM is the dump slot of unused products
  static constexpr int NT = n_tasks<D>();
  static constexpr int TPL = (NT + 31) / 32;               // tasks per lane
};

template <typename T, int D>
constexpr size_t warp_smem_bytes() {
  return (size_t)(2 * BATCH * MomN<D>::ES + BATCH) * sizeof(double) + (size_t)BATCH * MomN<D>::GS * sizeof(T);
}

// packed slot of the unordered pair (i <= j) in the solver's Gram order, or the dump slot
template <int D>
__device__ __forceinline__ int pair_slot(int i, int j) {
  constexpr int NG = MomN<D>::NG, NM = MomN<D>::NM;
  if (i > j || i >= D) return (i == D + 1 && j == D + 1) ? NM - 1 : NM;
  if (j < D) return i * D - i * (i - 1) / 2 + (j - i);
  if (j == D) return NG + i;
  return NM;
}

// moment component c -> the pair (i <= j) over (z_0..z_{d-1}, y, 1) whose product it sums (the inverse of pair_slot).
// Here and in row_valid the compared values come in by reference: by value, the compiler swaps the operands of their
// comparisons, and the chain scan and the packed kernel compile to different SASS.
__device__ __forceinline__ void component_pair(const int& component, int d, int& i_out, int& j_out) {
  const int ng = d * (d + 1) / 2;
  int c = component, i, j;
  if (c >= ng + d) { i = j = d + 1; }
  else if (c >= ng) { i = c - ng; j = d; }
  else { i = 0; while (c >= d - i) { c -= d - i; ++i; } j = i + c; }
  i_out = i; j_out = j;
}

// Whether row r gets a fit.  Rolling: its window is complete and, when null rows are skipped, holds at least min_rows
// finite rows.  Recursive: when skipping, row r is finite and at least min_rows finite rows lead up to it; otherwise
// r + row0 >= min_rows - 1.  `cnt` is the finite-row count of the window in the type the kernel holds it in.
// The lane-per-moment and packed kernels pass r as an expression (rb + lane, rb + 2 * lane), not as their local `r`:
// binding that local to the reference takes its address, which keeps it in memory until this function is inlined, and
// the compiler then folds the kernel's other comparisons on `r` differently (both kernels' SASS changes).  The generic
// kernel's `r` is its loop index; it is passed as it is, since that kernel is not tuned to the instruction.
template <typename Cnt>
__device__ __forceinline__ bool row_valid(bool rolling, const int64_t& r, bool fin, const Cnt& cnt, int64_t window,
                                          int64_t min_rows, int skip, int64_t row0) {
  if (rolling) return (r >= window - 1) && (!skip | (cnt >= (Cnt)min_rows - Cnt(0.5)));
  return skip ? (fin && cnt >= (Cnt)min_rows - Cnt(0.5)) : (r + row0 >= min_rows - 1);
}

// rows [lo, chain0) are inside the window of the chain's first row; kl is the chain that holds lo, so that the prefix
// up to lo is C[kl] plus the rows [kl * CHAIN_ROWS, lo)
__device__ __forceinline__ void rolling_head(int64_t chain0, int64_t window, int64_t& lo, int64_t& kl) {
  lo = max((int64_t)0, chain0 - window);
  kl = lo / CHAIN_ROWS;
}

// true when the row exists (inr) and y and every z_c are finite: y * 0 + sum z_c * 0 is 0 then, NaN otherwise
template <typename T, int D>
__device__ __forceinline__ bool row_finite(bool inr, const T* z, T yv) {
  T acc = yv * T(0);
#pragma unroll
  for (int c = 0; c < D; ++c) acc = fma(z[c], T(0), acc);
  return inr && (acc == T(0));
}

// The chain table of a grouped call: group g is rows [off[g], off[g + 1]) and chains [cbase[g], cbase[g + 1]).
struct ChainTab {
  const int64_t* off;     // [n_groups + 1] the group's first row
  const int64_t* cbase;   // [n_groups + 1] the group's first chain
  const int64_t* cgrp;    // [nchains] the chain's group
  const uint8_t* skip;    // [n_groups] the group's skip flag; nullptr: no group skips
  int cls;                // the skip class (0 or 1) whose groups this launch fits; -1: every group
};
// chain k of the call: its index inside its group, the group's first row, its rows and its skip flag.  ONE: the single
// column, the kernel's own n and skip.
struct ChainPos { int64_t k, r0, n; int skip; };
template <bool ONE>
__device__ __forceinline__ ChainPos chain_pos(const ChainTab& t, int64_t k, int64_t n, int skip) {
  if (ONE) return {k, 0, n, skip};
  const int64_t g = __ldg(t.cgrp + k), r0 = __ldg(t.off + g);
  return {k - __ldg(t.cbase + g), r0, __ldg(t.off + g + 1) - r0, t.skip ? (int)__ldg(t.skip + g) : 0};
}
// a grouped launch that serves one skip class leaves the other class's chains alone: it neither reads nor writes them.
// Any nonzero skip byte is the skip class (1), as it is to row_valid and group_class_counts.
template <bool ONE>
__device__ __forceinline__ bool other_class(const ChainTab& t, int skip) {
  return !ONE && t.cls >= 0 && (skip != 0 ? 1 : 0) != t.cls;
}

// task t -> offsets (in doubles) of e_a, e_b inside a staged row and the Gram slots of its two products
template <int D>
__device__ __forceinline__ void task_of(int t, int& a, int& b, int& k0, int& k1) {
  constexpr int NT = MomN<D>::NT;
  a = D + 1; b = (D + 1) & ~1;
  if (t < NT - 1) {
    int cur = 0;
    for (int aa = 0; aa < D; ++aa)
      for (int bb = aa & ~1; bb <= D; bb += 2) { if (cur == t) { a = aa; b = bb; } ++cur; }
  }
  if (t >= NT) { k0 = k1 = MomN<D>::NM; return; }
  k0 = pair_slot<D>(a, b);
  k1 = pair_slot<D>(a, b + 1);
}

// lane-per-row: raw loads of row r (clamped address, no branch); `inr` says whether the row exists
template <typename T, int D>
__device__ __forceinline__ void load_raw(const T* __restrict__ X, int64_t ldx, const T* __restrict__ y, int p,
                                         int64_t r, int64_t n, T* z, T& yv) {
  const int64_t rc = min(max(r, (int64_t)0), n - 1);
  const T* q = X + rc;
#pragma unroll
  for (int c = 0; c < D; ++c) {
    if (c < p) { z[c] = __ldg(q); q += ldx; }
    else z[c] = T(1);
  }
  yv = __ldg(y + rc);
}

// lane-per-row: e-vector of a row (all zero when the row is missing or not finite) -> dst[0..D+2)
template <typename T, int D>
__device__ __forceinline__ bool put_row(double* __restrict__ dst, const T* z, T yv, bool inr) {
  const bool fin = row_finite<T, D>(inr, z, yv);
#pragma unroll
  for (int c = 0; c < D; ++c) dst[c] = (double)(fin ? z[c] : T(0));
  dst[D] = (double)(fin ? yv : T(0));
  dst[D + 1] = fin ? 1.0 : 0.0;
  if (((D + 1) | 1) != D + 1) dst[(D + 1) | 1] = 0.0;
  return fin;
}

// lane-per-component: walk the 32 staged rows
template <typename T, int D, bool BOTH, bool STORE>
__device__ __forceinline__ void walk_batch(const double* __restrict__ ee, const double* __restrict__ el,
                                           const int* ta, const int* tb, const int* k0, const int* k1,
                                           double (*W)[2], T* __restrict__ gs, double* __restrict__ cnt, bool cnt_lane) {
  constexpr int ES = MomN<D>::ES, GS = MomN<D>::GS, TPL = MomN<D>::TPL, NT = MomN<D>::NT;
#pragma unroll
  for (int r = 0; r < BATCH; ++r) {
    const double* e = ee + r * ES;
    const double* l = el + r * ES;
#pragma unroll
    for (int m = 0; m < TPL; ++m) {
      const double ea = e[ta[m]];
      const double2 eb = *reinterpret_cast<const double2*>(e + tb[m]);
      W[m][0] = fma(ea, eb.x, W[m][0]);
      W[m][1] = fma(ea, eb.y, W[m][1]);
      if (BOTH) {
        const double la = l[ta[m]];
        const double2 lb = *reinterpret_cast<const double2*>(l + tb[m]);
        W[m][0] = fma(-la, lb.x, W[m][0]);
        W[m][1] = fma(-la, lb.y, W[m][1]);
      }
    }
    if (STORE) {
#pragma unroll
      for (int m = 0; m < TPL; ++m) {
        // products no moment wants (slot NM) are not stored: several lanes would write that slot, harmlessly, but
        // compute-sanitizer's racecheck reports every one of them as a WAW hazard
        if (k0[m] < MomN<D>::NM) gs[r * GS + k0[m]] = (T)W[m][0];
        if (k1[m] < MomN<D>::NM) gs[r * GS + k1[m]] = (T)W[m][1];
      }
      if (cnt_lane) cnt[r] = W[(NT - 1) / 32][(D + 1) & 1];     // the row count stays exact in f64
    }
  }
}

// ---------------- pass A: chain sums.  No per-row output here, so thread-per-row with all NM accumulators in
// registers is the cheap way: lane l takes rows chain0 + 32 j + l, one shuffle reduction per chain. ----------------
template <typename T, int D, typename A = T, bool ONE = true>
__global__ void __launch_bounds__(CTA_THREADS)
chain_sums_kernel(const T* __restrict__ X, int64_t ldx, const T* __restrict__ y, int64_t n, int p,
                  int64_t nchains, double* __restrict__ S /* [NM][nchains] */, ChainTab tab) {
  constexpr int NM = MomN<D>::NM;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int64_t k = (int64_t)blockIdx.x * WARPS + wid;
  if (k >= nchains) return;
  const ChainPos cp = chain_pos<ONE>(tab, k, n, 0);
  if (other_class<ONE>(tab, cp.skip)) return;
  X += cp.r0; y += cp.r0; n = cp.n;
  // Accumulation in A inside a lane (32 rows of the chain per lane), f64 across lanes.  A = the data type by default: for
  // f32 data the per-lane sums are 32-term f32 FMA chains, and a window of at least a chain only ever sees the DIFFERENCE
  // of a few chain sums, so the error does not grow with n.  (With f64 products this pass ran at 1.36 ms per 1e8 x 9 f32
  // = 40 % of the HBM peak: 45 DFMA + 9 conversions per row on a part whose FP64 pipe is narrow.)  That rounding is
  // relative to whole chains, though: a rolling window shorter than a chain, or thinned by skipped null rows, starts from
  // chain sums far larger than itself, and f32 chain sums put errors of 1e-5 relative on its coefficients.  Those fits
  // accumulate in A = double.
  constexpr int NMP = (NM + 31) / 32 * 32;               // padded to whole 32s for the transpose-reduce at the end
  A v[NM];
#pragma unroll
  for (int c = 0; c < NM; ++c) v[c] = A(0);
  const int64_t chain0 = cp.k * CHAIN_ROWS;
  // The pass is a pure stream (read (p+1) s bytes per row, keep NM sums): what bounds it is bytes in flight.  ncu, round
  // 2: with one 32-row batch of loads per warp outstanding the kernel sat at 25 % of the HBM peak (2.1 ms per 1e8 x 9
  // f32).  PF batches are kept in flight per warp (register ring, statically indexed by unrolling the loop PF times).
  // (f64 sums of f32 data at D = 12: 91 double accumulators leave room for one batch in flight without spilling)
  constexpr int PF = (D <= 6 || (sizeof(A) == 4 && D <= 9)) ? 4 : (sizeof(A) > sizeof(T) && D >= 12) ? 1 : 2;
  T zb[PF][D]; T yb[PF];
#pragma unroll
  for (int u = 0; u < PF; ++u) load_raw<T, D>(X, ldx, y, p, chain0 + (int64_t)u * 32 + lane, n, zb[u], yb[u]);
  for (int j0 = 0; j0 < CHAIN_ROWS / 32; j0 += PF) {
    // A group's last chain stops at the group's end: the rows after it are zero rows, and adding their +0.0 moments
    // leaves every sum's bits as they are (no sum is ever -0.0).  (The single column keeps the full loop, which only its
    // last chain runs past n on.)
    if (!ONE && chain0 + (int64_t)j0 * 32 >= n) break;
#pragma unroll
    for (int u = 0; u < PF; ++u) {
      const int j = j0 + u;
      const int64_t r = chain0 + (int64_t)j * 32 + lane;
      T z[D]; T yv;
#pragma unroll
      for (int c = 0; c < D; ++c) z[c] = zb[u][c];
      yv = yb[u];
      if (j + PF < CHAIN_ROWS / 32) load_raw<T, D>(X, ldx, y, p, r + PF * 32, n, zb[u], yb[u]);
      const bool fin = row_finite<T, D>(r < n, z, yv);
#pragma unroll
      for (int c = 0; c < D; ++c) z[c] = fin ? z[c] : T(0);
      yv = fin ? yv : T(0);
      int q = 0;
#pragma unroll
      for (int i = 0; i < D; ++i)
#pragma unroll
        for (int jj = i; jj < D; ++jj) { v[q] = fma((A)z[i], (A)z[jj], v[q]); ++q; }
#pragma unroll
      for (int i = 0; i < D; ++i) { v[q] = fma((A)z[i], (A)yv, v[q]); ++q; }
      v[q] += fin ? A(1) : A(0);
    }
  }
  // Transpose-reduce over the warp, in f64: at every step a lane hands the half of its values it does not keep to its
  // partner and adds the partner's half it keeps -> NMP - NMP / 32 double shuffles and DADDs for all NM sums, where the
  // butterfly per value cost 5 of each (a quarter of this kernel's instructions at NM = 46).  (The same tree in f32 was
  // 2 % faster still but put one rolling parity case outside the two-sided f32 rule of tests/parity_rule.py.)
  double dv[NMP];
#pragma unroll
  for (int c = 0; c < NMP; ++c) dv[c] = c < NM ? (double)v[c] : 0.0;
#pragma unroll
  for (int s = 16, m = NMP / 2; s >= 1; s >>= 1, m >>= 1) {
    const bool upper = (lane & s) != 0;
#pragma unroll
    for (int i = 0; i < m; ++i) {
      const double give = upper ? dv[i] : dv[i + m];
      const double keep = upper ? dv[i + m] : dv[i];
      dv[i] = keep + __shfl_xor_sync(0xffffffffu, give, s);
    }
  }
  const int cbase = ((lane >> 4) & 1) * (NMP / 2) + ((lane >> 3) & 1) * (NMP / 4) + ((lane >> 2) & 1) * (NMP / 8) +
                    ((lane >> 1) & 1) * (NMP / 16) + (lane & 1) * (NMP / 32);
#pragma unroll
  for (int j = 0; j < NMP / 32; ++j)
    if (cbase + j < NM) S[(size_t)(cbase + j) * nchains + k] = dv[j];
}

// ---------------- pass B: exclusive scan along tiles, one block per component ----------------
// M0 (optional): moments [X | y | 1]' [X | y | 1] ((p+2)^2, row-major f64) of the rows that precede this shard; they
// seed the prefix so that a row shard continues the expanding fit of the shards before it (SURVEY.md §8e).
__global__ void __launch_bounds__(1024) tile_scan_kernel(double* __restrict__ S, int64_t ntiles,
                                                         const double* __restrict__ M0, int p, int d) {
  __shared__ double warp_tot[32];
  __shared__ double carry;
  double* row = S + (size_t)blockIdx.x * ntiles;
  if (threadIdx.x == 0) {
    double c0 = 0.0;
    if (M0) {
      // z_c = x_c for c < p, the ones column otherwise
      int i, j;
      const int c = blockIdx.x;
      component_pair(c, d, i, j);
      auto col = [&](int a) { return a < p ? a : (a == d ? p : p + 1); };   // y -> p, bias / ones -> p + 1
      c0 = M0[(size_t)col(i) * (p + 2) + col(j)];
    }
    carry = c0;
  }
  __syncthreads();
  for (int64_t base = 0; base < ntiles; base += blockDim.x) {
    int64_t i = base + threadIdx.x;
    double v = (i < ntiles) ? row[i] : 0.0;
    double inc = v;
    for (int off = 1; off < 32; off <<= 1) { double t = __shfl_up_sync(0xffffffffu, inc, off); if ((threadIdx.x & 31) >= off) inc += t; }
    if ((threadIdx.x & 31) == 31) warp_tot[threadIdx.x >> 5] = inc;
    __syncthreads();
    double wpre = 0.0;
    for (int w = 0; w < (int)(threadIdx.x >> 5); ++w) wpre += warp_tot[w];
    double excl = carry + wpre + (inc - v);
    __syncthreads();
    if (i < ntiles) row[i] = excl;
    if (threadIdx.x == blockDim.x - 1) carry = excl + v;
    __syncthreads();
  }
}

// ---------------- pass B of a grouped call: every group's chains scanned alone ----------------
// One warp per (group, component) runs tile_scan_kernel's 1024-thread block on the group's chains, the block's 32 warps
// one after another: the same warp scans, the same running sum of the warp totals (wpre), the same carry from chunk to
// chunk of 1024 chains, starting at 0.0, and the same association carry + wpre + (inc - v).  Every value is therefore
// bit for bit the scan of a call on the group alone (a one-chain group gets (0.0 + 0.0) + (v - v)).  The block's warps
// past the group's last chain are not run: they only add zeros to wpre, and the carry they lead to is read only after a
// full chunk.  Work: one warp step per 32 chains of a group (at least one per group) and component.  A group of the other
// skip class (tab.cls) is left as it is.
constexpr int SCAN_WARPS = 8;
__global__ void __launch_bounds__(SCAN_WARPS * 32)
group_scan_kernel(double* __restrict__ S, int64_t nchains, ChainTab tab, int64_t n_groups) {
  const int lane = threadIdx.x & 31;
  const int64_t g = (int64_t)blockIdx.x * SCAN_WARPS + (threadIdx.x >> 5);
  if (g >= n_groups) return;
  if (other_class<false>(tab, tab.skip ? (int)__ldg(tab.skip + g) : 0)) return;
  const int64_t c0 = __ldg(tab.cbase + g), nch = __ldg(tab.cbase + g + 1) - c0;
  double* row = S + (size_t)blockIdx.y * nchains + c0;
  double carry = 0.0;
  for (int64_t base = 0; base < nch; base += 1024) {
    double wpre = 0.0, last = 0.0;
    for (int w = 0; w < 32 && base + 32 * w < nch; ++w) {
      const int64_t i = base + 32 * w + lane;
      const double v = (i < nch) ? row[i] : 0.0;
      double inc = v;
      for (int off = 1; off < 32; off <<= 1) { double t = __shfl_up_sync(0xffffffffu, inc, off); if (lane >= off) inc += t; }
      const double excl = carry + wpre + (inc - v);
      if (i < nch) row[i] = excl;
      last = excl + v;                                     // on lane 31 of the block's last warp: the next chunk's carry
      wpre += __shfl_sync(0xffffffffu, inc, 31);
    }
    carry = __shfl_sync(0xffffffffu, last, 31);
  }
}

// ---------------- in-register Cholesky solve on the packed Gram ----------------
// g: NM values in the component order (upper triangle row-major, then X'y, then the count).  lower(i, j) for i >= j
// lives at the slot of (j, i).  The diagonal is overwritten with 1/sqrt(pivot), so the substitutions multiply.
template <int D> __device__ __forceinline__ constexpr int gidx(int i, int j) { return j * D - j * (j - 1) / 2 + (i - j); }

template <typename T, int D>
__device__ __forceinline__ bool chol_solve_packed(T* g, T lambda, T* beta) {
  constexpr int NG = MomN<D>::NG;
  // The reference builds OnlineLR::new(lambda, false) on a matrix that already holds the physical ones column
  // (lr_online_solvers.rs:163-165, 195-197), so lambda lands on EVERY diagonal entry, the bias one included.
#pragma unroll
  for (int i = 0; i < D; ++i) { g[gidx<D>(i, i)] += lambda; beta[i] = g[NG + i]; }
  bool ok = true;
#pragma unroll
  for (int c = 0; c < D; ++c) {
    const T d = g[gidx<D>(c, c)];
    if (!(d > T(0)) || !isfinite(d)) ok = false;
    const T inv = rsqrt(d);
    g[gidx<D>(c, c)] = inv;
#pragma unroll
    for (int i = c + 1; i < D; ++i) g[gidx<D>(i, c)] *= inv;
#pragma unroll
    for (int j = c + 1; j < D; ++j)
#pragma unroll
      for (int i = j; i < D; ++i) g[gidx<D>(i, j)] -= g[gidx<D>(i, c)] * g[gidx<D>(j, c)];
  }
#pragma unroll
  for (int i = 0; i < D; ++i) {
    T s = beta[i];
#pragma unroll
    for (int j = 0; j < i; ++j) s -= g[gidx<D>(i, j)] * beta[j];
    beta[i] = s * g[gidx<D>(i, i)];
  }
#pragma unroll
  for (int i = D - 1; i >= 0; --i) {
    T s = beta[i];
#pragma unroll
    for (int j = i + 1; j < D; ++j) s -= g[gidx<D>(j, i)] * beta[j];
    beta[i] = s * g[gidx<D>(i, i)];
  }
  return ok;
}

// ---------------- pass C ----------------
// lane-per-moment kernel: rolling windows under half a chain start from their own rows, not from the chain sums
__host__ __device__ __forceinline__ bool online_direct_head(int64_t window) { return window > 0 && 2 * window < CHAIN_ROWS; }

// lane-per-moment kernel: acc += the moments of rows [a, b), staged and walked 32 rows at a time
template <typename T, int D>
__device__ __forceinline__ void walk_rows(const T* __restrict__ X, int64_t ldx, const T* __restrict__ y, int p, int64_t n,
                                          int64_t a, int64_t b, double* __restrict__ ee, int lane, const int* ta,
                                          const int* tb, const int* k0, const int* k1, double (*acc)[2]) {
  for (int64_t rb = a; rb < b; rb += BATCH) {
    T z[D]; T yv;
    const int64_t r = rb + lane;
    load_raw<T, D>(X, ldx, y, p, r, n, z, yv);
    put_row<T, D>(ee + lane * MomN<D>::ES, z, yv, r < b);
    __syncwarp();
    walk_batch<T, D, false, false>(ee, ee, ta, tb, k0, k1, acc, (T*)nullptr, (double*)nullptr, false);
    __syncwarp();
  }
}

// The body of the lane-per-moment kernels.  ONE: the single column, rolling when window > 0 (ROLL = true).  ONE = false:
// a grouped fit, recursive (ROLL = false: online_main_kernel<T, D, false>, no rolling code compiled in) or rolling
// (ROLL = true: online_rolling_kernel).
template <typename T, int D, bool ONE, bool ROLL>
__device__ __forceinline__ void
online_main(const T* __restrict__ X, int64_t ldx, const T* __restrict__ y, int64_t n, int p,
            int64_t window, int64_t min_rows, int skip, T lambda, int64_t row0, int64_t nchains,
            const double* __restrict__ C /* [NM][nchains] exclusive chain prefixes */,
            T* __restrict__ coeffs, T* __restrict__ pred, uint8_t* __restrict__ valid, const ChainTab& tab) {
  constexpr int NM = MomN<D>::NM, ES = MomN<D>::ES, GS = MomN<D>::GS, TPL = MomN<D>::TPL, NT = MomN<D>::NT;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int64_t k = (int64_t)blockIdx.x * WARPS + wid;
  if (k >= nchains) return;
  const ChainPos cp = chain_pos<ONE>(tab, k, n, skip);
  if (ROLL && other_class<ONE>(tab, cp.skip)) return;
  X += cp.r0; y += cp.r0; coeffs += cp.r0 * D; pred += cp.r0; valid += cp.r0; n = cp.n; skip = cp.skip;
  double* ee = reinterpret_cast<double*>(smem_raw + wid * warp_smem_bytes<T, D>());   // entering rows [32][ES]
  double* el = ee + BATCH * ES;                                                          // leaving rows  [32][ES]
  double* cnt = el + BATCH * ES;                                                         // finite-row count per row
  T* gs = reinterpret_cast<T*>(cnt + BATCH);                                             // W_t per row    [32][GS]
  const bool rolling = ROLL && window > 0;
  const int64_t chain0 = cp.k * CHAIN_ROWS;
  const bool cnt_lane = lane == ((NT - 1) & 31);
  // A window shorter than half a chain sums its rows [lo, chain0) directly: fewer rows than the head walk of the prefix
  // difference below, which also rounds relative to whole chains (1e-16 * 1024 rows in f64, 3e-8 relative on a window of
  // 2 rows).  Such fits do not read C (online_direct_head).
  const bool direct = ROLL && online_direct_head(window);

  int ta[TPL], tb[TPL], k0[TPL], k1[TPL];
  double W[TPL][2];
#pragma unroll
  for (int m = 0; m < TPL; ++m) {
    task_of<D>(lane + 32 * m, ta[m], tb[m], k0[m], k1[m]);
    W[m][0] = (!direct && k0[m] < NM) ? C[(size_t)k0[m] * nchains + k] : 0.0;
    W[m][1] = (!direct && k1[m] < NM) ? C[(size_t)k1[m] * nchains + k] : 0.0;
  }
  if (direct) {
    int64_t lo, kl;
    rolling_head(chain0, window, lo, kl);
    walk_rows<T, D>(X, ldx, y, p, n, lo, chain0, ee, lane, ta, tb, k0, k1, W);
  } else if (rolling) {
    int64_t lo, kl;
    rolling_head(chain0, window, lo, kl);
    // subtract the prefix up to lo = C[kl] + the rows [kl * CHAIN_ROWS, lo) (none when the window is a multiple of a
    // chain)
    double H[TPL][2];
#pragma unroll
    for (int m = 0; m < TPL; ++m) {
      H[m][0] = (k0[m] < NM) ? C[(size_t)k0[m] * nchains + (k - cp.k + kl)] : 0.0;
      H[m][1] = (k1[m] < NM) ? C[(size_t)k1[m] * nchains + (k - cp.k + kl)] : 0.0;
    }
    walk_rows<T, D>(X, ldx, y, p, n, kl * CHAIN_ROWS, lo, ee, lane, ta, tb, k0, k1, H);
#pragma unroll
    for (int m = 0; m < TPL; ++m) { W[m][0] -= H[m][0]; W[m][1] -= H[m][1]; }
  }

  // software pipeline: the raw rows of batch b+1 are in flight while batch b is walked and solved
  T zn[D], yn, zln[D], yln;
  load_raw<T, D>(X, ldx, y, p, chain0 + lane, n, zn, yn);
  if (rolling) load_raw<T, D>(X, ldx, y, p, chain0 + lane - window, n, zln, yln);
  for (int b = 0; b < CHAIN_ROWS / BATCH; ++b) {
    const int64_t rb = chain0 + (int64_t)b * BATCH;
    if (rb >= n) break;
    const int64_t r = rb + lane;
    // ---- lane-per-row: stage ----
    T z[D]; T yv;
#pragma unroll
    for (int c = 0; c < D; ++c) z[c] = zn[c];
    yv = yn;
    const bool fin = put_row<T, D>(ee + lane * ES, z, yv, r < n);
    if (rolling) put_row<T, D>(el + lane * ES, zln, yln, r - window >= 0 && r - window < n);
    load_raw<T, D>(X, ldx, y, p, r + BATCH, n, zn, yn);
    if (rolling) load_raw<T, D>(X, ldx, y, p, r + BATCH - window, n, zln, yln);
    __syncwarp();
    // ---- lane-per-component: walk ----
    if (rolling) walk_batch<T, D, true, true>(ee, el, ta, tb, k0, k1, W, gs, cnt, cnt_lane);
    else walk_batch<T, D, false, true>(ee, ee, ta, tb, k0, k1, W, gs, cnt, cnt_lane);
    __syncwarp();
    // ---- lane-per-row: solve ----
    T g[NM];
#pragma unroll
    for (int c = 0; c < NM; ++c) g[c] = gs[lane * GS + c];
    const double cn = cnt[lane];
    __syncwarp();
    const bool ok = row_valid(rolling, rb + lane, fin, cn, window, min_rows, skip, row0);
    T beta[D];
    T pr = T(0);
    if (ok) {
      const bool pd = chol_solve_packed<T, D>(g, lambda, beta);
      if (!pd) {
#pragma unroll
        for (int i = 0; i < D; ++i) beta[i] = (T)nan("");
      }
#pragma unroll
      for (int i = 0; i < D; ++i) pr = fma(z[i], beta[i], pr);
    } else {
#pragma unroll
      for (int i = 0; i < D; ++i) beta[i] = T(0);
    }
#pragma unroll
    for (int i = 0; i < D; ++i) gs[lane * D + i] = beta[i];
    __syncwarp();
    const int nout = (int)min((int64_t)BATCH, n - rb) * D;
    T* cdst = coeffs + rb * D;
#pragma unroll
    for (int i = 0; i < D; ++i) { const int idx = i * 32 + lane; if (idx < nout) cdst[idx] = gs[idx]; }   // coalesced
    if (r < n) { pred[r] = pr; valid[r] = ok ? 1 : 0; }
    __syncwarp();
  }
}

template <typename T, int D, bool ONE = true>
__global__ void __launch_bounds__(CTA_THREADS)
online_main_kernel(const T* __restrict__ X, int64_t ldx, const T* __restrict__ y, int64_t n, int p,
                   int64_t window, int64_t min_rows, int skip, T lambda, int64_t row0, int64_t nchains,
                   const double* __restrict__ C, T* __restrict__ coeffs, T* __restrict__ pred,
                   uint8_t* __restrict__ valid, ChainTab tab) {
  online_main<T, D, ONE, ONE>(X, ldx, y, n, p, window, min_rows, skip, lambda, row0, nchains, C, coeffs, pred, valid, tab);
}

template <typename T, int D>
__global__ void __launch_bounds__(CTA_THREADS)
online_rolling_kernel(const T* __restrict__ X, int64_t ldx, const T* __restrict__ y, int64_t n, int p,
                      int64_t window, int64_t min_rows, int skip, T lambda, int64_t row0, int64_t nchains,
                      const double* __restrict__ C, T* __restrict__ coeffs, T* __restrict__ pred,
                      uint8_t* __restrict__ valid, ChainTab tab) {
  online_main<T, D, false, true>(X, ldx, y, n, p, window, min_rows, skip, lambda, row0, nchains, C, coeffs, pred, valid,
                                 tab);
}

// =====================================================================================================================
// Pass C, f32, packed: the production kernel of rolling / recursive for float data (D <= 9).
//
// The kernel above is issue-slot-bound at ~40 warp-instructions per row — the f64
// lane-per-moment walk (4 LDS + 4 DFMA per row), the staging of e-vectors as doubles, and a 32-wide Cholesky.  This
// version does the same mathematics with a quarter of the instructions:
//   * a warp takes 64 rows per step and every lane owns the ADJACENT row pair (2l, 2l+1): all per-row arithmetic is
//     f32 pairs (ffma2 / fmul2 / fadd2 of f32x2.h), so products, window sums, the Cholesky and the prediction of two rows
//     cost one instruction stream;
//   * moments of a step are formed as products  m_k(t) = e_a e_b - l_a l_b  by the row lanes (2 packed instructions per
//     moment per 2 rows), written to shared memory [moment][row], and turned into running sums by lane-per-moment serial
//     scans over the 64 rows (LDS.128 / 4 FADD / STS.128) — in f32, from zero, so the rounding is that of a 64-term sum;
//   * f64 lives only at step boundaries: each moment lane keeps the exact-to-f64 base W_k (chain prefix from passes A/B
//     plus the step totals) and publishes it as f32 once per step;  W_t = base + scan(t)  is formed by the row lanes.
// The Gram the solver sees is an f32 rounding of the window moments, exactly as before (the old kernel cast its f64
// walk to T before the solve); what changes is 12 instead of 40 warp-instructions per row.
// =====================================================================================================================
constexpr int SB = 64;                   // rows per step of the packed kernel
constexpr int SBP = 68;                  // row stride of the product tile: 272 B = 16 (mod 128) -> conflict-free LDS.128 scans
constexpr int V2_WARPS = 4;

template <int D> struct V2 {
  static constexpr int NG = D * (D + 1) / 2;
  static constexpr int NM = NG + D + 1;
  static constexpr int TPL = (NM + 31) / 32;
  static constexpr int NB = (NM + 3) & ~3;
  static constexpr size_t warp_floats = (size_t)NM * SBP + NB;
};

__device__ __forceinline__ float2 f2(float a, float b) { return make_float2(a, b); }
__device__ __forceinline__ float2 bc(float a) { return make_float2(a, a); }

// raw pair load (rows r, r+1; clamped addresses, no branches); z[D] (features, ones for the bias slot) and y
template <int D, bool CLAMP = true>
__device__ __forceinline__ void load_pair(const float* __restrict__ X, int64_t ldx, const float* __restrict__ y, int p,
                                          int64_t r, int64_t n, float2* z, float2& yv) {
  const int64_t r0 = CLAMP ? min(max(r, (int64_t)0), n - 1) : r, r1 = CLAMP ? min(max(r + 1, (int64_t)0), n - 1) : r + 1;
  const float* q = X;
#pragma unroll
  for (int c = 0; c < D; ++c) {
    if (c < p) { z[c] = f2(__ldg(q + r0), __ldg(q + r1)); q += ldx; }
    else z[c] = f2(1.0f, 1.0f);
  }
  yv = f2(__ldg(y + r0), __ldg(y + r1));
}

// e-vector pair: zero where the row is missing or holds a non-finite value; fin = 1 / 0 per row
template <int D>
__device__ __forceinline__ void finish_pair(float2* z, float2& yv, bool in0, bool in1, float2& fin) {
  float2 acc = fmul2(yv, bc(0.0f));
#pragma unroll
  for (int c = 0; c < D; ++c) acc = ffma2(z[c], bc(0.0f), acc);      // 0 when every entry is finite, NaN otherwise
  const bool k0 = in0 && (acc.x == 0.0f), k1 = in1 && (acc.y == 0.0f);
  fin = f2(k0 ? 1.0f : 0.0f, k1 ? 1.0f : 0.0f);
  if (__all_sync(0xffffffffu, k0 && k1)) return;             // the usual case: every row of the step exists and is finite
#pragma unroll
  for (int c = 0; c < D; ++c) z[c] = f2(k0 ? z[c].x : 0.0f, k1 ? z[c].y : 0.0f);
  yv = f2(k0 ? yv.x : 0.0f, k1 ? yv.y : 0.0f);
}

// row lanes: products of one step -> tile[k][2 lane .. 2 lane + 1]
template <int D, bool BOTH>
__device__ __forceinline__ void put_products(float* __restrict__ tile, int lane, const float2* e, float2 ey, float2 ef,
                                             const float2* l, float2 ly, float2 lf) {
  constexpr int NG = V2<D>::NG, NM = V2<D>::NM;
  float2* out = reinterpret_cast<float2*>(tile) + lane;
  constexpr int ST = SBP / 2;                                // stride in float2
  int k = 0;
#pragma unroll
  for (int i = 0; i < D; ++i) {
    float2 nli = BOTH ? fmul2(l[i], bc(-1.0f)) : bc(0.0f);
#pragma unroll
    for (int j = i; j < D; ++j) {
      float2 m = BOTH ? ffma2(e[i], e[j], fmul2(nli, l[j])) : fmul2(e[i], e[j]);
      out[(size_t)k * ST] = m;
      ++k;
    }
    float2 my = BOTH ? ffma2(e[i], ey, fmul2(nli, ly)) : fmul2(e[i], ey);
    out[(size_t)(NG + i) * ST] = my;
  }
  out[(size_t)(NM - 1) * ST] = BOTH ? fadd2(ef, fmul2(lf, bc(-1.0f))) : ef;
}

// moment lanes: in-place inclusive scan of the 64 rows of their moments; returns the step totals.
// Two levels, so that nothing but a 16-long carry chain is serial: all 16 LDS.128 of a row are issued at once, the four
// values of every float4 are prefix-summed independently (16-way ILP), the carries run over the 16 group totals, and the
// carry is added back with packed adds.  (The first version walked the 64 values in one dependent LDS -> FADD chain:
// ncu attributed a quarter of all stall samples to those FADDs waiting on shared-memory loads.)
template <int D>
__device__ __forceinline__ void scan_products(float* __restrict__ tile, int lane, float* tot) {
  constexpr int NM = V2<D>::NM, TPL = V2<D>::TPL;
#pragma unroll
  for (int m = 0; m < TPL; ++m) {
    tot[m] = 0.0f;
    if (lane + 32 * m < NM) {
      float4* row = reinterpret_cast<float4*>(tile + (size_t)(lane + 32 * m) * SBP);
      float4 v[SB / 4];
#pragma unroll
      for (int i = 0; i < SB / 4; ++i) v[i] = row[i];
#pragma unroll
      for (int i = 0; i < SB / 4; ++i) { v[i].y += v[i].x; v[i].w += v[i].z; v[i].z += v[i].y; v[i].w += v[i].y; }
      float c = 0.0f;
#pragma unroll
      for (int i = 0; i < SB / 4; ++i) {
        const float t = v[i].w;
        const float2 lo = fadd2(make_float2(v[i].x, v[i].y), make_float2(c, c));
        const float2 hi = fadd2(make_float2(v[i].z, v[i].w), make_float2(c, c));
        row[i] = make_float4(lo.x, lo.y, hi.x, hi.y);
        c += t;
      }
      tot[m] = c;
    }
  }
}

// packed Cholesky solve of two rows at once (same algorithm as chol_solve_packed)
template <int D>
__device__ __forceinline__ void chol_solve_pair(float2* g, float lambda, float2* beta, bool& ok0, bool& ok1) {
  constexpr int NG = V2<D>::NG;
#pragma unroll
  for (int i = 0; i < D; ++i) { g[gidx<D>(i, i)] = fadd2(g[gidx<D>(i, i)], bc(lambda)); beta[i] = g[NG + i]; }
  ok0 = ok1 = true;
#pragma unroll
  for (int c = 0; c < D; ++c) {
    const float2 d = g[gidx<D>(c, c)];
    if (!(d.x > 0.0f) || !isfinite(d.x)) ok0 = false;
    if (!(d.y > 0.0f) || !isfinite(d.y)) ok1 = false;
    const float2 inv = f2(rsqrtf(d.x), rsqrtf(d.y));
    g[gidx<D>(c, c)] = inv;
#pragma unroll
    for (int i = c + 1; i < D; ++i) g[gidx<D>(i, c)] = fmul2(g[gidx<D>(i, c)], inv);
#pragma unroll
    for (int j = c + 1; j < D; ++j) {
      const float2 nj = fmul2(g[gidx<D>(j, c)], bc(-1.0f));
#pragma unroll
      for (int i = j; i < D; ++i) g[gidx<D>(i, j)] = ffma2(g[gidx<D>(i, c)], nj, g[gidx<D>(i, j)]);
    }
  }
  float2 nb[D];                       // -beta: the packed FMA has no negate modifier, so the sign is carried by the vector
#pragma unroll
  for (int i = 0; i < D; ++i) {
    float2 s = beta[i];
#pragma unroll
    for (int j = 0; j < i; ++j) s = ffma2(g[gidx<D>(i, j)], nb[j], s);
    beta[i] = fmul2(s, g[gidx<D>(i, i)]);
    nb[i] = fmul2(beta[i], bc(-1.0f));
  }
#pragma unroll
  for (int i = D - 1; i >= 0; --i) {
    float2 s = beta[i];
#pragma unroll
    for (int j = i + 1; j < D; ++j) s = ffma2(g[gidx<D>(j, i)], nb[j], s);
    beta[i] = fmul2(s, g[gidx<D>(i, i)]);
    nb[i] = fmul2(beta[i], bc(-1.0f));
  }
}

// The raw rows of the next step are prefetched into registers (4-warp CTAs, 2 CTAs per SM at D = 8).  Variants without
// the prefetch, capped for 3 or 4 CTAs per SM so that more warps hide the load latency instead, measured slower and
// were removed.
// ONE = false: a grouped fit.  A group's first row r0 may be odd, and the window may be odd.  Every global load is a
// scalar __ldg (load_pair pairs two of them in registers), entering rows and leaving rows r - window alike, so neither
// needs alignment.  The only float2 accesses to global memory are the coefficient stores of an even D, at float offset
// (r0 + r) D with r even: even, so 8-byte aligned for any r0 and window.  The float4 / float2 accesses of tile and basef
// are in shared memory, at offsets that do not depend on r0 or the window.
template <int D, bool ROLLING, bool ONE = true>
__global__ void __launch_bounds__(V2_WARPS * 32, 1)
online_main_f32x2_kernel(const float* __restrict__ X, int64_t ldx, const float* __restrict__ y, int64_t n, int p,
                         int64_t window, int64_t min_rows, int skip, float lambda, int64_t row0, int64_t nchains,
                         const double* __restrict__ C /* [NM][nchains] exclusive chain prefixes */,
                         float* __restrict__ coeffs, float* __restrict__ pred, uint8_t* __restrict__ valid,
                         ChainTab tab) {
  constexpr int NM = V2<D>::NM, TPL = V2<D>::TPL, NB = V2<D>::NB;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int64_t k = (int64_t)blockIdx.x * V2_WARPS + wid;
  if (k >= nchains) return;
  const ChainPos cp = chain_pos<ONE>(tab, k, n, skip);
  if (ROLLING && other_class<ONE>(tab, cp.skip)) return;     // a recursive plan does not depend on skip
  X += cp.r0; y += cp.r0; coeffs += cp.r0 * D; pred += cp.r0; valid += cp.r0; n = cp.n; skip = cp.skip;
  float* tile = reinterpret_cast<float*>(smem_raw) + (size_t)wid * V2<D>::warp_floats;     // [NM][SBP]
  float* basef = tile + (size_t)NM * SBP;                                                   // [NB]
  const int64_t chain0 = cp.k * CHAIN_ROWS;

  // moment lanes: f64 base of "their" moments at the chain start
  double W[TPL];
#pragma unroll
  for (int m = 0; m < TPL; ++m) W[m] = (lane + 32 * m < NM) ? C[(size_t)(lane + 32 * m) * nchains + k] : 0.0;
  if (ROLLING) {
    // subtract the prefix up to lo = C[kl] + the rows [kl * CHAIN_ROWS, lo)
    int64_t lo, kl;
    rolling_head(chain0, window, lo, kl);
#pragma unroll
    for (int m = 0; m < TPL; ++m) if (lane + 32 * m < NM) W[m] -= C[(size_t)(lane + 32 * m) * nchains + (k - cp.k + kl)];
    for (int64_t rb = kl * CHAIN_ROWS; rb < lo; rb += SB) {       // empty when the window is a multiple of the chain
      float2 z[D], yv, fin;
      const int64_t r = rb + 2 * lane;
      load_pair<D>(X, ldx, y, p, r, n, z, yv);
      finish_pair<D>(z, yv, r < lo, r + 1 < lo, fin);
      put_products<D, false>(tile, lane, z, yv, fin, z, yv, fin);
      __syncwarp();
      float tot[TPL];
      scan_products<D>(tile, lane, tot);
#pragma unroll
      for (int m = 0; m < TPL; ++m) W[m] -= (double)tot[m];
      __syncwarp();
    }
  }

  // interior chains (all but the first and the last few) need neither clamped addresses nor row-exists tests
  const bool interior = (chain0 + CHAIN_ROWS + SB <= n) && (!ROLLING || chain0 - window >= 0);
  // software pipeline: the raw rows of step b+1 are in flight while step b is scanned and solved
  float2 zn[D], yn, zln[D], yln;
  load_pair<D>(X, ldx, y, p, chain0 + 2 * lane, n, zn, yn);
  if (ROLLING) load_pair<D>(X, ldx, y, p, chain0 + 2 * lane - window, n, zln, yln);
  for (int b = 0; b < CHAIN_ROWS / SB; ++b) {
    const int64_t rb = chain0 + (int64_t)b * SB;
    if (rb >= n) break;
    const int64_t r = rb + 2 * lane;
    // ---- row lanes: products of the step ----
    float2 z[D], yv, fin, zl[D], yl;
#pragma unroll
    for (int c = 0; c < D; ++c) { z[c] = zn[c]; if (ROLLING) zl[c] = zln[c]; }
    yv = yn; yl = yln;
    finish_pair<D>(z, yv, interior || r < n, interior || r + 1 < n, fin);
    if (ROLLING) {
      float2 lf;
      finish_pair<D>(zl, yl, interior || (r - window >= 0 && r - window < n), interior || (r + 1 - window >= 0 && r + 1 - window < n), lf);
      put_products<D, true>(tile, lane, z, yv, fin, zl, yl, lf);
    } else {
      put_products<D, false>(tile, lane, z, yv, fin, z, yv, fin);
    }
    if (interior) {
      load_pair<D, false>(X, ldx, y, p, r + SB, n, zn, yn);
      if (ROLLING) load_pair<D, false>(X, ldx, y, p, r + SB - window, n, zln, yln);
    } else {
      load_pair<D>(X, ldx, y, p, r + SB, n, zn, yn);
      if (ROLLING) load_pair<D>(X, ldx, y, p, r + SB - window, n, zln, yln);
    }
    __syncwarp();
    // ---- moment lanes: publish the base, scan, advance the base ----
    {
      float tot[TPL];
#pragma unroll
      for (int m = 0; m < TPL; ++m) if (lane + 32 * m < NM) basef[lane + 32 * m] = (float)W[m];
      scan_products<D>(tile, lane, tot);
#pragma unroll
      for (int m = 0; m < TPL; ++m) W[m] += (double)tot[m];
    }
    __syncwarp();
    // ---- row lanes: W_t = base + scan(t), solve both rows, predict ----
    float2 g[NM];
    {
      const float2* src = reinterpret_cast<const float2*>(tile) + lane;
#pragma unroll
      for (int c4 = 0; c4 < NB / 4; ++c4) {
        const float4 b4 = *reinterpret_cast<const float4*>(basef + 4 * c4);
        const float bb[4] = {b4.x, b4.y, b4.z, b4.w};
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const int c = 4 * c4 + u;
          if (c < NM) g[c] = fadd2(src[(size_t)c * (SBP / 2)], bc(bb[u]));
        }
      }
    }
    __syncwarp();
    const float2 cn = g[NM - 1];
    const bool ok0 = row_valid(ROLLING, rb + 2 * lane, fin.x != 0.0f, cn.x, window, min_rows, skip, row0);
    const bool ok1 = row_valid(ROLLING, r + 1, fin.y != 0.0f, cn.y, window, min_rows, skip, row0);
    float2 beta[D];
    bool pd0, pd1;
    chol_solve_pair<D>(g, lambda, beta, pd0, pd1);
    float2 pr = bc(0.0f);
#pragma unroll
    for (int i = 0; i < D; ++i) {
      beta[i] = f2(ok0 ? (pd0 ? beta[i].x : nanf("")) : 0.0f, ok1 ? (pd1 ? beta[i].y : nanf("")) : 0.0f);
      pr = ffma2(z[i], beta[i], pr);
    }
    // rows 2l, 2l+1 are adjacent: 2 D consecutive floats per lane, consecutive lanes consecutive -> coalesced
    if (r + 1 < n) {
      float* cdst = coeffs + r * D;
      if ((D & 1) == 0) {
        float2* c2 = reinterpret_cast<float2*>(cdst);
#pragma unroll
        for (int i = 0; i < D / 2; ++i) c2[i] = f2(beta[2 * i].x, beta[2 * i + 1].x);
#pragma unroll
        for (int i = 0; i < D / 2; ++i) c2[D / 2 + i] = f2(beta[2 * i].y, beta[2 * i + 1].y);
      } else {
#pragma unroll
        for (int i = 0; i < D; ++i) cdst[i] = beta[i].x;
#pragma unroll
        for (int i = 0; i < D; ++i) cdst[D + i] = beta[i].y;
      }
      pred[r] = pr.x; pred[r + 1] = pr.y;
      valid[r] = ok0 ? 1 : 0; valid[r + 1] = ok1 ? 1 : 0;
    } else if (r < n) {
      float* cdst = coeffs + r * D;
#pragma unroll
      for (int i = 0; i < D; ++i) cdst[i] = beta[i].x;
      pred[r] = pr.x;
      valid[r] = ok0 ? 1 : 0;
    }
  }
}

// =====================================================================================================================
// Generic pass C for any number of coefficients (D > 12): the reference takes any p (lr_online_solvers.rs:148-301).
// One warp per chain, rows in order; the window moments live in shared memory as f64 ((D+2)(D+3)/2 packed upper
// triangle over (z, y, 1)), lanes stride over the moments for the rank-1 updates and cooperate on an f64 Cholesky of a
// scratch copy per row.  O(D^3 / 32) per row — a correctness path, not a roofline one.
// =====================================================================================================================

// one warp: row r over (z, y, 1) as doubles -> dst[0..d+2), all zero when the row is missing or not finite
template <typename T>
__device__ __forceinline__ bool load_row(const T* __restrict__ X, int64_t ldx, const T* __restrict__ y, int64_t n, int p,
                                         int d, int lane, int64_t r, double* dst) {
  bool fin = r >= 0 && r < n;
  double acc = 0.0;
  for (int c = lane; c <= d; c += 32) {
    double v = 0.0;
    if (fin) v = (c < p) ? (double)X[(size_t)c * ldx + r] : (c < d ? 1.0 : (double)y[r]);
    dst[c] = v;
    acc += v * 0.0;
  }
  for (int off = 16; off; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
  fin = fin && (acc == 0.0);
  __syncwarp();
  if (!fin) for (int c = lane; c <= d; c += 32) dst[c] = 0.0;
  if (lane == 0) dst[d + 1] = fin ? 1.0 : 0.0;
  __syncwarp();
  return fin;
}

// one warp: W += sgn * (the moments of row v), lanes striding over the components
__device__ __forceinline__ void rank1(double* W, const double* v, double sgn, int d, int lane) {
  const int nm = d * (d + 1) / 2 + d + 1;
  for (int c = lane; c < nm; c += 32) {
    int i, j;
    component_pair(c, d, i, j);
    W[c] += sgn * v[i] * v[j];
  }
  __syncwarp();
}

// ONE = false: a grouped fit, rolling when window > 0.
template <typename T, bool ONE = true>
__global__ void __launch_bounds__(32)
online_generic_kernel(const T* __restrict__ X, int64_t ldx, const T* __restrict__ y, int64_t n, int p, int d,
                      int64_t window, int64_t min_rows, int skip, double lambda, int64_t row0, int64_t nchains,
                      const double* __restrict__ C /* [NM][nchains] */, T* __restrict__ coeffs, T* __restrict__ pred,
                      uint8_t* __restrict__ valid, ChainTab tab) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int lane = threadIdx.x;
  const int64_t k = blockIdx.x;
  const ChainPos cp = chain_pos<ONE>(tab, k, n, skip);
  if (other_class<ONE>(tab, cp.skip)) return;
  X += cp.r0; y += cp.r0; coeffs += cp.r0 * d; pred += cp.r0; valid += cp.r0; n = cp.n; skip = cp.skip;
  const int ng = d * (d + 1) / 2, nm = ng + d + 1;
  double* W = reinterpret_cast<double*>(smem_raw);      // [nm] window moments, component order of the chain sums
  double* A = W + nm;                                   // [d*d] scratch (lower triangle used)
  double* e = A + d * d;                                // [d+2] entering row
  double* l = e + d + 2;                                // [d+2] leaving row
  double* bt = l + d + 2;                               // [d]
  const bool rolling = window > 0;
  const int64_t chain0 = cp.k * CHAIN_ROWS;
  for (int c = lane; c < nm; c += 32) W[c] = C[(size_t)c * nchains + k];
  __syncwarp();
  if (rolling) {
    int64_t lo, kl;
    rolling_head(chain0, window, lo, kl);
    for (int c = lane; c < nm; c += 32) W[c] -= C[(size_t)c * nchains + (k - cp.k + kl)];
    __syncwarp();
    for (int64_t r = kl * CHAIN_ROWS; r < lo; ++r) { load_row(X, ldx, y, n, p, d, lane, r, e); rank1(W, e, -1.0, d, lane); }
  }
  for (int64_t r = chain0; r < min(chain0 + (int64_t)CHAIN_ROWS, n); ++r) {
    const bool fin = load_row(X, ldx, y, n, p, d, lane, r, e);
    rank1(W, e, 1.0, d, lane);
    if (rolling) { load_row(X, ldx, y, n, p, d, lane, r - window, l); rank1(W, l, -1.0, d, lane); }
    const bool ok = row_valid(rolling, r, fin, W[nm - 1], window, min_rows, skip, row0);
    bool pd = true;
    if (ok) {
      // A = lower triangle of G + lambda I, rounded through T like the packed kernels; bt = X'y
      for (int c = lane; c < ng; c += 32) {
        int i, j;
        component_pair(c, d, i, j);
        A[j * d + i] = (double)(T)W[c] + (i == j ? lambda : 0.0);
      }
      for (int c = lane; c < d; c += 32) bt[c] = (double)(T)W[ng + c];
      __syncwarp();
      for (int c = 0; c < d; ++c) {
        const double dg = A[c * d + c];
        if (!(dg > 0.0) || !isfinite(dg)) pd = false;
        const double inv = rsqrt(dg);
        __syncwarp();
        for (int i = c + 1 + lane; i < d; i += 32) A[i * d + c] *= inv;
        if (lane == 0) A[c * d + c] = inv;
        __syncwarp();
        for (int idx = lane; idx < (d - c - 1) * (d - c - 1); idx += 32) {
          const int j = c + 1 + idx / (d - c - 1), i = c + 1 + idx % (d - c - 1);
          if (i >= j) A[i * d + j] -= A[i * d + c] * A[j * d + c];
        }
        __syncwarp();
      }
      for (int i = 0; i < d; ++i) {            // forward substitution (lane-parallel dot)
        double s = 0.0;
        for (int j = lane; j < i; j += 32) s += A[i * d + j] * bt[j];
        for (int off = 16; off; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
        if (lane == 0) bt[i] = (bt[i] - s) * A[i * d + i];
        __syncwarp();
      }
      for (int i = d - 1; i >= 0; --i) {       // backward
        double s = 0.0;
        for (int j = i + 1 + lane; j < d; j += 32) s += A[j * d + i] * bt[j];
        for (int off = 16; off; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
        if (lane == 0) bt[i] = (bt[i] - s) * A[i * d + i];
        __syncwarp();
      }
    }
    double prs = 0.0;
    for (int c = lane; c < d; c += 32) {
      const double bv = ok ? (pd ? bt[c] : nan("")) : 0.0;
      coeffs[r * d + c] = (T)bv;
      const double zc = (c < p) ? (double)X[(size_t)c * ldx + r] : 1.0;
      prs += ok ? zc * (double)(T)bv : 0.0;
    }
    for (int off = 16; off; off >>= 1) prs += __shfl_xor_sync(0xffffffffu, prs, off);
    if (lane == 0) { pred[r] = (T)prs; valid[r] = ok ? 1 : 0; }
    __syncwarp();
  }
}

// chain sums for any d (generic path): one warp per chain, lanes stride over the moments
template <typename T, bool ONE = true>
__global__ void __launch_bounds__(32)
chain_sums_generic_kernel(const T* __restrict__ X, int64_t ldx, const T* __restrict__ y, int64_t n, int p, int d,
                          int64_t nchains, double* __restrict__ S, ChainTab tab) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int lane = threadIdx.x;
  const int64_t k = blockIdx.x;
  const ChainPos cp = chain_pos<ONE>(tab, k, n, 0);
  if (other_class<ONE>(tab, cp.skip)) return;
  X += cp.r0; y += cp.r0; n = cp.n;
  const int nm = d * (d + 1) / 2 + d + 1;
  double* acc = reinterpret_cast<double*>(smem_raw);   // [nm]
  double* e = acc + nm;                                // [d+2]
  for (int c = lane; c < nm; c += 32) acc[c] = 0.0;
  __syncwarp();
  // a non-finite row adds its zeroed moments: the sums start at +0.0, so that leaves every bit as it is
  for (int64_t r = cp.k * CHAIN_ROWS; r < min((cp.k + 1) * (int64_t)CHAIN_ROWS, n); ++r) {
    load_row(X, ldx, y, n, p, d, lane, r, e);
    rank1(acc, e, 1.0, d, lane);
  }
  for (int c = lane; c < nm; c += 32) S[(size_t)c * nchains + k] = acc[c];
}

// ---------------- which kernels run, and the driver that runs them ----------------
enum class PassA { none, data_type, f64, generic };     // chain sums: none, in the data type, in f64, generic kernel
enum class PassC { packed = 1, lane = 2, generic = 3 };  // numbered as pdsb_last_online_path reports them
struct OnlinePlan { PassA a; PassC c; };

// The kernels of one call (window 0: recursive).
// * The templated kernels take 1 to 12 coefficients; any other number runs the generic kernels.
// * Packed pass C: f32 with at most 9 coefficients (up to 255 registers at D = 8 and 9; wider fits would spill),
//   recursive, or rolling with window >= SB that does not skip null rows.  The packed kernel sums a step's products in f32
//   from zero: for a window shorter than the 64-row step the partial sums (a random walk over 64 rows) are larger than
//   the window sum they end in and the rounding shows (3e-6 relative at window 2).  A window thinned by skipped nulls
//   (6 finite rows of 127) is far smaller than the f32 step sums of every row that entered or left since the chain
//   start, and its coefficients were off by 2e-5 relative; the packed kernel also zeroes a null row before predicting,
//   where the reference predicts x . beta from the raw row (NaN for a null feature, finite when only y is null), and
//   reloading the row there cost 4-5 % on the no-null path.  Every other fit takes the lane-per-moment kernel, which
//   sums exact products in f64 and predicts from the raw row.
// * Passes A and B feed every fit but the lane-per-moment kernel's short windows (online_direct_head), which start
//   from their own rows.
// * f32 chain sums round relative to whole chains: an f32 rolling window shorter than a chain, or one that skips null
//   rows, takes f64 chain sums (see chain_sums_kernel).
OnlinePlan online_plan(bool f32, int d, int64_t window, bool skip) {
  if (d < 1 || d > 12) return {PassA::generic, PassC::generic};
  const bool packed = f32 && d <= 9 && (window == 0 || (window >= SB && !skip));
  if (!packed && online_direct_head(window)) return {PassA::none, PassC::lane};
  const bool f64_sums = f32 && window > 0 && (skip || window < CHAIN_ROWS);
  return {f64_sums ? PassA::f64 : PassA::data_type, packed ? PassC::packed : PassC::lane};
}

// raises the kernel's dynamic shared-memory limit when it needs more than the default 48 KB, then launches it
template <typename... P, typename... A>
cudaError_t launch_kernel(void (*kernel)(P...), dim3 grid, unsigned block, size_t smem, cudaStream_t s, A... args) {
  if (smem > 48 * 1024) {
    const cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
  }
  kernel<<<grid, block, smem, s>>>(args...);
  count_launch();
  return cudaGetLastError();
}

// shared memory of the generic pass C for d coefficients (online_generic_kernel: the window moments, d x d scratch, the
// entering and leaving rows and beta), and the most coefficients it takes: the largest d that fits GENERIC_C_SMEM (129)
constexpr size_t GENERIC_C_SMEM = 200 * 1024;
constexpr size_t generic_c_smem(int d) { return (size_t)(d * (d + 1) / 2 + d + 1 + d * d + 2 * (d + 2) + d) * sizeof(double); }
constexpr int generic_c_max_coeffs() {
  int d = 1;
  while (generic_c_smem(d + 1) <= GENERIC_C_SMEM) ++d;
  return d;
}
static_assert(generic_c_max_coeffs() == 129, "DESIGN.md (deviations) and the tests state this bound");

// Runs the plan: passes A and B if it has them, then pass C.  D = 1..12 runs the kernels templated on that number of
// coefficients, D = 0 the generic ones.  ONE: the single column of n rows (nchains = its chains, tab unused); otherwise
// the grouped fit over the chain table (nchains = every group's chains, n_groups groups; m0 null, row0 0), of the groups
// of skip class tab.cls only when that is 0 or 1.
template <typename T, int D, bool ONE>
int run_online(const OnlinePlan& plan, const T* X, int64_t ldx, const T* y, int64_t n, int p, int d, int64_t window,
               int64_t min_rows, int skip, double lambda, const double* m0, int64_t row0, T* coeffs, T* pred,
               uint8_t* valid, int64_t nchains, const ChainTab& tab, int64_t n_groups, cudaStream_t s) {
  const int nm = d * (d + 1) / 2 + d + 1;
  const size_t smem_generic_a = (size_t)(nm + d + 2) * sizeof(double);
  const size_t smem_generic_c = generic_c_smem(d);
  if (D == 0 && smem_generic_c > GENERIC_C_SMEM) {
    set_error("rolling/recursive lin_reg: %d coefficients exceed the device limit of %d", d, generic_c_max_coeffs());
    return 1;
  }
  double* S = nullptr;
  if (plan.a != PassA::none && dev_alloc((void**)&S, (size_t)nm * nchains * sizeof(double), s)) return 1;
  cudaError_t e = cudaSuccess;
  if (plan.a != PassA::none) {
    if constexpr (D == 0)
      e = launch_kernel(chain_sums_generic_kernel<T, ONE>, (unsigned)nchains, 32, smem_generic_a, s, X, ldx, y, n, p, d,
                        nchains, S, tab);
    else
      e = launch_kernel(plan.a == PassA::f64 ? chain_sums_kernel<T, D, double, ONE> : chain_sums_kernel<T, D, T, ONE>,
                        (unsigned)ceil_div(nchains, WARPS), CTA_THREADS, 0, s, X, ldx, y, n, p, nchains, S, tab);
    if (e == cudaSuccess) {
      if (ONE) e = launch_kernel(tile_scan_kernel, (unsigned)nm, 1024, 0, s, S, nchains, m0, p, d);
      else e = launch_kernel(group_scan_kernel, dim3((unsigned)ceil_div(n_groups, SCAN_WARPS), (unsigned)nm), SCAN_WARPS * 32,
                             0, s, S, nchains, tab, n_groups);
    }
  }
  if (e == cudaSuccess) {
    if constexpr (D == 0) {
      e = launch_kernel(online_generic_kernel<T, ONE>, (unsigned)nchains, 32, smem_generic_c, s, X, ldx, y, n, p, d, window,
                        min_rows, skip, lambda, row0, nchains, S, coeffs, pred, valid, tab);
    } else if (plan.c == PassC::lane) {
      // the single column and a grouped recursive fit: online_main_kernel; a grouped fit with a window: the rolling
      // instance.  online_plan gives a grouped recursive f32 fit of <= 9 coefficients the packed kernel, so that case has
      // no lane instance: should a plan ever ask for it, the call fails here instead of running another kernel.
      auto kernel = online_rolling_kernel<T, D>;
      if constexpr (ONE || !std::is_same<T, float>::value || D > 9) {
        if (ONE || window == 0) kernel = online_main_kernel<T, D, ONE>;
      } else if (window == 0) {
        e = cudaErrorNotSupported;
      }
      if (e == cudaSuccess)
        e = launch_kernel(kernel, (unsigned)ceil_div(nchains, WARPS), CTA_THREADS, WARPS * warp_smem_bytes<T, D>(), s, X,
                          ldx, y, n, p, window, min_rows, skip, (T)lambda, row0, nchains, S, coeffs, pred, valid, tab);
    } else if constexpr (std::is_same<T, float>::value && D <= 9) {
      e = launch_kernel(window > 0 ? online_main_f32x2_kernel<D, true, ONE> : online_main_f32x2_kernel<D, false, ONE>,
                        (unsigned)ceil_div(nchains, V2_WARPS), V2_WARPS * 32, V2_WARPS * V2<D>::warp_floats * sizeof(float),
                        s, X, ldx, y, n, p, window, min_rows, skip, (float)lambda, row0, nchains, S, coeffs, pred, valid,
                        tab);
    } else {
      e = cudaErrorNotSupported;   // a packed plan for data the packed kernel does not take (online_plan never makes one)
    }
  }
  dev_free(S, s);
  if (e != cudaSuccess) { set_error("online lin_reg launch failed: %s", cudaGetErrorString(e)); return 1; }
  t_last_online_path = (int)plan.c;
  return 0;
}

// cnt[g] = the chains of group g (its rows cut into CHAIN_ROWS from its first row); cnt[n_groups] = 0
__global__ void group_chain_counts(const int64_t* __restrict__ off, int64_t n_groups, int64_t* __restrict__ cnt) {
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g <= n_groups; g += (int64_t)gridDim.x * blockDim.x)
    cnt[g] = g < n_groups ? (__ldg(off + g + 1) - __ldg(off + g) + CHAIN_ROWS - 1) / CHAIN_ROWS : 0;
}

// cls[c] += the groups with rows whose skip flag is c (0 or 1): which of a rolling call's two plans have work
__global__ void group_class_counts(const int64_t* __restrict__ off, const uint8_t* __restrict__ skip, int64_t n_groups,
                                   unsigned long long* __restrict__ cls) {
  unsigned long long c0 = 0, c1 = 0;
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < n_groups; g += (int64_t)gridDim.x * blockDim.x)
    if (__ldg(off + g + 1) > __ldg(off + g)) { if (__ldg(skip + g)) ++c1; else ++c0; }
  for (int o = 16; o; o >>= 1) {
    c0 += __shfl_down_sync(0xffffffffu, c0, o);
    c1 += __shfl_down_sync(0xffffffffu, c1, o);
  }
  if ((threadIdx.x & 31) == 0) {
    if (c0) atomicAdd(cls, c0);
    if (c1) atomicAdd(cls + 1, c1);
  }
}

}  // namespace

template <typename T>
int online_lin_reg(const T* X, int64_t ldx, const T* y, int64_t n, int p, int add_bias, int64_t window,
                   int64_t min_rows, int skip, double lambda, const double* m0, int64_t row0, T* coeffs, T* pred,
                   uint8_t* valid, cudaStream_t s) {
  t_last_online_path = 0;
  if (n <= 0) return 0;
  if (window > 0 && m0) { set_error("online lin_reg: preceding-row moments only apply to the recursive fit"); return 1; }
  const int d = p + (add_bias ? 1 : 0);
  if (n / CHAIN_ROWS > 2000000000LL) { set_error("online lin_reg: too many rows"); return 1; }
  const OnlinePlan plan = online_plan(std::is_same<T, float>::value, d, window, skip);
  const int64_t nchains = ceil_div(n, CHAIN_ROWS);
#define CASE_D(DD) case DD: return run_online<T, DD, true>(plan, X, ldx, y, n, p, d, window, min_rows, skip, lambda, m0, row0, coeffs, pred, valid, nchains, ChainTab{}, 1, s);
  switch (plan.c == PassC::generic ? 0 : d) {
    CASE_D(1) CASE_D(2) CASE_D(3) CASE_D(4) CASE_D(5) CASE_D(6) CASE_D(7) CASE_D(8) CASE_D(9) CASE_D(10)
    CASE_D(11) CASE_D(12)
    default:   // any number of coefficients, like the reference (lr_online_solvers.rs:148-301)
      CASE_D(0)
  }
#undef CASE_D
}

namespace {

// The chain table takes one read-back of the total chain count (one host synchronisation), so that the scratch, the
// grids and the table are exact; sizing them for the bound n / CHAIN_ROWS + n_groups instead would spend up to n_groups
// chains of NM doubles each on a call of short groups, where the read-back costs microseconds.
// A rolling plan depends on skip (online_plan).  When the two skip classes' plans differ, the same read-back brings the
// number of groups with rows in each class: a class that is present runs its own plan over its own groups (tab.cls), the
// no-skip class first, so pdsb_last_online_path reports the skip class's pass C.  Each plan's passes A and B write the
// chain sums and prefixes of its class's chains only, and its pass C reads only those.
template <typename T>
int grouped_online_lin_reg(const T* X, int64_t ldx, const T* y, const int64_t* offsets, const uint8_t* skip,
                           int64_t n_groups, int64_t n, int p, int add_bias, int64_t window, int64_t min_rows,
                           double lambda, T* coeffs, T* pred, uint8_t* valid, cudaStream_t s) {
  t_last_online_path = 0;
  const char* what = window > 0 ? "rolling lin_reg" : "recursive lin_reg";
  if (n < 0 || n_groups < 0 || p < 1 || window < 0 ||
      (n > 0 && (!X || !y || !offsets || !coeffs || !pred || !valid || n_groups < 1))) {
    set_error("%s: invalid arguments", what);
    return 1;
  }
  if (n == 0) return 0;
  const int d = p + (add_bias ? 1 : 0);
  const bool f32 = std::is_same<T, float>::value;
  // a recursive plan does not depend on skip: one plan, and one pass-C kernel, for every group
  const OnlinePlan plans[2] = {online_plan(f32, d, window, false), online_plan(f32, d, window, window > 0)};
  const bool split = skip && (plans[0].a != plans[1].a || plans[0].c != plans[1].c);
  DevBag bag(s);
  int64_t* cnt = bag.alloc<int64_t>((size_t)n_groups + 1);
  int64_t* cbase = bag.alloc<int64_t>((size_t)n_groups + 1);
  unsigned long long* dcls = split ? bag.alloc<unsigned long long>(2) : nullptr;
  if (!cnt || !cbase || (split && !dcls)) return 1;
  group_chain_counts<<<(int)std::min<int64_t>(ceil_div(n_groups + 1, 256), 4096), 256, 0, s>>>(offsets, n_groups, cnt);
  PDSB_LAUNCH_OK();
  count_launch();
  unsigned long long ncls[2] = {(unsigned long long)n_groups, 0};
  if (split) {
    PDSB_CUDA_OK(cudaMemsetAsync(dcls, 0, 2 * sizeof(unsigned long long), s));
    group_class_counts<<<(int)std::min<int64_t>(ceil_div(n_groups, 256), 4096), 256, 0, s>>>(offsets, skip, n_groups, dcls);
    PDSB_LAUNCH_OK();
    count_launch();
    PDSB_CUDA_OK(cudaMemcpyAsync(ncls, dcls, sizeof(ncls), cudaMemcpyDeviceToHost, s));
  }
  size_t tb = 0;
  PDSB_CUDA_OK(cub::DeviceScan::ExclusiveSum(nullptr, tb, cnt, cbase, n_groups + 1, s));
  void* tmp = bag.alloc<unsigned char>(std::max<size_t>(tb, 1));
  if (!tmp) return 1;
  PDSB_CUDA_OK(cub::DeviceScan::ExclusiveSum(tmp, tb, cnt, cbase, n_groups + 1, s));
  int64_t nchains = 0;
  PDSB_CUDA_OK(cudaMemcpyAsync(&nchains, cbase + n_groups, sizeof(int64_t), cudaMemcpyDeviceToHost, s));
  PDSB_CUDA_OK(cudaStreamSynchronize(s));
  if (nchains > 2000000000LL) { set_error("%s: too many rows", what); return 1; }
  if (nchains == 0) return 0;
  int64_t* cgrp = bag.alloc<int64_t>((size_t)nchains);
  if (!cgrp) return 1;
  segment_groups<<<(int)std::min<int64_t>(ceil_div(nchains, 256), 8192), 256, 0, s>>>(cbase, n_groups, nchains, cgrp);
  PDSB_LAUNCH_OK();
  count_launch();
  // (plan, class) of each run: one plan over every group, unless both classes are present and their plans differ
  const bool both = split && ncls[0] > 0 && ncls[1] > 0;
  const int first = split && ncls[0] == 0 ? 1 : 0;
  for (int run = first; run < (both ? 2 : first + 1); ++run) {
    const OnlinePlan& plan = plans[run];
    const ChainTab tab{offsets, cbase, cgrp, skip, both ? run : -1};
    int rc = 0;
#define CASE_D(DD) case DD: rc = run_online<T, DD, false>(plan, X, ldx, y, n, p, d, window, min_rows, 0, lambda, nullptr, 0, coeffs, pred, valid, nchains, tab, n_groups, s); break;
    switch (plan.c == PassC::generic ? 0 : d) {
      CASE_D(1) CASE_D(2) CASE_D(3) CASE_D(4) CASE_D(5) CASE_D(6) CASE_D(7) CASE_D(8) CASE_D(9) CASE_D(10)
      CASE_D(11) CASE_D(12)
      default:
        CASE_D(0)
    }
#undef CASE_D
    if (rc) return rc;
  }
  return 0;
}

}  // namespace

template <typename T>
int grouped_recursive_lin_reg(const T* X, int64_t ldx, const T* y, const int64_t* offsets, const uint8_t* skip,
                              int64_t n_groups, int64_t n, int p, int add_bias, int64_t min_rows, double lambda,
                              T* coeffs, T* pred, uint8_t* valid, cudaStream_t s) {
  return grouped_online_lin_reg<T>(X, ldx, y, offsets, skip, n_groups, n, p, add_bias, 0, min_rows, lambda, coeffs, pred,
                                   valid, s);
}

template <typename T>
int grouped_rolling_lin_reg(const T* X, int64_t ldx, const T* y, const int64_t* offsets, const uint8_t* skip,
                            int64_t n_groups, int64_t n, int p, int add_bias, int64_t window, int64_t min_rows,
                            double lambda, T* coeffs, T* pred, uint8_t* valid, cudaStream_t s) {
  t_last_online_path = 0;
  if (window < 1) { set_error("grouped rolling_lin_reg: window must be >= 1 (got %lld)", (long long)window); return 1; }
  return grouped_online_lin_reg<T>(X, ldx, y, offsets, skip, n_groups, n, p, add_bias, window, min_rows, lambda, coeffs,
                                   pred, valid, s);
}

template int online_lin_reg<float>(const float*, int64_t, const float*, int64_t, int, int, int64_t, int64_t, int,
                                   double, const double*, int64_t, float*, float*, uint8_t*, cudaStream_t);
template int online_lin_reg<double>(const double*, int64_t, const double*, int64_t, int, int, int64_t, int64_t, int,
                                    double, const double*, int64_t, double*, double*, uint8_t*, cudaStream_t);
template int grouped_recursive_lin_reg<float>(const float*, int64_t, const float*, const int64_t*, const uint8_t*, int64_t,
                                              int64_t, int, int, int64_t, double, float*, float*, uint8_t*, cudaStream_t);
template int grouped_recursive_lin_reg<double>(const double*, int64_t, const double*, const int64_t*, const uint8_t*,
                                               int64_t, int64_t, int, int, int64_t, double, double*, double*, uint8_t*,
                                               cudaStream_t);
template int grouped_rolling_lin_reg<float>(const float*, int64_t, const float*, const int64_t*, const uint8_t*, int64_t,
                                            int64_t, int, int, int64_t, int64_t, double, float*, float*, uint8_t*,
                                            cudaStream_t);
template int grouped_rolling_lin_reg<double>(const double*, int64_t, const double*, const int64_t*, const uint8_t*,
                                             int64_t, int64_t, int, int, int64_t, int64_t, double, double*, double*,
                                             uint8_t*, cudaStream_t);

}  // namespace pdsb
