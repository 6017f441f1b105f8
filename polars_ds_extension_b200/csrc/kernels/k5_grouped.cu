// K5 — group_by(seg).agg(pds.lin_reg(...)) as a batched, segmented problem.
//
// In the reference there is no grouped code: Polars calls `_polars_plugin_pl_lr` once per group from its rayon pool
// (SURVEY.md §3.6; /root/reference/src/utils/mod.rs:81-84 "tight group-by loops"; tests/test_linear_exprs.py:918-953).
// Each call packs the group, builds X'X / X'y with a sequential matmul (lr_solvers.rs:186-190) and runs the gated
// QR solve (:329-382).  Here the whole frame stays in HBM in key order and one launch sequence does all groups:
//   pass 0  work list: a group of len rows becomes ceil(len / CHUNK) items of EQUAL size; item -> rows map (one thread per item);
//   pass 1  group moments: one warp per item, taken from a global counter by the warps of a persistent grid; lanes stride
//           rows (coalesced column reads), the (p+2)(p+3)/2 moments live in registers (f32 FMA chains of <= CHUNK/32
//           terms -> f64 warp reduce); item partials are combined in a fixed order -> bit-reproducible whatever warp ran them;
//   pass 2  batched solve: one thread per group on an interleaved (component-major) workspace — shared memory of a
//           32-thread CTA up to ~20 coefficients, global memory (coalesced across groups) above: ridge, rank gate
//           (ln|det| - sum ln diag <= ln tol), pivoted Householder QR (or Cholesky for solver="choleskey"),
//           back-substitution, coordinate descent / NNLS per group.
// HBM-bound: algorithmic bytes per row = (p+1) * s.
#include "../common.h"
#include "../host/host.h"
#include "kernels.h"
#include "k5_solve.h"
#include "glm_links.h"
#include "predict_row.h"

namespace pdsb {

namespace {

// rows per work item: a group of len rows is cut into ceil(len / CHUNK) items of EQUAL size (see item_range); the
// whole-frame caller cuts the frame at CHUNK boundaries
constexpr int CHUNK = 8192;

// rows [r0, r1) of item `item` of group g: the group's rows are dealt EVENLY over its items (rounded up to 128 rows, one
// trip of the register kernel).  Cutting at fixed CHUNK boundaries left a 1e4-row group as 8192 + 1808 rows, and with
// items dealt round-robin over an even number of warps half the warps got only the long ones (56 % of the HBM peak).
__device__ __forceinline__ void item_range(const int64_t* __restrict__ offsets, const int64_t* __restrict__ item_start, int64_t g,
                                           int64_t item, int64_t& r0, int64_t& r1) {
  const int64_t beg = offsets[g], end = offsets[g + 1];
  const int64_t cnt = item_start[g + 1] - item_start[g];
  const int64_t per = (((end - beg) + cnt - 1) / cnt + 127) & ~int64_t(127);
  r0 = min(beg + (item - item_start[g]) * per, end);
  r1 = min(r0 + per, end);
}
// the group of item: item_start[g] <= item < item_start[g + 1]
__device__ __forceinline__ int64_t item_group(const int64_t* __restrict__ item_start, int64_t n_groups, int64_t item) {
  int64_t lo = 0, hi = n_groups;
  while (hi - lo > 1) { int64_t mid = (lo + hi) >> 1; if (item_start[mid] <= item) lo = mid; else hi = mid; }
  return lo;
}

// ---------------- pass 0: work list ----------------
__global__ void count_items_kernel(const int64_t* __restrict__ offsets, int64_t n_groups, int64_t chunk, int64_t* __restrict__ item_start) {
  // item_start[g] = number of chunks of group g (scanned on the host side of this file by a tiny kernel below)
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < n_groups; g += (int64_t)gridDim.x * blockDim.x) {
    int64_t len = offsets[g + 1] - offsets[g];
    item_start[g] = len > 0 ? (len + chunk - 1) / chunk : 1;
  }
}

__global__ void scan_items_kernel(int64_t* __restrict__ item_start, int64_t n_groups) {
  // single block exclusive scan with running carry (n_groups is at most a few million)
  __shared__ int64_t warp_tot[32];
  __shared__ int64_t carry;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (int64_t base = 0; base < n_groups + 1; base += blockDim.x) {
    int64_t i = base + threadIdx.x;
    int64_t v = (i < n_groups) ? item_start[i] : 0;
    int64_t inc = v;
    for (int off = 1; off < 32; off <<= 1) { int64_t y = __shfl_up_sync(0xffffffffu, inc, off); if ((threadIdx.x & 31) >= off) inc += y; }
    if ((threadIdx.x & 31) == 31) warp_tot[threadIdx.x >> 5] = inc;
    __syncthreads();
    int64_t wpre = 0;
    for (int w = 0; w < (int)(threadIdx.x >> 5); ++w) wpre += warp_tot[w];
    int64_t excl = carry + wpre + inc - v;
    __syncthreads();
    if (i <= n_groups) item_start[i] = excl;
    if (threadIdx.x == blockDim.x - 1) carry = excl + v;
    __syncthreads();
  }
}

// ---------------- pass 1: per-(group, chunk) moments ----------------
// Z = [x_0 .. x_{P-1}, y, 1];  Q1 = P + 2 columns; NM = Q1 (Q1+1) / 2 packed upper-triangular moments.
// GROUPED (the grouped path): null rows arrive as NaN and drop out of their group.  The item's rows come from a
// precomputed [n_items][2] array (item_rows_kernel) instead of a 14-step binary search in front of every item, and warps
// take items from a global counter (persistent grid) instead of a fixed stride, so a warp with a short item does not idle
// while its CTA's longest one finishes; together these measured fastest of the four combinations.
// !GROUPED (moments_small, the whole frame): a NaN poisons the moments exactly like in the other moments kernels, and the
// items of the single "group" are dealt at a fixed stride (rows and queue are unused).
// WEIGHTED (the weighted fit, GROUPED only): row weight w joins the finiteness probe, every product is
// fma(w z_i, z_j, acc) in the same lanes, trips and order (so w = 1 gives the unweighted moments bit for bit), the ones
// column carries sum w, and part gains a row NM: the item's kept rows.
template <typename T, int P, bool GROUPED, bool WEIGHTED>
__device__ __forceinline__ void group_moments_body(const T* __restrict__ X, int64_t ldx, const T* __restrict__ y,
                                                   const T* __restrict__ w, const int64_t* __restrict__ offsets,
                                                   const int64_t* __restrict__ item_start, int64_t n_groups,
                                                   int64_t n_items, double* __restrict__ part,
                                                   const int64_t* __restrict__ rows, unsigned long long* __restrict__ queue) {
  constexpr int Q1 = P + 2;
  constexpr int NM = Q1 * (Q1 + 1) / 2;
  const int lane = threadIdx.x & 31;
  const int64_t warp_global = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  auto next_item = [&](int64_t cur) -> int64_t {
    if constexpr (GROUPED) return pop_item(queue);
    else return cur + nwarps;
  };
  for (int64_t item = GROUPED ? next_item(0) : warp_global; item < n_items; item = next_item(item)) {
    int64_t r0, r1;
    if constexpr (GROUPED) {
      r0 = rows[2 * item];
      r1 = rows[2 * item + 1];
    } else {
      item_range(offsets, item_start, item_group(item_start, n_groups, item), item, r0, r1);
    }
    T acc[NM];
#pragma unroll
    for (int k = 0; k < NM; ++k) acc[k] = T(0);
    int kept = 0;                                     // WEIGHTED: this lane's kept rows
    // U rows per lane and trip: all U x (P+1) loads are issued before the first FMA (memory-level parallelism is what
    // this kernel lives on: one row per trip left ~9 loads in flight per warp and 29 % of the HBM roofline)
    constexpr int U = 4;
    for (int64_t r = r0 + lane; r < r1; r += 32 * U) {
      T z[U][Q1];
      T wv[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int64_t rr = r + 32 * u;
        const int64_t rc = rr < r1 ? rr : r;          // clamped address; the row is zeroed below
#pragma unroll
        for (int c = 0; c < P; ++c) z[u][c] = X[(int64_t)c * ldx + rc];
        z[u][P] = y[rc];
        if constexpr (WEIGHTED) wv[u] = w[rc];
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        // null rows arrive as NaN (null_policy="skip"): they drop out of their group -> the whole row becomes 0
        T probe = T(0);
#pragma unroll
        for (int c = 0; c <= P; ++c) probe = fma(z[u][c], T(0), probe);
        if constexpr (WEIGHTED) probe = fma(wv[u], T(0), probe);
        const bool use = (r + 32 * u < r1) && (!GROUPED || probe == T(0));
#pragma unroll
        for (int c = 0; c <= P; ++c) z[u][c] = use ? z[u][c] : T(0);
        z[u][P + 1] = use ? T(1) : T(0);
        if constexpr (WEIGHTED) { wv[u] = use ? wv[u] : T(0); kept += use ? 1 : 0; }
        int k = 0;
#pragma unroll
        for (int i = 0; i < Q1; ++i) {
          const T zi = WEIGHTED ? wv[u] * z[u][i] : z[u][i];
#pragma unroll
          for (int j = i; j < Q1; ++j) { acc[k] = fma(zi, z[u][j], acc[k]); ++k; }
        }
      }
    }
    // (a transpose-reduce in T — NM - NM / 32 shuffles instead of 5 f64 shuffles per value — was measured slower: ptxas
    // then keeps fewer of the U x (P + 1) loads in flight)
#pragma unroll
    for (int k = 0; k < NM; ++k) {
      double v = (double)acc[k];
      for (int off = 16; off; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
      if (lane == 0) part[(size_t)k * n_items + item] = v;
    }
    if constexpr (WEIGHTED) {
      for (int off = 16; off; off >>= 1) kept += __shfl_xor_sync(0xffffffffu, kept, off);
      if (lane == 0) part[(size_t)NM * n_items + item] = (double)kept;
    }
  }
}
template <typename T, int P, bool GROUPED>
__global__ void __launch_bounds__(256)
group_moments_kernel(const T* __restrict__ X, int64_t ldx, const T* __restrict__ y,
                     const int64_t* __restrict__ offsets, const int64_t* __restrict__ item_start,
                     int64_t n_groups, int64_t n_items, double* __restrict__ part /* [NM][n_items] */,
                     const int64_t* __restrict__ rows = nullptr, unsigned long long* __restrict__ queue = nullptr) {
  group_moments_body<T, P, GROUPED, false>(X, ldx, y, nullptr, offsets, item_start, n_groups, n_items, part, rows, queue);
}
// the weighted fit's pass 1 on the work list's rows and queue: part [NM + 1][n_items]
template <typename T, int P>
__global__ void __launch_bounds__(256)
group_wls_moments_kernel(const T* __restrict__ X, int64_t ldx, const T* __restrict__ y, const T* __restrict__ w,
                         int64_t n_items, double* __restrict__ part, const int64_t* __restrict__ rows,
                         unsigned long long* __restrict__ queue) {
  group_moments_body<T, P, true, true>(X, ldx, y, w, nullptr, nullptr, 0, n_items, part, rows, queue);
}

// whole-frame use of the register kernel (moments_small): one "group" = all rows, item i = rows [i CHUNK, (i+1) CHUNK)
__global__ void small_items_kernel(int64_t n, int64_t n_items, int64_t* __restrict__ offsets /* [2] */, int64_t* __restrict__ item_start /* [2] */) {
  if (threadIdx.x == 0 && blockIdx.x == 0) { offsets[0] = 0; offsets[1] = n; item_start[0] = 0; item_start[1] = n_items; }
}
// packed moment k of Z = [x.., y, 1] summed over the items in a fixed order -> M[(i, j)] and M[(j, i)]
__global__ void __launch_bounds__(128) small_reduce_kernel(const double* __restrict__ part, int64_t n_items, int q1, double* __restrict__ M) {
  __shared__ double red[128];
  const int k = blockIdx.x;
  double v = 0.0;
  for (int64_t it = threadIdx.x; it < n_items; it += 128) v += part[(size_t)k * n_items + it];
  red[threadIdx.x] = v;
  __syncthreads();
  for (int off = 64; off; off >>= 1) { if ((int)threadIdx.x < off) red[threadIdx.x] += red[threadIdx.x + off]; __syncthreads(); }
  if (threadIdx.x == 0) {
    int i, j;
    packed_pair(k, q1, i, j);
    M[(size_t)i * q1 + j] = red[0];
    M[(size_t)j * q1 + i] = red[0];
  }
}

// item -> (first row, end row): one thread per item, so that the grouped moments warps never run the binary search
// (14 dependent global loads per item) in front of their loads.  group (nullable): item -> its group, for the predict pass
__global__ void item_rows_kernel(const int64_t* __restrict__ offsets, const int64_t* __restrict__ item_start, int64_t n_groups,
                                 int64_t n_items, int64_t* __restrict__ rows /* [n_items][2] */,
                                 int64_t* __restrict__ group = nullptr) {
  for (int64_t item = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; item < n_items; item += (int64_t)gridDim.x * blockDim.x) {
    const int64_t g = item_group(item_start, n_groups, item);
    int64_t r0, r1;
    item_range(offsets, item_start, g, item, r0, r1);
    rows[2 * item] = r0;
    rows[2 * item + 1] = r1;
    if (group) group[item] = g;
  }
}

// generic-P variant: lanes still stride rows but moments are accumulated through shared memory per warp.
// SHIFT (the mixed model's group pass): every value of [X | y] is taken relative to its group's first row, so a column
// that is constant within a group contributes exact zeros, and no row is dropped (a NaN reaches the moments).
// WEIGHTED (the weighted fit, !SHIFT): the row's weight joins the finiteness test and sits in the tile's padding column
// q1, where tile_triangle_sum takes it as s = fma(w a_i, a_j, s); part gains a row nm, the item's kept rows.
template <typename T, bool SHIFT, bool WEIGHTED = false>
__device__ __forceinline__ void group_moments_generic(const T* __restrict__ X, int64_t ldx, const T* __restrict__ y,
                                                      const int64_t* __restrict__ offsets, const int64_t* __restrict__ item_start,
                                                      int64_t n_groups, int64_t n_items, int p, double* __restrict__ part,
                                                      unsigned char* smem_raw, const T* __restrict__ w = nullptr) {
  const int q1 = p + 2;
  const int nm = q1 * (q1 + 1) / 2;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  T* tile = reinterpret_cast<T*>(smem_raw) + (size_t)wid * 32 * (q1 + 1);   // [32][q1+1]
  const int64_t warp_global = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const int per_lane = (nm + 31) / 32;
  for (int64_t item = warp_global; item < n_items; item += nwarps) {
    const int64_t g = item_group(item_start, n_groups, item);
    int64_t r0, r1;
    item_range(offsets, item_start, g, item, r0, r1);
    double acc[PACKED_ACC];
    for (int k = 0; k < PACKED_ACC; ++k) acc[k] = 0.0;
    int kept = 0;                                     // WEIGHTED: the item's kept rows so far (every lane)
    for (int64_t rb = r0; rb < r1; rb += 32) {
      const int64_t r = rb + lane;
      bool fin = r < r1;
      for (int c = 0; c < q1; ++c) {
        T v = T(0);
        if (r < r1) v = (c < p) ? X[(int64_t)c * ldx + r] : (c == p ? y[r] : T(1));
        if constexpr (SHIFT) {
          const int64_t f = offsets[g];
          if (r < r1 && c <= p) v -= (c < p) ? X[(int64_t)c * ldx + f] : y[f];
        }
        fin = fin && isfinite(v);
        tile[lane * (q1 + 1) + c] = v;
      }
      if constexpr (WEIGHTED) {
        const T wr = r < r1 ? w[r] : T(0);
        fin = fin && isfinite(wr);
        tile[lane * (q1 + 1) + q1] = fin ? wr : T(0);
        kept += __popc(__ballot_sync(0xffffffffu, fin));
      }
      if (!SHIFT && !fin) for (int c = 0; c < q1; ++c) tile[lane * (q1 + 1) + c] = T(0);
      __syncwarp();
      if constexpr (WEIGHTED) tile_triangle_sum(tile, q1 + 1, q1, tile + q1, q1 + 1, acc);
      else tile_triangle_sum(tile, q1 + 1, q1, nullptr, 0, acc);
      __syncwarp();
    }
    for (int m = 0; m < per_lane; ++m) {
      int k = lane + 32 * m;
      if (k < nm) part[(size_t)k * n_items + item] = acc[m];
    }
    if (WEIGHTED && lane == 0) part[(size_t)nm * n_items + item] = (double)kept;
  }
}
template <typename T>
__global__ void __launch_bounds__(128)
group_moments_generic_kernel(const T* __restrict__ X, int64_t ldx, const T* __restrict__ y,
                             const int64_t* __restrict__ offsets, const int64_t* __restrict__ item_start,
                             int64_t n_groups, int64_t n_items, int p, double* __restrict__ part) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  group_moments_generic<T, false>(X, ldx, y, offsets, item_start, n_groups, n_items, p, part, smem_raw);
}
template <typename T>
__global__ void __launch_bounds__(128)
group_wls_moments_generic_kernel(const T* __restrict__ X, int64_t ldx, const T* __restrict__ y, const T* __restrict__ w,
                                 const int64_t* __restrict__ offsets, const int64_t* __restrict__ item_start,
                                 int64_t n_groups, int64_t n_items, int p, double* __restrict__ part) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  group_moments_generic<T, false, true>(X, ldx, y, offsets, item_start, n_groups, n_items, p, part, smem_raw, w);
}
__global__ void __launch_bounds__(128)
group_moments_shifted_kernel(const double* __restrict__ X, int64_t ldx, const double* __restrict__ y,
                             const int64_t* __restrict__ offsets, const int64_t* __restrict__ item_start,
                             int64_t n_groups, int64_t n_items, int p, double* __restrict__ part) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  group_moments_generic<double, true>(X, ldx, y, offsets, item_start, n_groups, n_items, p, part, smem_raw);
}

// ---------------- pass 2: batched solve (group_solve, k5_solve.h) ----------------
// l1 and l2 are the args' own: lin_reg's penalties, 0 for the report's PDSB_METHOD_INV solve
__global__ void __launch_bounds__(128) group_solve_kernel(GroupSolveArgs a) {
  const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= a.n_groups) return;
  group_solve(a, g, a.item_start[g], a.item_start[g + 1], a.l1, a.l2, false);
}
// the multi-target fit: group_solve with t right-hand sides.  A kernel of its own, so that group_solve_kernel keeps its
// compile-time t = 1 and its code
__global__ void __launch_bounds__(128) group_solve_targets_kernel(GroupSolveArgs a, int t) {
  const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= a.n_groups) return;
  group_solve(a, g, a.item_start[g], a.item_start[g + 1], a.l1, a.l2, false, t);
}
// the weighted fit: the "fewer rows than coefficients" gate reads the kept rows of part row nm, not sum w
__global__ void __launch_bounds__(128) group_solve_wls_kernel(GroupSolveArgs a) {
  const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= a.n_groups) return;
  group_solve(a, g, a.item_start[g], a.item_start[g + 1], a.l1, a.l2, false, 1, true);
}

// ---------------- pass 3: segmented predict / residual (lin_reg(return_pred=True).over(key)) ----------------
// pred = [X | 1] beta_g and resid = y - pred for every row of group g, with K4's per-row arithmetic
// (k4_predict.cu::predict_kernel): beta rounded to T, the accumulator starts at the bias (0 without one), one fma per
// feature in column order, resid = y - pred.  A group's pred / resid are therefore bit for bit what pdsb_dev_predict_*
// gives on its rows with the same beta.  valid = 0 for a masked row and for every row of a group whose status is not
// PDSB_OK (its beta reads as 0 there, as K4's does for a gated fit).  One warp per item of the pass-0 work list, taken
// from the queue as in pass 1; the warp puts its group's beta in shared memory once, then streams the item's rows, VEC
// consecutive rows per lane with 16-byte loads where the rows are aligned and one row per lane in the head and tail.
// Bytes per row: (p + 1) s read, 2 s + 1 written.
constexpr int GP_WARPS = 8;     // warps per CTA of the predict pass
constexpr int GP_MAXP = 64;     // the feature limit of grouped_lin_reg

// rows [row, row + VEC), by the rule of predict_row.h.  L: the inverse link.  glm::Gaussian (identity) writes pred and
// resid; glm::Binomial (logistic_reg) writes pred = L::inv(eta), K10's predict_strided rule, and no resid.
template <typename T, int VEC, class L>
__device__ __forceinline__ void predict_rows(const T* __restrict__ X, int64_t ldx, const T* __restrict__ y,
                                             const T* __restrict__ mask, int64_t row, int p, const T* sb, bool ok,
                                             T* __restrict__ pred, T* __restrict__ resid, uint8_t* __restrict__ valid) {
  constexpr bool IDENTITY = std::is_same<L, glm::Gaussian>::value;
  T acc[VEC];
  predict_acc<T, VEC>(sb, p, [&](int c, T (&xv)[VEC]) { load_rows<T, VEC>(X + (int64_t)c * ldx + row, xv); }, acc);
  if constexpr (IDENTITY) {
    T yv[VEC], rv[VEC];
    load_rows<T, VEC>(y + row, yv);
#pragma unroll
    for (int v = 0; v < VEC; ++v) rv[v] = resid_of(yv[v], acc[v]);
    store_rows<T, VEC>(pred + row, acc);
    store_rows<T, VEC>(resid + row, rv);
  } else {
#pragma unroll
    for (int v = 0; v < VEC; ++v) acc[v] = L::inv(acc[v]);
    store_rows<T, VEC>(pred + row, acc);
  }
  T mv[VEC];
  if (mask) load_rows<T, VEC>(mask + row, mv);
  // valid_of's rule, written out: through the helper this instance compiled to different code that ran the C3 predict
  // pass 6 % slower (H100 80GB HBM3, 700 W)
#pragma unroll
  for (int v = 0; v < VEC; ++v) valid[row + v] = (ok && (!mask || mv[v] != T(0))) ? 1 : 0;
}

// L = glm::Binomial: status is not read (every fit counts as OK; a failed logistic fit arrives as NaN beta, so its rows
// come out NaN), y and resid are not touched, and valid comes from the mask alone.
template <typename T, bool VECTOR, class L = glm::Gaussian>
__global__ void __launch_bounds__(GP_WARPS * 32)
group_predict_kernel(const T* __restrict__ X, int64_t ldx, const T* __restrict__ y, const T* __restrict__ mask,
                     const int64_t* __restrict__ rows, const int64_t* __restrict__ group, int64_t n_items, int p,
                     int add_bias, const double* __restrict__ beta, const int* __restrict__ status, T* __restrict__ pred,
                     T* __restrict__ resid, uint8_t* __restrict__ valid, unsigned long long* __restrict__ queue) {
  constexpr bool IDENTITY = std::is_same<L, glm::Gaussian>::value;
  constexpr int VEC = VECTOR ? 16 / sizeof(T) : 1;
  __shared__ T sbeta[GP_WARPS][GP_MAXP + 1];
  const int lane = threadIdx.x & 31;
  T* sb = sbeta[threadIdx.x >> 5];
  const int q = p + (add_bias ? 1 : 0);
  for (int64_t item = pop_item(queue); item < n_items; item = pop_item(queue)) {
    const int64_t r0 = rows[2 * item], r1 = rows[2 * item + 1];
    if (r0 >= r1) continue;                        // an empty group, or an item past the end of the work list
    const int64_t g = group[item];
    const bool ok = !IDENTITY || status[g] == PDSB_OK;
    __syncwarp();                                  // the previous item's reads of sb are done
    for (int i = lane; i <= p; i += 32) sb[i] = staged_beta<T>(beta, (size_t)g * q, i, p, add_bias, ok);
    __syncwarp();
    walk_item_rows<VEC>(r0, r1, [&](int64_t row, auto v) {
      predict_rows<T, decltype(v)::value, L>(X, ldx, y, mask, row, p, sb, ok, pred, resid, valid);
    });
  }
}

template <typename T, int P>
int launch_moments_p(const T* X, int64_t ldx, const T* y, const GroupWork& wl, double* part, cudaStream_t s) {
  // (a 16-byte-load variant of the register kernel — 140 registers, two 16-byte loads per column in flight instead of four
  // 4-byte ones — measured slower and was removed.  So was a bulk-copy staged variant: its 110 accumulator registers left
  // one CTA per SM, and the per-item CTA-wide reduction drained its ring every 16 tiles.)
  auto kern = group_moments_kernel<T, P, true>;
  const int grid = persistent_grid(kern, 256, 0, wl.n_items, 2);
  if (!grid) return 1;
  PDSB_CUDA_OK(cudaMemsetAsync(wl.queue, 0, sizeof(unsigned long long), s));
  kern<<<grid, 256, 0, s>>>(X, ldx, y, nullptr, nullptr, 0, wl.n_items, part, wl.rows, wl.queue);
  PDSB_LAUNCH_OK();
  count_launch();
  return 0;
}

template <typename T, int P>
int launch_wls_moments_p(const T* X, int64_t ldx, const T* y, const T* w, const GroupWork& wl, double* part, cudaStream_t s) {
  auto kern = group_wls_moments_kernel<T, P>;
  const int grid = persistent_grid(kern, 256, 0, wl.n_items, 2);
  if (!grid) return 1;
  PDSB_CUDA_OK(cudaMemsetAsync(wl.queue, 0, sizeof(unsigned long long), s));
  kern<<<grid, 256, 0, s>>>(X, ldx, y, w, wl.n_items, part, wl.rows, wl.queue);
  PDSB_LAUNCH_OK();
  count_launch();
  return 0;
}

// ---------------- autoregression: group_by().agg(query_ar_coeffs(x, lag)) from one column ----------------
// Group g of m rows has the design pl_lr_by sees on its lagged columns materialised per group: target rows t = L .. m-1,
// y_t = x_t, features (x_{t-1}, .., x_{t-L}).  Pass 0 builds the work list on the sliced offsets (max(m - L, 0) rows per
// group), so every item holds the rows it would hold on the materialised columns; ar_rebase_kernel then moves each item
// to its physical rows of x.  A row's lags are the L rows before it, all inside its group.  Pass 1 below gives every row
// to the lane, trip and FMA order of the K5 kernel it would meet on the materialised columns (the register kernel for
// L <= 10, the generic one above), so the partials, and through pass 2 beta and status, are bit for bit pl_lr_by's.
// x is read once: each warp stages a trip's rows plus the L rows before them in shared memory with coalesced loads, and
// every lane takes its lags from there.  Bytes per row: s (+ s for the mask when x has nulls under a fill policy).
template <typename T>
__device__ __forceinline__ T nan_of() { return sizeof(T) == 4 ? (T)__int_as_float(0x7fc00000) : (T)__longlong_as_double(0x7ff8000000000000LL); }

// so[g] = max(m_g - L, 0) target rows, so[n_groups] = 0: scan_items_kernel turns it into the sliced offsets in place
__global__ void ar_lengths_kernel(const int64_t* __restrict__ offsets, int64_t n_groups, int lag, int64_t* __restrict__ so) {
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g <= n_groups; g += (int64_t)gridDim.x * blockDim.x)
    so[g] = g < n_groups ? max(offsets[g + 1] - offsets[g] - lag, (int64_t)0) : 0;
}
// sliced row r of group g is physical row offsets[g] + L + (r - so[g])
__global__ void ar_rebase_kernel(const int64_t* __restrict__ offsets, const int64_t* __restrict__ so,
                                 const int64_t* __restrict__ group, int64_t n_items, int lag, int64_t* __restrict__ rows) {
  for (int64_t item = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; item < n_items; item += (int64_t)gridDim.x * blockDim.x) {
    const int64_t g = group[item], d = offsets[g] + lag - so[g];
    rows[2 * item] += d;
    rows[2 * item + 1] += d;
  }
}

// L = P <= 10: group_moments_kernel<T, P, true>'s rows, trips and arithmetic.  Per 4 x 32-row trip the warp stages rows
// [base - P, base + 128) in `win`; the next trip's loads are issued before this trip's FMAs.  mask (nullable): a row with
// mask 0 gets a NaN target, which is how a null y reaches the K5 kernel.
template <typename T, int P>
__global__ void __launch_bounds__(256)
ar_moments_kernel(const T* __restrict__ x, const T* __restrict__ mask, const int64_t* __restrict__ rows, int64_t n_items,
                  double* __restrict__ part /* [NM][n_items] */, unsigned long long* __restrict__ queue) {
  constexpr int Q1 = P + 2;
  constexpr int NM = Q1 * (Q1 + 1) / 2;
  constexpr int U = 4, TRIP = 32 * U;
  constexpr int J = (TRIP + P + 31) / 32;          // window loads per lane
  __shared__ T win[8][32 * J];
  const int lane = threadIdx.x & 31;
  T* w = win[threadIdx.x >> 5];
  for (int64_t item = pop_item(queue); item < n_items; item = pop_item(queue)) {
    const int64_t r0 = rows[2 * item], r1 = rows[2 * item + 1];
    T acc[NM];
#pragma unroll
    for (int k = 0; k < NM; ++k) acc[k] = T(0);
    T xv[J], mv[U];
    auto load = [&](int64_t base) {
#pragma unroll
      for (int j = 0; j < J; ++j) {
        const int64_t row = base - P + lane + 32 * j;
        xv[j] = row < r1 ? x[row] : T(0);
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int64_t row = base + lane + 32 * u;
        mv[u] = (mask && row < r1) ? mask[row] : T(1);
      }
    };
    if (r0 < r1) load(r0);
    for (int64_t base = r0; base < r1; base += TRIP) {
      __syncwarp();                                 // the previous trip's reads of w are done
#pragma unroll
      for (int j = 0; j < J; ++j) w[lane + 32 * j] = xv[j];
      T mc[U];
#pragma unroll
      for (int u = 0; u < U; ++u) mc[u] = mv[u];
      __syncwarp();
      if (base + TRIP < r1) load(base + TRIP);
      if (base + lane >= r1) continue;              // the lane has no row left (last trip): K5's lane loop has ended
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int o = lane + 32 * u + P;            // the row's place in w; lag c + 1 sits at o - 1 - c
        T z[Q1];
#pragma unroll
        for (int c = 0; c < P; ++c) z[c] = w[o - 1 - c];
        z[P] = mc[u] != T(0) ? w[o] : nan_of<T>();
        T probe = T(0);
#pragma unroll
        for (int c = 0; c <= P; ++c) probe = fma(z[c], T(0), probe);
        const bool use = (base + lane + 32 * u < r1) && probe == T(0);
#pragma unroll
        for (int c = 0; c <= P; ++c) z[c] = use ? z[c] : T(0);
        z[P + 1] = use ? T(1) : T(0);
        int k = 0;
#pragma unroll
        for (int i = 0; i < Q1; ++i)
#pragma unroll
          for (int j = i; j < Q1; ++j) { acc[k] = fma(z[i], z[j], acc[k]); ++k; }
      }
    }
#pragma unroll
    for (int k = 0; k < NM; ++k) {
      double v = (double)acc[k];
      for (int off = 16; off; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
      if (lane == 0) part[(size_t)k * n_items + item] = v;
    }
  }
}

// L > 10: group_moments_generic's 32-row blocks and tile sums.  Per block the warp stages rows [rb - L, rb + 32) in `win`
// and fills the [32][L + 3] tile from there.  Dynamic shared memory: 4 warps x (32 (L + 3) + L + 32) T.
template <typename T>
__global__ void __launch_bounds__(128)
ar_moments_generic_kernel(const T* __restrict__ x, const T* __restrict__ mask, const int64_t* __restrict__ rows,
                          int64_t n_items, int p, double* __restrict__ part, unsigned long long* __restrict__ queue) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const int q1 = p + 2, ld = q1 + 1;
  const int nm = q1 * (q1 + 1) / 2;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  T* tile = reinterpret_cast<T*>(smem_raw) + (size_t)wid * (32 * ld + p + 32);
  T* win = tile + 32 * ld;
  const int per_lane = (nm + 31) / 32;
  for (int64_t item = pop_item(queue); item < n_items; item = pop_item(queue)) {
    const int64_t r0 = rows[2 * item], r1 = rows[2 * item + 1];
    double acc[PACKED_ACC];
    for (int k = 0; k < PACKED_ACC; ++k) acc[k] = 0.0;
    for (int64_t rb = r0; rb < r1; rb += 32) {
      for (int k = lane; k < p + 32; k += 32) {
        const int64_t row = rb - p + k;
        win[k] = row < r1 ? x[row] : T(0);
      }
      __syncwarp();
      const int64_t r = rb + lane;
      bool fin = r < r1;
      const bool ykept = r < r1 && (!mask || mask[r] != T(0));
      for (int c = 0; c < q1; ++c) {
        T v = T(0);
        if (r < r1) v = (c < p) ? win[lane + p - 1 - c] : (c == p ? (ykept ? win[lane + p] : nan_of<T>()) : T(1));
        fin = fin && isfinite(v);
        tile[lane * ld + c] = v;
      }
      if (!fin) for (int c = 0; c < q1; ++c) tile[lane * ld + c] = T(0);
      __syncwarp();
      tile_triangle_sum(tile, ld, q1, nullptr, 0, acc);
      __syncwarp();
    }
    for (int m = 0; m < per_lane; ++m) {
      int k = lane + 32 * m;
      if (k < nm) part[(size_t)k * n_items + item] = acc[m];
    }
  }
}

template <typename T, int P>
int launch_ar_moments_p(const T* x, const T* mask, const GroupWork& wl, double* part, cudaStream_t s) {
  auto kern = ar_moments_kernel<T, P>;
  const int grid = persistent_grid(kern, 256, 0, wl.n_items, 2);
  if (!grid) return 1;
  PDSB_CUDA_OK(cudaMemsetAsync(wl.queue, 0, sizeof(unsigned long long), s));
  kern<<<grid, 256, 0, s>>>(x, mask, wl.rows, wl.n_items, part, wl.queue);
  PDSB_LAUNCH_OK();
  count_launch();
  return 0;
}

}  // namespace

int64_t group_items_bound(int64_t n, int64_t n_groups) { return n_groups + ceil_div(n, (int64_t)CHUNK); }

int build_work_list(const int64_t* offsets, int64_t n_groups, int64_t n, ItemCount count, ItemMaps maps, DevBag& bag,
                    GroupWork& wl, cudaStream_t s) {
  wl = GroupWork{};
  wl.item_start = bag.alloc<int64_t>((size_t)n_groups + 1);
  wl.queue = bag.alloc<unsigned long long>(2);
  if (!wl.item_start || !wl.queue) return 1;
  count_items_kernel<<<(int)std::min<int64_t>(ceil_div(n_groups, 256), 1024), 256, 0, s>>>(offsets, n_groups, CHUNK,
                                                                                         wl.item_start);
  count_launch();
  scan_items_kernel<<<1, 1024, 0, s>>>(wl.item_start, n_groups);
  count_launch();
  PDSB_LAUNCH_OK();
  if (count == ItemCount::EXACT) {
    PDSB_CUDA_OK(cudaMemcpyAsync(&wl.n_items, wl.item_start + n_groups, sizeof(int64_t), cudaMemcpyDeviceToHost, s));
    PDSB_CUDA_OK(cudaStreamSynchronize(s));
  } else {
    wl.n_items = group_items_bound(n, n_groups);
  }
  if (maps == ItemMaps::NONE) return 0;
  // every group has at least one item, so n_items >= n_groups >= 1
  wl.rows = bag.alloc<int64_t>((size_t)wl.n_items * (maps == ItemMaps::ROWS_AND_GROUP ? 3 : 2));
  if (!wl.rows) return 1;
  if (maps == ItemMaps::ROWS_AND_GROUP) wl.group = wl.rows + 2 * wl.n_items;
  item_rows_kernel<<<(int)std::min<int64_t>(ceil_div(wl.n_items, 256), 2048), 256, 0, s>>>(
      offsets, wl.item_start, n_groups, wl.n_items, wl.rows, wl.group);
  PDSB_LAUNCH_OK();
  count_launch();
  return 0;
}

int smem_opt_in(const void* kernel, size_t smem) {
  if (smem > 48 * 1024) PDSB_CUDA_OK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  return 0;
}

int persistent_grid(const void* kernel, int threads, size_t smem, int64_t n_items, int fallback_occ) {
  if (smem_opt_in(kernel, smem)) return 0;
  int occ = fallback_occ;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kernel, threads, smem) != cudaSuccess || occ < 1) {
    (void)cudaGetLastError();
    occ = fallback_occ;
  }
  return (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div(n_items, threads / 32), (int64_t)sm_count() * occ));
}

int launch_group_solve(const GroupSolveArgs& a, cudaStream_t s, int t, bool kept) {
  const int q = a.p + (a.add_bias ? 1 : 0);
  const GroupSolveLaunch L = group_solve_launch(a.p, q, group_solve_nrhs(a.method, q, t), t);
  const int grid = (int)ceil_div(a.n_groups, L.threads);
  if (kept) {
    if (smem_opt_in(group_solve_wls_kernel, L.smem)) return 1;
    group_solve_wls_kernel<<<grid, L.threads, L.smem, s>>>(a);
  } else if (t == 1) {
    if (smem_opt_in(group_solve_kernel, L.smem)) return 1;
    group_solve_kernel<<<grid, L.threads, L.smem, s>>>(a);
  } else {
    if (smem_opt_in(group_solve_targets_kernel, L.smem)) return 1;
    group_solve_targets_kernel<<<grid, L.threads, L.smem, s>>>(a, t);
  }
  PDSB_LAUNCH_OK();
  count_launch();
  return 0;
}

// Moments [X | y | 1]' [X | y | 1] of a whole frame with few features on the register kernel above.  The tensor-core
// kernel pays a fixed cost per 128-row stage whatever the stage holds, while 45..105 FMAs per row fit under the HBM time
// on the FP32 pipes.  f32 chains of CHUNK / 32 rows per
// lane, f64 across lanes and items, fixed order -> reproducible.  Column-major, one target, 1 to 10 features.
bool moments_small_supported(int64_t n, int p, int t, int64_t bstride) {
  return bstride == 0 && t == 1 && p >= 1 && p <= 10 && n >= 1;
}

template <typename T>
int moments_small(const T* X, int64_t ldx, const T* y, int64_t n, int p, double* M, cudaStream_t s) {
  const int q1 = p + 2, nm = q1 * (q1 + 1) / 2;
  const int64_t n_items = ceil_div(n, (int64_t)CHUNK);
  int64_t* meta = nullptr;
  double* part = nullptr;
  if (dev_alloc((void**)&meta, 4 * sizeof(int64_t), s)) return 1;
  if (dev_alloc((void**)&part, (size_t)nm * n_items * sizeof(double), s)) { dev_free(meta, s); return 1; }
  small_items_kernel<<<1, 32, 0, s>>>(n, n_items, meta, meta + 2);
  count_launch();
  int grid = (int)std::min<int64_t>(ceil_div(n_items, (int64_t)8), (int64_t)sm_count() * 16);
  if (grid < 1) grid = 1;
  int rc = 0;
#define CASE_P(PP) case PP: group_moments_kernel<T, PP, false><<<grid, 256, 0, s>>>(X, ldx, y, meta, meta + 2, 1, n_items, part); break;
  switch (p) {
    CASE_P(1) CASE_P(2) CASE_P(3) CASE_P(4) CASE_P(5) CASE_P(6) CASE_P(7) CASE_P(8) CASE_P(9) CASE_P(10)
    default: set_error("small moments: %d features", p); rc = 1;
  }
#undef CASE_P
  if (!rc) {
    cudaError_t e = cudaGetLastError();
    count_launch();
    if (e != cudaSuccess) { set_error("small moments launch failed: %s", cudaGetErrorString(e)); rc = 1; }
  }
  if (!rc) {
    small_reduce_kernel<<<nm, 128, 0, s>>>(part, n_items, q1, M);
    cudaError_t e = cudaGetLastError();
    count_launch();
    if (e != cudaSuccess) { set_error("small moments reduce launch failed: %s", cudaGetErrorString(e)); rc = 1; }
  }
  dev_free(part, s);
  dev_free(meta, s);
  return rc;
}
template int moments_small<float>(const float*, int64_t, const float*, int64_t, int, double*, cudaStream_t);

template <typename T>
int group_moments(const T* X, int64_t ldx, const T* y, const int64_t* offsets, int64_t n_groups, int p,
                  const GroupWork& wl, DevBag& bag, double** part_out, cudaStream_t s) {
  const int q1 = p + 2, nm = q1 * (q1 + 1) / 2;
  double* part = *part_out = bag.alloc<double>((size_t)nm * wl.n_items);
  if (!part) return 1;
#define CASE_P(PP) case PP: return launch_moments_p<T, PP>(X, ldx, y, wl, part, s);
  switch (p) {
    CASE_P(1) CASE_P(2) CASE_P(3) CASE_P(4) CASE_P(5) CASE_P(6) CASE_P(7) CASE_P(8) CASE_P(9) CASE_P(10)
    default: break;
  }
#undef CASE_P
  // four warps' [32][q1 + 1] tiles
  const size_t smem = (size_t)4 * 32 * (q1 + 1) * sizeof(T);
  const int grid = (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div(wl.n_items, 4), (int64_t)sm_count() * 16));
  if (smem_opt_in(group_moments_generic_kernel<T>, smem)) return 1;
  group_moments_generic_kernel<T><<<grid, 128, smem, s>>>(X, ldx, y, offsets, wl.item_start, n_groups, wl.n_items, p, part);
  PDSB_LAUNCH_OK();
  count_launch();
  return 0;
}

template int group_moments<float>(const float*, int64_t, const float*, const int64_t*, int64_t, int, const GroupWork&,
                                  DevBag&, double**, cudaStream_t);
template int group_moments<double>(const double*, int64_t, const double*, const int64_t*, int64_t, int, const GroupWork&,
                                   DevBag&, double**, cudaStream_t);

// pass 2 of a lin_reg fit on the partials of wl: lin_reg's solver settings in o, the workspace from bag; t targets
// (the partials of p + t - 1 features, group_solve), beta [n_groups][t][q]
static int solve_groups(const double* part, const GroupWork& wl, const int64_t* offsets, int64_t n_groups, int p,
                        const pdsb_solve_opts& o, double* beta, int* status, DevBag& bag, cudaStream_t s, int t = 1,
                        bool kept = false) {
  const int q = p + (o.add_bias ? 1 : 0);
  double* ws = nullptr;
  if (!group_solve_launch(p, q, t, t).shared && !(ws = bag.alloc<double>(((size_t)q * q + (size_t)q * t + q) * n_groups)))
    return 1;
  GroupSolveArgs a;
  a.part = part; a.item_start = wl.item_start; a.offsets = offsets; a.n_groups = n_groups; a.n_items = wl.n_items;
  a.p = p; a.add_bias = o.add_bias; a.solver = o.solver; a.l2 = o.l2_reg; a.tol = o.singular_x_tol;
  a.method = o.method; a.positive = o.positive; a.max_iter = o.max_iter; a.l1 = o.l1_reg; a.cd_tol = o.tol;
  a.ws = ws; a.beta = beta; a.status = status;
  return launch_group_solve(a, s, t, kept);
}

template <typename T>
int grouped_lin_reg(const T* X, int64_t ldx, const T* y, const int64_t* offsets, int64_t n_groups, int64_t n,
                    int p, const pdsb_solve_opts& o, double* beta, int* status, cudaStream_t s, DevBag* bag,
                    GroupWork* wl_out) {
  if (n_groups <= 0) return 0;
  if (o.method != PDSB_METHOD_LSTSQ && o.method != PDSB_METHOD_CD && o.method != PDSB_METHOD_NNLS) {
    set_error("grouped lin_reg: method %d is not batched", o.method);
    return 1;
  }
  if (p < 1 || p > 64) { set_error("grouped lin_reg: p=%d not supported (1..64)", p); return 1; }
  DevBag scratch(s);
  GroupWork wl;
  // the item count comes back to the host to size the partials: sized for group_items_bound instead, the fit of one
  // 5e7-row group and 1e5 small groups measured 70 % slower (6.9 -> 11.9 ms, H100 80GB HBM3 at 700 W)
  const ItemMaps maps = wl_out ? ItemMaps::ROWS_AND_GROUP : (p <= 10 ? ItemMaps::ROWS : ItemMaps::NONE);
  if (build_work_list(offsets, n_groups, n, ItemCount::EXACT, maps, bag ? *bag : scratch, wl, s)) return 1;
  if (wl_out) *wl_out = wl;
  double* part = nullptr;
  if (group_moments<T>(X, ldx, y, offsets, n_groups, p, wl, scratch, &part, s)) return 1;
  return solve_groups(part, wl, offsets, n_groups, p, o, beta, status, scratch, s);
}

int group_moments_shifted(const double* X, int64_t ldx, const double* y, const int64_t* offsets, int64_t n_groups, int p,
                          const GroupWork& wl, double* part, cudaStream_t s) {
  if (p < 1 || p > 64) { set_error("group moments: p=%d not supported (1..64)", p); return 1; }
  const int q1 = p + 2;
  const size_t smem = (size_t)4 * 32 * (q1 + 1) * sizeof(double);
  if (smem_opt_in(group_moments_shifted_kernel, smem)) return 1;
  const int grid = (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div(wl.n_items, 4), (int64_t)sm_count() * 16));
  group_moments_shifted_kernel<<<grid, 128, smem, s>>>(X, ldx, y, offsets, wl.item_start, n_groups, wl.n_items, p, part);
  PDSB_LAUNCH_OK();
  count_launch();
  return 0;
}

template <typename T>
int grouped_predict(const T* X, int64_t ldx, const T* y, const int64_t* offsets, int64_t n_groups, int64_t n, int p,
                    int add_bias, const double* beta, const int* status, const T* mask, T* pred, T* resid,
                    uint8_t* valid, cudaStream_t s, int inv_link, const GroupWork* fit_wl) {
  if (n_groups <= 0 || n <= 0) return 0;
  if (p < 1 || p > GP_MAXP) { set_error("grouped predict: p=%d not supported (1..%d)", p, GP_MAXP); return 1; }
  const bool logistic = inv_link == PDSB_GLM_BINOMIAL;
  if (inv_link != PDSB_GLM_GAUSSIAN && !(logistic && sizeof(T) == 8)) { set_error("grouped predict: link %d not supported", inv_link); return 1; }
  if (!X || !offsets || !beta || !pred || !valid || (!logistic && (!y || !status || !resid))) {
    set_error("grouped predict: null argument"); return 1;
  }
  // each row's output depends only on its item's rows and group, so the fit's exact list and the bound one agree
  DevBag bag(s);
  GroupWork own;
  if (!fit_wl && build_work_list(offsets, n_groups, n, ItemCount::BOUND, ItemMaps::ROWS_AND_GROUP, bag, own, s)) return 1;
  const GroupWork& wl = fit_wl ? *fit_wl : own;
  const bool vec_ok = rows_vec_ok<T>(ldx, {X, y, mask, pred, resid});
  auto kern = vec_ok ? group_predict_kernel<T, true> : group_predict_kernel<T, false>;
  if constexpr (sizeof(T) == 8)
    if (logistic) kern = vec_ok ? group_predict_kernel<T, true, glm::Binomial> : group_predict_kernel<T, false, glm::Binomial>;
  const int grid = persistent_grid(kern, GP_WARPS * 32, 0, wl.n_items, 4);
  if (!grid) return 1;
  PDSB_CUDA_OK(cudaMemsetAsync(wl.queue, 0, sizeof(unsigned long long), s));
  kern<<<grid, GP_WARPS * 32, 0, s>>>(X, ldx, y, mask, wl.rows, wl.group, wl.n_items, p, add_bias, beta, status, pred,
                                      resid, valid, wl.queue);
  PDSB_LAUNCH_OK();
  count_launch();
  return 0;
}

template int grouped_predict<float>(const float*, int64_t, const float*, const int64_t*, int64_t, int64_t, int, int,
                                    const double*, const int*, const float*, float*, float*, uint8_t*, cudaStream_t, int,
                                    const GroupWork*);
template int grouped_predict<double>(const double*, int64_t, const double*, const int64_t*, int64_t, int64_t, int, int,
                                     const double*, const int*, const double*, double*, double*, uint8_t*, cudaStream_t,
                                     int, const GroupWork*);

template int grouped_lin_reg<float>(const float*, int64_t, const float*, const int64_t*, int64_t, int64_t, int,
                                    const pdsb_solve_opts&, double*, int*, cudaStream_t, DevBag*, GroupWork*);
template int grouped_lin_reg<double>(const double*, int64_t, const double*, const int64_t*, int64_t, int64_t, int,
                                     const pdsb_solve_opts&, double*, int*, cudaStream_t, DevBag*, GroupWork*);

// The weighted fit: grouped_lin_reg's work list, pass 1 with the row weights (group_wls_moments_kernel up to 10
// features, group_wls_moments_generic_kernel above; part [nm + 1][n_items], the last row the kept rows), and pass 2 with
// the row-count gate on those kept rows.  Same launches as grouped_lin_reg.  Bytes per row: (p + 2) s.
template <typename T>
int grouped_wls_lin_reg(const T* X, int64_t ldx, const T* y, const T* w, const int64_t* offsets, int64_t n_groups,
                        int64_t n, int p, const pdsb_solve_opts& o, double* beta, int* status, cudaStream_t s,
                        DevBag* bag, GroupWork* wl_out) {
  if (n_groups <= 0) return 0;
  if (o.method != PDSB_METHOD_LSTSQ) { set_error("grouped weighted lin_reg: method %d is not batched", o.method); return 1; }
  if (p < 1 || p > 64) { set_error("grouped weighted lin_reg: p=%d not supported (1..64)", p); return 1; }
  DevBag scratch(s);
  GroupWork wl;
  const ItemMaps maps = wl_out ? ItemMaps::ROWS_AND_GROUP : (p <= 10 ? ItemMaps::ROWS : ItemMaps::NONE);
  if (build_work_list(offsets, n_groups, n, ItemCount::EXACT, maps, bag ? *bag : scratch, wl, s)) return 1;
  if (wl_out) *wl_out = wl;
  const int q1 = p + 2, nm = q1 * (q1 + 1) / 2;
  double* part = scratch.alloc<double>((size_t)(nm + 1) * wl.n_items);
  if (!part) return 1;
#define CASE_P(PP) case PP: \
    if (launch_wls_moments_p<T, PP>(X, ldx, y, w, wl, part, s)) return 1; \
    return solve_groups(part, wl, offsets, n_groups, p, o, beta, status, scratch, s, 1, true);
  switch (p) {
    CASE_P(1) CASE_P(2) CASE_P(3) CASE_P(4) CASE_P(5) CASE_P(6) CASE_P(7) CASE_P(8) CASE_P(9) CASE_P(10)
    default: break;
  }
#undef CASE_P
  const size_t smem = (size_t)4 * 32 * (q1 + 1) * sizeof(T);
  const int grid = (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div(wl.n_items, 4), (int64_t)sm_count() * 16));
  if (smem_opt_in(group_wls_moments_generic_kernel<T>, smem)) return 1;
  group_wls_moments_generic_kernel<T><<<grid, 128, smem, s>>>(X, ldx, y, w, offsets, wl.item_start, n_groups, wl.n_items,
                                                               p, part);
  PDSB_LAUNCH_OK();
  count_launch();
  return solve_groups(part, wl, offsets, n_groups, p, o, beta, status, scratch, s, 1, true);
}

template int grouped_wls_lin_reg<float>(const float*, int64_t, const float*, const float*, const int64_t*, int64_t,
                                        int64_t, int, const pdsb_solve_opts&, double*, int*, cudaStream_t, DevBag*,
                                        GroupWork*);
template int grouped_wls_lin_reg<double>(const double*, int64_t, const double*, const double*, const int64_t*, int64_t,
                                         int64_t, int, const pdsb_solve_opts&, double*, int*, cudaStream_t, DevBag*,
                                         GroupWork*);

// The multi-target fit on Z = [y_0 .. y_{t-1} | x_0 .. x_{p-1}] (one leading dimension): pass 1 is K5's moments pass on
// the p + t - 1 columns from y_1 as "X" and y_0 as "y", so the packed moments of [y_1 .. y_{t-1}, x.., y_0, 1] hold X'X,
// X'y_c for every target and the row count (and t (t - 1) / 2 Y'Y entries nobody reads).  Every moment is its own FMA
// chain over the item's rows in the same order wherever its column sits, and fma(a, b, c) == fma(b, a, c), so target c's
// moments are bit for bit grouped_lin_reg's on [x | y_c] whenever both meet the same kernel variant (the register kernel
// up to 10 "features", the tile kernel above), and pass 2 solves them as grouped_lin_reg does.  A row with a NaN / inf in
// any column drops out for every target.
template <typename T>
int grouped_lin_reg_multi(const T* Z, int64_t ld, int t, int p, const int64_t* offsets, int64_t n_groups, int64_t n,
                          const pdsb_solve_opts& o, double* beta, int* status, cudaStream_t s) {
  if (n_groups <= 0) return 0;
  if (o.method != PDSB_METHOD_LSTSQ) { set_error("grouped multi-target lin_reg: method %d is not batched", o.method); return 1; }
  if (t < 1 || p < 1 || p + t > 65) {
    set_error("grouped multi-target lin_reg: %d targets and %d features; the batched fit takes 1 to 65 targets and "
              "features together, at least one of each (use the per-group loop)", t, p);
    return 1;
  }
  const int pf = p + t - 1;          // the moments pass's "features"
  DevBag scratch(s);
  GroupWork wl;
  if (build_work_list(offsets, n_groups, n, ItemCount::EXACT, pf <= 10 ? ItemMaps::ROWS : ItemMaps::NONE, scratch, wl, s))
    return 1;
  double* part = nullptr;
  if (group_moments<T>(Z + ld, ld, Z, offsets, n_groups, pf, wl, scratch, &part, s)) return 1;
  return solve_groups(part, wl, offsets, n_groups, p, o, beta, status, scratch, s, t);
}

template int grouped_lin_reg_multi<float>(const float*, int64_t, int, int, const int64_t*, int64_t, int64_t,
                                          const pdsb_solve_opts&, double*, int*, cudaStream_t);
template int grouped_lin_reg_multi<double>(const double*, int64_t, int, int, const int64_t*, int64_t, int64_t,
                                           const pdsb_solve_opts&, double*, int*, cudaStream_t);

template <typename T>
int grouped_ar_lin_reg(const T* x, const T* mask, const int64_t* offsets, int64_t n_groups, int64_t n, int lag,
                       const pdsb_solve_opts& o, double* beta, int* status, cudaStream_t s) {
  if (n_groups <= 0) return 0;
  if (o.method != PDSB_METHOD_LSTSQ && o.method != PDSB_METHOD_CD && o.method != PDSB_METHOD_NNLS) {
    set_error("grouped AR: method %d is not batched", o.method);
    return 1;
  }
  if (lag < 1 || lag > 64) { set_error("grouped AR: lag=%d not supported (1..64)", lag); return 1; }
  const int p = lag, q1 = p + 2, nm = q1 * (q1 + 1) / 2;
  DevBag scratch(s);
  int64_t* so = scratch.alloc<int64_t>((size_t)n_groups + 1);
  if (!so) return 1;
  ar_lengths_kernel<<<(int)std::min<int64_t>(ceil_div(n_groups + 1, 256), 1024), 256, 0, s>>>(offsets, n_groups, lag, so);
  count_launch();
  scan_items_kernel<<<1, 1024, 0, s>>>(so, n_groups);
  count_launch();
  PDSB_LAUNCH_OK();
  GroupWork wl;
  if (build_work_list(so, n_groups, n, ItemCount::EXACT, ItemMaps::ROWS_AND_GROUP, scratch, wl, s)) return 1;
  ar_rebase_kernel<<<(int)std::min<int64_t>(ceil_div(wl.n_items, 256), 2048), 256, 0, s>>>(offsets, so, wl.group,
                                                                                         wl.n_items, lag, wl.rows);
  PDSB_LAUNCH_OK();
  count_launch();
  double* part = scratch.alloc<double>((size_t)nm * wl.n_items);
  if (!part) return 1;
  int rc = -1;
#define CASE_P(PP) case PP: rc = launch_ar_moments_p<T, PP>(x, mask, wl, part, s); break;
  switch (p) {
    CASE_P(1) CASE_P(2) CASE_P(3) CASE_P(4) CASE_P(5) CASE_P(6) CASE_P(7) CASE_P(8) CASE_P(9) CASE_P(10)
    default: break;
  }
#undef CASE_P
  if (rc > 0) return 1;
  if (rc < 0) {
    const size_t smem = (size_t)4 * (32 * (q1 + 1) + p + 32) * sizeof(T);
    auto kern = ar_moments_generic_kernel<T>;
    const int grid = persistent_grid(kern, 128, smem, wl.n_items, 4);
    if (!grid) return 1;
    PDSB_CUDA_OK(cudaMemsetAsync(wl.queue, 0, sizeof(unsigned long long), s));
    kern<<<grid, 128, smem, s>>>(x, mask, wl.rows, wl.n_items, p, part, wl.queue);
    PDSB_LAUNCH_OK();
    count_launch();
  }
  return solve_groups(part, wl, so, n_groups, p, o, beta, status, scratch, s);
}

template int grouped_ar_lin_reg<float>(const float*, const float*, const int64_t*, int64_t, int64_t, int,
                                       const pdsb_solve_opts&, double*, int*, cudaStream_t);
template int grouped_ar_lin_reg<double>(const double*, const double*, const int64_t*, int64_t, int64_t, int,
                                        const pdsb_solve_opts&, double*, int*, cudaStream_t);

}  // namespace pdsb
