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
constexpr int GEN_ACC = 70;   // moments per lane of the generic-p kernel: (p+2)(p+3)/2 <= 2240 -> p <= 64

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
template <typename T, int P, bool GROUPED>
__global__ void __launch_bounds__(256)
group_moments_kernel(const T* __restrict__ X, int64_t ldx, const T* __restrict__ y,
                     const int64_t* __restrict__ offsets, const int64_t* __restrict__ item_start,
                     int64_t n_groups, int64_t n_items, double* __restrict__ part /* [NM][n_items] */,
                     const int64_t* __restrict__ rows = nullptr, unsigned long long* __restrict__ queue = nullptr) {
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
    // U rows per lane and trip: all U x (P+1) loads are issued before the first FMA (memory-level parallelism is what
    // this kernel lives on: one row per trip left ~9 loads in flight per warp and 29 % of the HBM roofline)
    constexpr int U = 4;
    for (int64_t r = r0 + lane; r < r1; r += 32 * U) {
      T z[U][Q1];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int64_t rr = r + 32 * u;
        const int64_t rc = rr < r1 ? rr : r;          // clamped address; the row is zeroed below
#pragma unroll
        for (int c = 0; c < P; ++c) z[u][c] = X[(int64_t)c * ldx + rc];
        z[u][P] = y[rc];
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        // null rows arrive as NaN (null_policy="skip"): they drop out of their group -> the whole row becomes 0
        T probe = T(0);
#pragma unroll
        for (int c = 0; c <= P; ++c) probe = fma(z[u][c], T(0), probe);
        const bool use = (r + 32 * u < r1) && (!GROUPED || probe == T(0));
#pragma unroll
        for (int c = 0; c <= P; ++c) z[u][c] = use ? z[u][c] : T(0);
        z[u][P + 1] = use ? T(1) : T(0);
        int k = 0;
#pragma unroll
        for (int i = 0; i < Q1; ++i)
#pragma unroll
          for (int j = i; j < Q1; ++j) { acc[k] = fma(z[u][i], z[u][j], acc[k]); ++k; }
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
  }
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
    int i = 0, rem = k;
    while (rem >= q1 - i) { rem -= q1 - i; ++i; }
    const int j = i + rem;
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
template <typename T, bool SHIFT>
__device__ __forceinline__ void group_moments_generic(const T* __restrict__ X, int64_t ldx, const T* __restrict__ y,
                                                      const int64_t* __restrict__ offsets, const int64_t* __restrict__ item_start,
                                                      int64_t n_groups, int64_t n_items, int p, double* __restrict__ part,
                                                      unsigned char* smem_raw) {
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
    double acc[GEN_ACC];   // supports nm <= 32 * GEN_ACC (p <= 64)
    for (int k = 0; k < GEN_ACC; ++k) acc[k] = 0.0;
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
      if (!SHIFT && !fin) for (int c = 0; c < q1; ++c) tile[lane * (q1 + 1) + c] = T(0);
      __syncwarp();
      for (int m = 0; m < per_lane; ++m) {
        int k = lane + 32 * m;
        if (k < nm) {
          int i = 0, rem = k;
          while (rem >= q1 - i) { rem -= q1 - i; ++i; }
          int j = i + rem;
          T s = T(0);
          for (int rr = 0; rr < 32; ++rr) s = fma(tile[rr * (q1 + 1) + i], tile[rr * (q1 + 1) + j], s);
          acc[m] += (double)s;
        }
      }
      __syncwarp();
    }
    for (int m = 0; m < per_lane; ++m) {
      int k = lane + 32 * m;
      if (k < nm) part[(size_t)k * n_items + item] = acc[m];
    }
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
__global__ void __launch_bounds__(128)
group_moments_shifted_kernel(const double* __restrict__ X, int64_t ldx, const double* __restrict__ y,
                             const int64_t* __restrict__ offsets, const int64_t* __restrict__ item_start,
                             int64_t n_groups, int64_t n_items, int p, double* __restrict__ part) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  group_moments_generic<double, true>(X, ldx, y, offsets, item_start, n_groups, n_items, p, part, smem_raw);
}

// ---------------- pass 2: batched solve (group_solve, k5_solve.h) ----------------
__global__ void __launch_bounds__(128) group_solve_kernel(GroupSolveArgs a) {
  const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= a.n_groups) return;
  group_solve(a, g, a.item_start[g], a.item_start[g + 1], a.l1, a.l2, false);
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
    // rows [a0, a1) as whole VEC-row vectors from aligned addresses; the fewer than VEC rows on either side one per lane
    const int64_t a0 = min((r0 + VEC - 1) / VEC * VEC, r1);
    const int64_t a1 = max(r1 / VEC * VEC, a0);
    for (int64_t r = a0 + (int64_t)lane * VEC; r < a1; r += 32 * VEC)
      predict_rows<T, VEC, L>(X, ldx, y, mask, r, p, sb, ok, pred, resid, valid);
    const int nh = (int)(a0 - r0);
    if (lane < nh) predict_rows<T, 1, L>(X, ldx, y, mask, r0 + lane, p, sb, ok, pred, resid, valid);
    else if (lane - nh < r1 - a1) predict_rows<T, 1, L>(X, ldx, y, mask, a1 + (lane - nh), p, sb, ok, pred, resid, valid);
  }
}

template <typename T, int P>
int launch_moments_p(const T* X, int64_t ldx, const T* y, const int64_t* offsets, const int64_t* item_start,
                     int64_t n_groups, int64_t n_items, double* part, cudaStream_t s) {
  // (a 16-byte-load variant of the register kernel — 140 registers, two 16-byte loads per column in flight instead of four
  // 4-byte ones — measured slower and was removed.  So was a bulk-copy staged variant: its 110 accumulator registers left
  // one CTA per SM, and the per-item CTA-wide reduction drained its ring every 16 tiles.)
  int64_t* rows = nullptr;
  unsigned long long* queue = nullptr;
  if (dev_alloc((void**)&rows, (size_t)n_items * 2 * sizeof(int64_t), s)) return 1;
  item_rows_kernel<<<(int)std::min<int64_t>(ceil_div(n_items, 256), 2048), 256, 0, s>>>(offsets, item_start, n_groups, n_items, rows);
  count_launch();
  if (dev_alloc((void**)&queue, sizeof(unsigned long long), s)) { dev_free(rows, s); return 1; }
  PDSB_CUDA_OK(cudaMemsetAsync(queue, 0, sizeof(unsigned long long), s));
  // persistent grid: exactly the resident CTAs
  auto kern = group_moments_kernel<T, P, true>;
  int occ = 2;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, 256, 0) != cudaSuccess || occ < 1) { (void)cudaGetLastError(); occ = 2; }
  int grid = (int)std::min<int64_t>(ceil_div(n_items, (int64_t)8), (int64_t)sm_count() * occ);
  if (grid < 1) grid = 1;
  kern<<<grid, 256, 0, s>>>(X, ldx, y, offsets, item_start, n_groups, n_items, part, rows, queue);
  dev_free(rows, s);
  dev_free(queue, s);
  PDSB_LAUNCH_OK();
  count_launch();
  return 0;
}

}  // namespace

// Pass 0: item_start [n_groups + 1] and, with rows, each of n_items items' row range [n_items][2] and, with group (which
// needs rows), its group [n_items].  For n_items = group_items_bound(n, n_groups) nothing has to come back to the host:
// the items past the real count lie after the last group's rows, so they are empty and their partials are zeros that no
// group reads.
int work_list(const int64_t* offsets, int64_t n_groups, int64_t n_items, int64_t* item_start, int64_t* rows,
              int64_t* group, cudaStream_t s) {
  count_items_kernel<<<(int)std::min<int64_t>(ceil_div(n_groups, 256), 1024), 256, 0, s>>>(offsets, n_groups, CHUNK, item_start);
  count_launch();
  scan_items_kernel<<<1, 1024, 0, s>>>(item_start, n_groups);
  count_launch();
  if (rows) {
    item_rows_kernel<<<(int)std::min<int64_t>(ceil_div(n_items, 256), 2048), 256, 0, s>>>(offsets, item_start, n_groups,
                                                                                        n_items, rows, group);
    count_launch();
  }
  PDSB_LAUNCH_OK();
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
int grouped_lin_reg(const T* X, int64_t ldx, const T* y, const int64_t* offsets, int64_t n_groups, int64_t n,
                    int p, const pdsb_solve_opts& o, double* beta, int* status, cudaStream_t s) {
  if (n_groups <= 0) return 0;
  if (o.method != PDSB_METHOD_LSTSQ && o.method != PDSB_METHOD_CD && o.method != PDSB_METHOD_NNLS) {
    set_error("grouped lin_reg: method %d is not batched", o.method);
    return 1;
  }
  const int q = p + (o.add_bias ? 1 : 0);
  if (p < 1 || p > 64) { set_error("grouped lin_reg: p=%d not supported (1..64)", p); return 1; }
  const int q1 = p + 2, nm = q1 * (q1 + 1) / 2;
  // the item count comes back to the host to size the partials: sized for group_items_bound instead, the fit of one
  // 5e7-row group and 1e5 small groups measured 70 % slower (6.9 -> 11.9 ms, H100 80GB HBM3 at 700 W)
  int64_t* item_start = nullptr;
  if (dev_alloc((void**)&item_start, (size_t)(n_groups + 1) * sizeof(int64_t), s)) return 1;
  if (work_list(offsets, n_groups, 0, item_start, nullptr, nullptr, s)) { dev_free(item_start, s); return 1; }
  int64_t n_items = 0;
  PDSB_CUDA_OK(cudaMemcpyAsync(&n_items, item_start + n_groups, sizeof(int64_t), cudaMemcpyDeviceToHost, s));
  PDSB_CUDA_OK(cudaStreamSynchronize(s));
  double* part = nullptr;
  if (dev_alloc((void**)&part, (size_t)nm * n_items * sizeof(double), s)) { dev_free(item_start, s); return 1; }
  int rc = 0;
#define CASE_P(PP) case PP: rc = launch_moments_p<T, PP>(X, ldx, y, offsets, item_start, n_groups, n_items, part, s); break;
  switch (p) {
    CASE_P(1) CASE_P(2) CASE_P(3) CASE_P(4) CASE_P(5) CASE_P(6) CASE_P(7) CASE_P(8) CASE_P(9) CASE_P(10)
    default: {
      size_t smem = (size_t)4 * 32 * (q1 + 1) * sizeof(T);
      int grid = (int)std::min<int64_t>(ceil_div(n_items, 4), (int64_t)sm_count() * 16);
      if (grid < 1) grid = 1;
      group_moments_generic_kernel<T><<<grid, 128, smem, s>>>(X, ldx, y, offsets, item_start, n_groups, n_items, p, part);
      cudaError_t e = cudaGetLastError();
      count_launch();
      if (e != cudaSuccess) { set_error("group moments launch failed: %s", cudaGetErrorString(e)); rc = 1; }
    }
  }
#undef CASE_P
  double* ws = nullptr;
  const GroupSolveLaunch L = group_solve_launch(p, q);
  if (!rc && !L.shared && dev_alloc((void**)&ws, ((size_t)q * q + 2 * q) * sizeof(double) * n_groups, s)) rc = 1;
  if (!rc) {
    GroupSolveArgs a;
    a.part = part; a.item_start = item_start; a.offsets = offsets; a.n_groups = n_groups; a.n_items = n_items;
    a.p = p; a.add_bias = o.add_bias; a.solver = o.solver; a.l2 = o.l2_reg; a.tol = o.singular_x_tol;
    a.method = o.method; a.positive = o.positive; a.max_iter = o.max_iter; a.l1 = o.l1_reg; a.cd_tol = o.tol;
    a.ws = ws; a.beta = beta; a.status = status;
    if (L.smem > 48 * 1024) PDSB_CUDA_OK(cudaFuncSetAttribute(group_solve_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)L.smem));
    group_solve_kernel<<<(int)ceil_div(n_groups, L.threads), L.threads, L.smem, s>>>(a);
    cudaError_t e = cudaGetLastError();
    count_launch();
    if (e != cudaSuccess) { set_error("group solve launch failed: %s", cudaGetErrorString(e)); rc = 1; }
  }
  dev_free(ws, s);
  dev_free(part, s);
  dev_free(item_start, s);
  return rc;
}

int64_t group_items_bound(int64_t n, int64_t n_groups) { return n_groups + ceil_div(n, (int64_t)CHUNK); }

int group_moments_shifted(const double* X, int64_t ldx, const double* y, const int64_t* offsets, int64_t n_groups,
                          int64_t n, int p, int64_t* item_start, double* part, cudaStream_t s) {
  if (p < 1 || p > 64) { set_error("group moments: p=%d not supported (1..64)", p); return 1; }
  const int64_t n_items = group_items_bound(n, n_groups);
  if (work_list(offsets, n_groups, n_items, item_start, nullptr, nullptr, s)) return 1;
  const int q1 = p + 2;
  const size_t smem = (size_t)4 * 32 * (q1 + 1) * sizeof(double);
  if (smem > 48 * 1024)
    PDSB_CUDA_OK(cudaFuncSetAttribute(group_moments_shifted_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const int grid = (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div(n_items, 4), (int64_t)sm_count() * 16));
  group_moments_shifted_kernel<<<grid, 128, smem, s>>>(X, ldx, y, offsets, item_start, n_groups, n_items, p, part);
  PDSB_LAUNCH_OK();
  count_launch();
  return 0;
}

// The work list is rebuilt here from the offsets, so the entry stands alone.
template <typename T>
int grouped_predict(const T* X, int64_t ldx, const T* y, const int64_t* offsets, int64_t n_groups, int64_t n, int p,
                    int add_bias, const double* beta, const int* status, const T* mask, T* pred, T* resid,
                    uint8_t* valid, cudaStream_t s, int inv_link) {
  if (n_groups <= 0 || n <= 0) return 0;
  if (p < 1 || p > GP_MAXP) { set_error("grouped predict: p=%d not supported (1..%d)", p, GP_MAXP); return 1; }
  const bool logistic = inv_link == PDSB_GLM_BINOMIAL;
  if (inv_link != PDSB_GLM_GAUSSIAN && !(logistic && sizeof(T) == 8)) { set_error("grouped predict: link %d not supported", inv_link); return 1; }
  if (!X || !offsets || !beta || !pred || !valid || (!logistic && (!y || !status || !resid))) {
    set_error("grouped predict: null argument"); return 1;
  }
  const int64_t n_items = group_items_bound(n, n_groups);
  int64_t* item_start = nullptr;
  int64_t* rows = nullptr;
  unsigned long long* queue = nullptr;
  if (dev_alloc((void**)&item_start, (size_t)(n_groups + 1) * sizeof(int64_t), s)) return 1;
  if (dev_alloc((void**)&rows, (size_t)n_items * 3 * sizeof(int64_t), s)) { dev_free(item_start, s); return 1; }
  if (dev_alloc((void**)&queue, sizeof(unsigned long long), s)) { dev_free(rows, s); dev_free(item_start, s); return 1; }
  int64_t* group = rows + 2 * n_items;
  int rc = work_list(offsets, n_groups, n_items, item_start, rows, group, s);
  if (!rc) {
    cudaError_t e = cudaMemsetAsync(queue, 0, sizeof(unsigned long long), s);
    if (e == cudaSuccess) {
      constexpr int VEC = 16 / sizeof(T);
      auto aligned = [&](const void* ptr) { return !ptr || (reinterpret_cast<uintptr_t>(ptr) & 15) == 0; };
      const bool vec_ok = aligned(X) && aligned(y) && aligned(mask) && aligned(pred) && aligned(resid) && ldx % VEC == 0;
      auto kern = vec_ok ? group_predict_kernel<T, true> : group_predict_kernel<T, false>;
      if constexpr (sizeof(T) == 8)
        if (logistic) kern = vec_ok ? group_predict_kernel<T, true, glm::Binomial> : group_predict_kernel<T, false, glm::Binomial>;
      int occ = 4;
      if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, GP_WARPS * 32, 0) != cudaSuccess || occ < 1) { (void)cudaGetLastError(); occ = 4; }
      const int grid = (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div(n_items, GP_WARPS), (int64_t)sm_count() * occ));
      kern<<<grid, GP_WARPS * 32, 0, s>>>(X, ldx, y, mask, rows, group, n_items, p, add_bias, beta, status, pred, resid, valid, queue);
      e = cudaGetLastError();
      count_launch();
    }
    if (e != cudaSuccess) { set_error("grouped predict launch failed: %s", cudaGetErrorString(e)); rc = 1; }
  }
  dev_free(queue, s);
  dev_free(rows, s);
  dev_free(item_start, s);
  return rc;
}

template int grouped_predict<float>(const float*, int64_t, const float*, const int64_t*, int64_t, int64_t, int, int,
                                    const double*, const int*, const float*, float*, float*, uint8_t*, cudaStream_t, int);
template int grouped_predict<double>(const double*, int64_t, const double*, const int64_t*, int64_t, int64_t, int, int,
                                     const double*, const int*, const double*, double*, double*, uint8_t*, cudaStream_t,
                                     int);

template int grouped_lin_reg<float>(const float*, int64_t, const float*, const int64_t*, int64_t, int64_t, int,
                                    const pdsb_solve_opts&, double*, int*, cudaStream_t);
template int grouped_lin_reg<double>(const double*, int64_t, const double*, const int64_t*, int64_t, int64_t, int,
                                     const pdsb_solve_opts&, double*, int*, cudaStream_t);

}  // namespace pdsb
