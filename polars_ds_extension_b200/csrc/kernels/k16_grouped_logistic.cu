// K16 — group_by(key).agg(pds.logistic_reg(...)) and pds.logistic_reg(..., return_pred=True).over(key): every group's
// Newton / IRLS fit in one launch sequence.
//
// Polars runs these as one pl_logistic_coeffs / pl_logistic_pred call per group, and each call is host_logistic
// (csrc/host/lr_host.cc): a host-driven loop that pays two device -> host copies and two synchronises per iteration.
// Here every group runs host_logistic's control flow on its own state, in lockstep:
//   once      K5's work list (equal items of <= 8192 rows per group, item -> rows, item -> group), and every group's
//             state: beta = beta_prev = 0, cost_prev = inf, no halvings, status "running";
//   pass A    fused row pass and weighted moments.  Warps of a persistent grid take items from a counter.  An item of a
//             finished group is dropped without reading a row; otherwise the warp stages its group's beta once and,
//             per row, computes eta, mu, w and z by K11's rule (logistic_rows.h) and accumulates in f64
//             sum w a_i a_j over the packed upper triangle of [X | z | 1], the log-loss and the kept-row count.
//             w and z never reach memory: (p + 1) * 8 bytes per row (+ 8 with a mask), where the single-fit path moves
//             about (2p + 6) * 8 (K11 reads X, y and writes w, z; K2a reads X, z, w).  A register kernel for p <= 10,
//             a shared-memory tile up to p = 64, as K5 pass 1;
//   pass B0   (only when some group has more than one item) the item partials of each running group summed in item
//             order into its first item's column, one thread per (partial, group);
//   pass B    one thread per running group: cost, step halving, gradient and stopping test from the summed moments,
//             then K5's solve (group_solve) for the next beta; it counts the groups still running.
// The host reads that count (4 bytes) after every iteration and stops at 0 or after max_iter iterations: one
// synchronise per iteration whatever the group count.
// Reproducible: a row's lane is fixed relative to its item's first row, items are fixed by the group's own length, and
// partials are combined in a fixed order, so a group's result is bit for bit the same run to run and whichever other
// groups share the call.
//
// GLM.fit_by (grouped_glm) runs every group's faer_irls on the same passes: pass A takes the family's row rule
// (GlmRows<L>, logistic_rows.h; the first iteration's instance starts from y and the group's mean of y, which one pass
// over y computes once per call), and pass B is glm_step_kernel: the finiteness test, the QR solve and the
// max |beta - beta_new| < tol test.
#include <cfloat>
#include <cmath>
#include "../common.h"
#include "../host/host.h"
#include "kernels.h"
#include "k5_solve.h"
#include "logistic_rows.h"

namespace pdsb {

namespace {

using glm::LogisticRows;

// a group still iterating carries MAX_ITER: when the iterations run out, that is its status
constexpr int RUNNING = PDSB_LOGISTIC_MAX_ITER;
static_assert(PDSB_GLM_MAX_ITER == RUNNING, "the GLM fit shares the logistic fit's running mark");
constexpr int GEN_WARPS = 4;       // warps per CTA of the generic-p pass A

// ---------------- once per call ----------------
__global__ void logistic_init_kernel(int64_t n_groups, int q, double* __restrict__ beta, double* __restrict__ best,
                                     double* __restrict__ cost_prev, int* __restrict__ halvings, int* __restrict__ status) {
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < n_groups; g += (int64_t)gridDim.x * blockDim.x) {
    for (int j = 0; j < q; ++j) { beta[(size_t)g * q + j] = 0.0; best[(size_t)g * q + j] = 0.0; }
    cost_prev[g] = INFINITY;
    halvings[g] = 0;
    status[g] = RUNNING;
  }
}

// ---------------- pass A: fused row pass + weighted moments, p <= 10 (registers) ----------------
// part [(NM + 2)][n_items]: the NM packed moments of [X | z | 1] weighted by w, then the loss, then the kept rows.
// U rows per lane and trip; fewer for larger P so that the NM + 2 f64 accumulators and the loads stay in registers.
template <int P, class R = LogisticRows, bool INIT = false>
__global__ void __launch_bounds__(256)
logistic_moments_kernel(const double* __restrict__ X, int64_t ldx, const double* __restrict__ y,
                        const double* __restrict__ mask, const int64_t* __restrict__ rows,
                        const int64_t* __restrict__ group, int64_t n_items, int add_bias,
                        const double* __restrict__ beta, const int* __restrict__ status, double* __restrict__ part,
                        unsigned long long* __restrict__ queue, const double* __restrict__ ybar = nullptr) {
  constexpr int Q1 = P + 2;
  constexpr int NM = Q1 * (Q1 + 1) / 2;
  constexpr int U = P <= 4 ? 4 : (P <= 7 ? 2 : 1);
  const int q = P + (add_bias ? 1 : 0);
  const int lane = threadIdx.x & 31;
  for (int64_t item = pop_item(queue); item < n_items; item = pop_item(queue)) {
    const int64_t g = group[item];
    if (status[g] != RUNNING) continue;
    const int64_t r0 = rows[2 * item], r1 = rows[2 * item + 1];
    double b[P], b0 = 0.0, yb = 0.0;
    if constexpr (INIT) {
      yb = ybar[g];
    } else {
#pragma unroll
      for (int c = 0; c < P; ++c) b[c] = beta[(size_t)g * q + c];
      b0 = add_bias ? beta[(size_t)g * q + P] : 0.0;
    }
    double acc[NM + 2];
#pragma unroll
    for (int k = 0; k < NM + 2; ++k) acc[k] = 0.0;
    for (int64_t r = r0 + lane; r < r1; r += 32 * U) {
      double x[U][P], yv[U], mv[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int64_t rr = r + 32 * u;
        const int64_t rc = rr < r1 ? rr : r;            // clamped address; the row is dropped below
#pragma unroll
        for (int c = 0; c < P; ++c) x[u][c] = X[(int64_t)c * ldx + rc];
        yv[u] = y[rc];
        mv[u] = mask ? mask[rc] : 1.0;
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        double eta, mu;
        if constexpr (INIT) {                             // faer_irls's first iteration: mu_0 from y, eta_0 = g(mu_0)
          mu = R::start(yv[u], yb);
          eta = R::link(mu);
        } else {
          eta = b0;                                       // K11's order: the bias, then one fma per feature
#pragma unroll
          for (int c = 0; c < P; ++c) eta = fma(x[u][c], b[c], eta);
          mu = R::inv(eta);
        }
        double wt, z;
        R::weight_response(eta, mu, yv[u], wt, z);
        const double loss = R::loss(yv[u], eta);          // GLM: 0, and the slot is never added to
        const bool use = r + 32 * u < r1 && mv[u] != 0.0;
        double a[Q1];
#pragma unroll
        for (int c = 0; c < P; ++c) a[c] = use ? x[u][c] : 0.0;
        a[P] = use ? z : 0.0;
        a[P + 1] = use ? 1.0 : 0.0;
        wt = use ? wt : 0.0;
        int k = 0;
#pragma unroll
        for (int i = 0; i < Q1; ++i) {
          const double wa = wt * a[i];
#pragma unroll
          for (int j = i; j < Q1; ++j) { acc[k] = fma(wa, a[j], acc[k]); ++k; }
        }
        if constexpr (R::kLoss) acc[NM] += use ? loss : 0.0;
        acc[NM + 1] += a[P + 1];
      }
    }
#pragma unroll
    for (int k = 0; k < NM + 2; ++k) {
      double v = acc[k];
      for (int off = 16; off; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
      if (lane == 0) part[(size_t)k * n_items + item] = v;
    }
  }
}

// ---------------- pass A, 11 <= p <= 64: rows staged in a per-warp shared tile ----------------
// Each lane computes its row's eta, w, z and loss and writes [x | z | 1] and w to the tile; then lane l sums the partials
// k = l, l + 32, ... over the tile's 32 rows (like K5's group_moments_generic).  Shared memory per warp:
// [32][p + 3] + 32 + p + 1 doubles.
template <class R = LogisticRows, bool INIT = false>
__global__ void __launch_bounds__(GEN_WARPS * 32)
logistic_moments_generic_kernel(const double* __restrict__ X, int64_t ldx, const double* __restrict__ y,
                                const double* __restrict__ mask, const int64_t* __restrict__ rows,
                                const int64_t* __restrict__ group, int64_t n_items, int p, int add_bias,
                                const double* __restrict__ beta, const int* __restrict__ status,
                                double* __restrict__ part, unsigned long long* __restrict__ queue,
                                const double* __restrict__ ybar = nullptr) {
  extern __shared__ __align__(16) double gen_smem[];
  const int q = p + (add_bias ? 1 : 0), q1 = p + 2, ld = q1 + 1;
  const int nm = q1 * (q1 + 1) / 2;
  const int per_lane = (nm + 31) / 32;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  double* tile = gen_smem + (size_t)wid * (32 * ld + 32 + p + 1);   // [32][ld]: x_0 .. x_{p-1}, z, 1
  double* wv = tile + 32 * ld;                                       // [32] weights
  double* sb = wv + 32;                                              // [p + 1] beta, bias (or 0) last
  for (int64_t item = pop_item(queue); item < n_items; item = pop_item(queue)) {
    const int64_t g = group[item];
    if (status[g] != RUNNING) continue;
    const int64_t r0 = rows[2 * item], r1 = rows[2 * item + 1];
    double yb = 0.0;
    if constexpr (INIT) {
      yb = ybar[g];
    } else {
      __syncwarp();                                // the previous item's reads of sb are done
      for (int i = lane; i <= p; i += 32) sb[i] = i < p ? beta[(size_t)g * q + i] : (add_bias ? beta[(size_t)g * q + p] : 0.0);
      __syncwarp();
    }
    double acc[PACKED_ACC];
    for (int m = 0; m < per_lane; ++m) acc[m] = 0.0;
    double loss = 0.0, kept = 0.0;
    for (int64_t rb = r0; rb < r1; rb += 32) {
      const int64_t r = rb + lane;
      const bool in = r < r1;
      double* row = tile + lane * ld;
      double eta, mu;
      if constexpr (INIT) {
        for (int c = 0; c < p; ++c) row[c] = in ? X[(int64_t)c * ldx + r] : 0.0;
      } else {
        eta = sb[p];                               // K11's order: the bias, then one fma per feature
        for (int c = 0; c < p; ++c) {
          const double v = in ? X[(int64_t)c * ldx + r] : 0.0;
          row[c] = v;
          eta = fma(v, sb[c], eta);
        }
      }
      const double yv = in ? y[r] : 0.0;
      const bool use = in && (!mask || mask[r] != 0.0);
      if constexpr (INIT) {                        // faer_irls's first iteration: mu_0 from y, eta_0 = g(mu_0)
        mu = R::start(yv, yb);
        eta = R::link(mu);
      } else {
        mu = R::inv(eta);
      }
      double wt, z;
      R::weight_response(eta, mu, yv, wt, z);
      if (use) {
        if constexpr (R::kLoss) loss += R::loss(yv, eta);
      } else {
        for (int c = 0; c < p; ++c) row[c] = 0.0;
      }
      row[p] = use ? z : 0.0;
      row[p + 1] = use ? 1.0 : 0.0;
      wv[lane] = use ? wt : 0.0;
      kept += use ? 1.0 : 0.0;
      __syncwarp();
      tile_triangle_sum(tile, ld, q1, wv, 1, acc);
      __syncwarp();
    }
    for (int off = 16; off; off >>= 1) {
      loss += __shfl_xor_sync(0xffffffffu, loss, off);
      kept += __shfl_xor_sync(0xffffffffu, kept, off);
    }
    for (int m = 0; m < per_lane; ++m) {
      const int k = lane + 32 * m;
      if (k < nm) part[(size_t)k * n_items + item] = acc[m];
    }
    if (lane == 0) {
      part[(size_t)nm * n_items + item] = loss;
      part[(size_t)(nm + 1) * n_items + item] = kept;
    }
  }
}

// ---------------- pass B0: each running group's partials, summed over its items in item order ----------------
// The sum replaces the partial of the group's first item; a group of one item has nothing to do.
__global__ void logistic_reduce_kernel(double* __restrict__ part, const int64_t* __restrict__ item_start,
                                       int64_t n_groups, int64_t n_items, int nk, const int* __restrict__ status) {
  const int64_t total = (int64_t)nk * n_groups;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int64_t k = idx / n_groups, g = idx - k * n_groups;
    const int64_t it0 = item_start[g], it1 = item_start[g + 1];
    if (it1 - it0 < 2 || status[g] != RUNNING) continue;
    double s = part[(size_t)k * n_items + it0];
    for (int64_t it = it0 + 1; it < it1; ++it) s += part[(size_t)k * n_items + it];
    part[(size_t)k * n_items + it0] = s;
  }
}

// ---------------- pass A's instances ----------------
using PassA = void (*)(const double*, int64_t, const double*, const double*, const int64_t*, const int64_t*, int64_t,
                       int, const double*, const int*, double*, unsigned long long*, const double*);
using PassAGeneric = void (*)(const double*, int64_t, const double*, const double*, const int64_t*, const int64_t*,
                              int64_t, int, int, const double*, const int*, double*, unsigned long long*,
                              const double*);

// the register kernel of p features under row rule R (nullptr above 10 features)
template <class R, bool INIT>
PassA pass_a_regs(int p) {
  switch (p) {
    case 1: return logistic_moments_kernel<1, R, INIT>;
    case 2: return logistic_moments_kernel<2, R, INIT>;
    case 3: return logistic_moments_kernel<3, R, INIT>;
    case 4: return logistic_moments_kernel<4, R, INIT>;
    case 5: return logistic_moments_kernel<5, R, INIT>;
    case 6: return logistic_moments_kernel<6, R, INIT>;
    case 7: return logistic_moments_kernel<7, R, INIT>;
    case 8: return logistic_moments_kernel<8, R, INIT>;
    case 9: return logistic_moments_kernel<9, R, INIT>;
    case 10: return logistic_moments_kernel<10, R, INIT>;
    default: return nullptr;
  }
}
// the generic kernel's shared memory per CTA
size_t pass_a_smem(int p) { return (size_t)GEN_WARPS * (32 * (p + 3) + 32 + p + 1) * sizeof(double); }

// ---------------- pass B: host_logistic's control flow, one thread per running group ----------------
struct StepArgs {
  GroupSolveArgs a;     // part: the item partials (a group's sums in its first item's column); beta = the current
                        // iterate; status = the solve's scratch
  double* best;         // [n_groups][q] the last accepted iterate: the result
  double* cost_prev;
  int* halvings;
  int* status;
  int* n_running;
  double l1, l2, gtol;
  int64_t it;
};

__global__ void __launch_bounds__(128) logistic_step_kernel(StepArgs s) {
  const GroupSolveArgs& a = s.a;
  const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= a.n_groups || s.status[g] != RUNNING) return;
  const int p = a.p, q = p + (a.add_bias ? 1 : 0), q1 = p + 2, nm = q1 * (q1 + 1) / 2;
  const int64_t col0 = a.item_start[g];
  const double* pg = a.part + col0;                               // partial k of the group at pg[k * n_items]
  auto M = [&](int i, int j) { return pg[(size_t)packed_index(i, j, q1) * a.n_items]; };
  const double loss = pg[(size_t)nm * a.n_items];
  const double m = pg[(size_t)(nm + 1) * a.n_items];            // kept rows
  double* b = a.beta + (size_t)g * q;
  double* best = s.best + (size_t)g * q;
  auto finish = [&](int st) {
    s.status[g] = st;
    if (st != PDSB_LOGISTIC_CONVERGED) for (int j = 0; j < q; ++j) best[j] = nan("");
  };
  if (!(m >= 1.0)) { finish(PDSB_LOGISTIC_EMPTY); return; }
  double pen = 0.0, l1n = 0.0;
  for (int j = 0; j < p; ++j) { pen += b[j] * b[j]; l1n += fabs(b[j]); }
  const double cost = loss / m + 0.5 * s.l2 * pen + s.l1 * l1n;
  if (!isfinite(cost)) { finish(PDSB_LOGISTIC_FAILED); return; }
  if (s.it > 0 && cost > s.cost_prev[g] + 1e-14 * fabs(s.cost_prev[g]) && s.halvings[g] < 40) {
    // the full Newton step overshot: halve it and evaluate again
    for (int j = 0; j < q; ++j) b[j] = 0.5 * (b[j] + best[j]);
    ++s.halvings[g];
    atomicAdd(s.n_running, 1);
    return;
  }
  s.halvings[g] = 0;
  // gradient of the smooth part from the weighted moments [X | z | 1]: X'(mu - y) = (X'WX) b - X'Wz
  auto col = [&](int j) { return j < p ? j : p + 1; };            // coefficient j -> moments column (bias = ones)
  double g2 = 0.0;
  for (int j = 0; j < q; ++j) {
    double gj = -M(col(j), p);
    for (int k = 0; k < q; ++k) gj += M(col(j), col(k)) * b[k];
    gj = gj / m + (j < p ? s.l2 * b[j] : 0.0);
    if (s.l1 > 0.0 && j < p) {       // minimum-norm subgradient of the l1 term
      if (b[j] > 0.0) gj += s.l1; else if (b[j] < 0.0) gj -= s.l1;
      else gj = fabs(gj) <= s.l1 ? 0.0 : (gj > 0.0 ? gj - s.l1 : gj + s.l1);
    }
    g2 += gj * gj;
  }
  s.cost_prev[g] = cost;
  for (int j = 0; j < q; ++j) best[j] = b[j];
  if (sqrt(g2) < s.gtol) { finish(PDSB_LOGISTIC_CONVERGED); return; }
  const double sum_w = M(p + 1, p + 1);
  if (!(sum_w > 0.0)) { finish(PDSB_LOGISTIC_FAILED); return; }
  // the step: ridge solve, or coordinate descent on the weighted Gram with l1 (its penalties scale by sum w)
  if (s.l1 > 0.0) group_solve(a, g, col0, col0 + 1, s.l1 * m / sum_w, s.l2 * m / sum_w, true);
  else group_solve(a, g, col0, col0 + 1, 0.0, s.l2 * m, true);
  for (int j = 0; j < q; ++j)
    if (!isfinite(b[j])) { finish(PDSB_LOGISTIC_FAILED); return; }
  atomicAdd(s.n_running, 1);
}

// ---------------- GLM: every group's faer_irls (glm_solvers.rs:249-359) ----------------
// Once per call, ybar_g: the mean of y over the group's kept rows, for the first iteration's mu_0.  One warp per item
// sums y and counts the kept rows (lanes stride the rows, then a fixed butterfly) into part[0][item] and part[1][item];
// then one thread per group adds its items' pairs in item order.  8 bytes per row (+ 8 with a mask).
__global__ void glm_item_ysum_kernel(const double* __restrict__ y, const double* __restrict__ mask,
                                     const int64_t* __restrict__ rows, int64_t n_items, double* __restrict__ part) {
  const int lane = threadIdx.x & 31;
  const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
  for (int64_t item = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; item < n_items; item += warps) {
    const int64_t r0 = rows[2 * item], r1 = rows[2 * item + 1];
    double sy = 0.0, kept = 0.0;
    for (int64_t r = r0 + lane; r < r1; r += 32) {
      const bool use = !mask || mask[r] != 0.0;
      sy += use ? y[r] : 0.0;
      kept += use ? 1.0 : 0.0;
    }
    for (int off = 16; off; off >>= 1) {
      sy += __shfl_xor_sync(0xffffffffu, sy, off);
      kept += __shfl_xor_sync(0xffffffffu, kept, off);
    }
    if (lane == 0) { part[item] = sy; part[n_items + item] = kept; }
  }
}

__global__ void glm_mean_kernel(const double* __restrict__ part, const int64_t* __restrict__ item_start,
                                int64_t n_groups, int64_t n_items, double* __restrict__ ybar) {
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < n_groups; g += (int64_t)gridDim.x * blockDim.x) {
    double sy = 0.0, kept = 0.0;
    for (int64_t it = item_start[g]; it < item_start[g + 1]; ++it) { sy += part[it]; kept += part[n_items + it]; }
    ybar[g] = sy / kept;
  }
}

__global__ void glm_init_kernel(int64_t n_groups, int q, double* __restrict__ beta, int* __restrict__ status,
                                int64_t* __restrict__ n_iter) {
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < n_groups; g += (int64_t)gridDim.x * blockDim.x) {
    for (int j = 0; j < q; ++j) beta[(size_t)g * q + j] = 0.0;
    status[g] = RUNNING;
    n_iter[g] = 0;
  }
}

// Pass B for GLM: faer_irls's step and stopping test, one thread per running group.  The moments pass A summed are
// [X | z | 1]' W [X | z | 1] (the loss slot is 0, the last slot counts the kept rows).
struct GlmStepArgs {
  GroupSolveArgs a;     // part: the item partials (a group's sums in its first item's column); beta = the new iterate
                        // (scratch); status = the solve's scratch
  double* beta;         // [n_groups][q] the current iterate, which pass A reads: the result
  int* status;
  int64_t* n_iter;
  int* n_running;
  double tol;
  int64_t it;
};

__global__ void __launch_bounds__(128) glm_step_kernel(GlmStepArgs s) {
  const GroupSolveArgs& a = s.a;
  const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= a.n_groups || s.status[g] != RUNNING) return;
  const int p = a.p, q = p + (a.add_bias ? 1 : 0), q1 = p + 2, nm = q1 * (q1 + 1) / 2;
  const int64_t col0 = a.item_start[g];
  const double* pg = a.part + col0;                               // partial k of the group at pg[k * n_items]
  double* b = s.beta + (size_t)g * q;
  double* bn = a.beta + (size_t)g * q;
  if (!(pg[(size_t)(nm + 1) * a.n_items] >= 1.0)) {               // no kept row
    s.status[g] = PDSB_GLM_EMPTY;
    for (int j = 0; j < q; ++j) b[j] = nan("");
    return;
  }
  s.n_iter[g] = s.it + 1;
  // faer's QR propagates a NaN or inf of X'WX or X'Wz into the solution, where group_solve zeroes a zero pivot: a
  // non-finite moment the solve reads (features, z, and the ones when biased) gives NaN coefficients, as pdsb_glm_fit
  auto mi = [&](int j) { return j < p ? j : (j == p ? p : p + 1); };
  bool finite = true;
  for (int j = 0; j <= q; ++j)
    for (int k = 0; k <= j; ++k) finite &= isfinite(pg[(size_t)packed_index(mi(j), mi(k), q1) * a.n_items]);
  if (finite) group_solve(a, g, col0, col0 + 1, 0.0, 0.0, true);      // pivoted QR, no ridge, no gate
  else for (int j = 0; j < q; ++j) bn[j] = nan("");
  double max_diff = 0.0;                                          // f64::max ignores a NaN operand, as fmax does
  bool failed = false;
  for (int j = 0; j < q; ++j) {
    max_diff = fmax(max_diff, fabs(b[j] - bn[j]));
    failed |= isnan(bn[j]);
    b[j] = bn[j];
  }
  if (max_diff < s.tol) { s.status[g] = failed ? PDSB_GLM_FAILED : PDSB_GLM_CONVERGED; return; }
  atomicAdd(s.n_running, 1);
}

template <class L>
int grouped_glm_family(const double* X, int64_t ldx, const double* y, const double* mask, const int64_t* offsets,
                       int64_t n_groups, int64_t n, int p, int add_bias, double tol, int64_t max_iter, double* beta,
                       int* status, int64_t* n_iter, cudaStream_t s) {
  using R = glm::GlmRows<L>;
  const int q = p + add_bias, q1 = p + 2, nm = q1 * (q1 + 1) / 2, nk = nm + 2;
  DevBag bag(s);
  GroupWork wl;
  if (build_work_list(offsets, n_groups, n, ItemCount::EXACT, ItemMaps::ROWS_AND_GROUP, bag, wl, s)) return 1;
  const int64_t n_items = wl.n_items;
  double* part = bag.alloc<double>((size_t)nk * n_items);
  double* bnew = bag.alloc<double>((size_t)n_groups * q);
  double* ybar = bag.alloc<double>((size_t)n_groups);
  int* solve_status = bag.alloc<int>((size_t)n_groups);
  if (!part || !bnew || !ybar || !solve_status) return 1;
  int* n_running = reinterpret_cast<int*>(wl.queue + 1);     // the work list's second counter: the running groups
  const GroupSolveLaunch GS = group_solve_launch(p, q);
  double* ws = nullptr;
  if (!GS.shared && !(ws = bag.alloc<double>(((size_t)q * q + 2 * q) * n_groups))) return 1;
  const int grid_g = (int)std::min<int64_t>(ceil_div(n_groups, 256), 1024);
  glm_init_kernel<<<grid_g, 256, 0, s>>>(n_groups, q, beta, status, n_iter);
  PDSB_LAUNCH_OK();
  glm_item_ysum_kernel<<<(int)std::min<int64_t>(ceil_div(n_items, 8), (int64_t)sm_count() * 16), 256, 0, s>>>(
      y, mask, wl.rows, n_items, part);
  PDSB_LAUNCH_OK();
  glm_mean_kernel<<<grid_g, 256, 0, s>>>(part, wl.item_start, n_groups, n_items, ybar);
  PDSB_LAUNCH_OK();
  count_launch(3);

  // pass A's launches: the first iteration's instance starts from y and ybar, the others from beta
  const bool regs = p <= 10;
  const size_t gen_smem = pass_a_smem(p);
  const PassA kern_0 = pass_a_regs<R, true>(p), kern_p = pass_a_regs<R, false>(p);
  const PassAGeneric gen_0 = logistic_moments_generic_kernel<R, true>, gen_p = logistic_moments_generic_kernel<R, false>;
  const int grid_0 = regs ? persistent_grid(kern_0, 256, 0, n_items, 1)
                          : persistent_grid(gen_0, GEN_WARPS * 32, gen_smem, n_items, 1);
  const int grid_a = regs ? persistent_grid(kern_p, 256, 0, n_items, 1)
                          : persistent_grid(gen_p, GEN_WARPS * 32, gen_smem, n_items, 1);
  if (!grid_0 || !grid_a) return 1;
  const int grid_b0 = (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div((int64_t)nk * n_groups, 256), (int64_t)sm_count() * 16));
  if (smem_opt_in(glm_step_kernel, GS.smem)) return 1;

  GlmStepArgs st;
  GroupSolveArgs& a = st.a;
  a.part = part; a.item_start = wl.item_start; a.offsets = offsets; a.n_groups = n_groups; a.n_items = n_items;
  a.p = p; a.add_bias = add_bias; a.solver = PDSB_SOLVER_QR; a.l2 = 0.0; a.tol = 0.0;   // faer_weighted_lr: col_piv_qr,
  a.method = PDSB_METHOD_LSTSQ; a.positive = 0; a.max_iter = 0; a.l1 = 0.0; a.cd_tol = 0.0;  // no ridge, no gate
  a.ws = ws; a.beta = bnew; a.status = solve_status;
  st.beta = beta; st.status = status; st.n_iter = n_iter; st.n_running = n_running; st.tol = tol;

  const bool multi_item = n_items > n_groups;
  for (int64_t it = 0; it < max_iter; ++it) {
    PDSB_CUDA_OK(cudaMemsetAsync(wl.queue, 0, 2 * sizeof(unsigned long long), s));
    const int grid = it == 0 ? grid_0 : grid_a;
    if (regs) {
      const PassA k = it == 0 ? kern_0 : kern_p;
      k<<<grid, 256, 0, s>>>(X, ldx, y, mask, wl.rows, wl.group, n_items, add_bias, beta, status, part, wl.queue, ybar);
    } else {
      const PassAGeneric k = it == 0 ? gen_0 : gen_p;
      k<<<grid, GEN_WARPS * 32, gen_smem, s>>>(X, ldx, y, mask, wl.rows, wl.group, n_items, p, add_bias, beta, status,
                                               part, wl.queue, ybar);
    }
    PDSB_LAUNCH_OK();
    if (multi_item) {
      logistic_reduce_kernel<<<grid_b0, 256, 0, s>>>(part, wl.item_start, n_groups, n_items, nk, status);
      PDSB_LAUNCH_OK();
      count_launch();
    }
    st.it = it;
    glm_step_kernel<<<(int)ceil_div(n_groups, GS.threads), GS.threads, GS.smem, s>>>(st);
    PDSB_LAUNCH_OK();
    count_launch(2);
    int running = 0;
    PDSB_CUDA_OK(cudaMemcpyAsync(&running, n_running, sizeof(int), cudaMemcpyDeviceToHost, s));
    PDSB_CUDA_OK(cudaStreamSynchronize(s));
    if (running == 0) break;
  }
  return 0;
}

}  // namespace

int grouped_logistic(const double* X, int64_t ldx, const double* y, const double* mask, const int64_t* offsets,
                     int64_t n_groups, int64_t n, int p, int add_bias, double l1_reg, double l2_reg, double tol,
                     int64_t max_iter_kw, double* beta, int* status, int64_t* n_iter, cudaStream_t s) {
  if (n_iter) *n_iter = 0;
  if (n_groups <= 0) return 0;
  if (p < 1 || p > 64) { set_error("grouped logistic_reg: p=%d not supported (1..64)", p); return 1; }
  if (!X || !y || !offsets || !beta || !status) { set_error("grouped logistic_reg: null argument"); return 1; }
  // logistic_reg's kwargs as host_logistic reads them (logistic_solver.rs:127, 131-133)
  const double l1 = l1_reg > 0.0 ? std::max(l1_reg, DBL_EPSILON) : 0.0;
  const double l2 = l2_reg > 0.0 ? l2_reg : 0.0;
  const double gtol = std::max(std::sqrt(DBL_EPSILON), tol);
  const int64_t max_iter = max_iter_kw > 0 ? max_iter_kw : 200;
  const int q = p + (add_bias ? 1 : 0), q1 = p + 2, nm = q1 * (q1 + 1) / 2, nk = nm + 2;
  add_bias = add_bias ? 1 : 0;

  DevBag bag(s);
  GroupWork wl;
  if (build_work_list(offsets, n_groups, n, ItemCount::EXACT, ItemMaps::ROWS_AND_GROUP, bag, wl, s)) return 1;
  const int64_t n_items = wl.n_items;
  double* part = bag.alloc<double>((size_t)nk * n_items);
  double* bcur = bag.alloc<double>((size_t)n_groups * q);
  double* cost_prev = bag.alloc<double>((size_t)n_groups);
  int* halvings = bag.alloc<int>((size_t)n_groups);
  int* solve_status = bag.alloc<int>((size_t)n_groups);
  if (!part || !bcur || !cost_prev || !halvings || !solve_status) return 1;
  int* n_running = reinterpret_cast<int*>(wl.queue + 1);     // the work list's second counter: the running groups
  const GroupSolveLaunch L = group_solve_launch(p, q);
  double* ws = nullptr;
  if (!L.shared && !(ws = bag.alloc<double>(((size_t)q * q + 2 * q) * n_groups))) return 1;
  logistic_init_kernel<<<(int)std::min<int64_t>(ceil_div(n_groups, 256), 1024), 256, 0, s>>>(n_groups, q, bcur, beta,
                                                                                          cost_prev, halvings, status);
  PDSB_LAUNCH_OK();
  count_launch();

  // pass A's launch: a persistent grid of the resident CTAs
  const bool regs = p <= 10;
  const size_t gen_smem = pass_a_smem(p);
  const PassA kern_p = pass_a_regs<LogisticRows, false>(p);
  const int grid_a = regs ? persistent_grid(kern_p, 256, 0, n_items, 1)
                          : persistent_grid(logistic_moments_generic_kernel<>, GEN_WARPS * 32, gen_smem, n_items, 1);
  if (!grid_a) return 1;
  const int grid_b0 = (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div((int64_t)nk * n_groups, 256), (int64_t)sm_count() * 16));
  if (smem_opt_in(logistic_step_kernel, L.smem)) return 1;

  StepArgs st;
  GroupSolveArgs& a = st.a;
  a.part = part; a.item_start = wl.item_start; a.offsets = offsets; a.n_groups = n_groups; a.n_items = n_items;
  a.p = p; a.add_bias = add_bias; a.solver = PDSB_SOLVER_QR; a.l2 = 0.0; a.tol = 0.0;     // host_logistic's K3 options:
  a.method = l1 > 0.0 ? PDSB_METHOD_CD : PDSB_METHOD_LSTSQ;                                // QR, no gate; CD with l1
  a.positive = 0; a.max_iter = 2000; a.l1 = 0.0; a.cd_tol = 1e-12;
  a.ws = ws; a.beta = bcur; a.status = solve_status;
  st.best = beta; st.cost_prev = cost_prev; st.halvings = halvings; st.status = status; st.n_running = n_running;
  st.l1 = l1; st.l2 = l2; st.gtol = gtol;

  const bool multi_item = n_items > n_groups;
  for (int64_t it = 0; it < max_iter; ++it) {
    PDSB_CUDA_OK(cudaMemsetAsync(wl.queue, 0, 2 * sizeof(unsigned long long), s));
    if (regs) kern_p<<<grid_a, 256, 0, s>>>(X, ldx, y, mask, wl.rows, wl.group, n_items, add_bias, bcur, status, part,
                                            wl.queue, nullptr);
    else logistic_moments_generic_kernel<><<<grid_a, GEN_WARPS * 32, gen_smem, s>>>(X, ldx, y, mask, wl.rows, wl.group,
                                                                                      n_items, p, add_bias, bcur, status,
                                                                                      part, wl.queue);
    PDSB_LAUNCH_OK();
    if (multi_item) {
      logistic_reduce_kernel<<<grid_b0, 256, 0, s>>>(part, wl.item_start, n_groups, n_items, nk, status);
      PDSB_LAUNCH_OK();
      count_launch();
    }
    st.it = it;
    logistic_step_kernel<<<(int)ceil_div(n_groups, L.threads), L.threads, L.smem, s>>>(st);
    PDSB_LAUNCH_OK();
    count_launch(2);
    int running = 0;
    PDSB_CUDA_OK(cudaMemcpyAsync(&running, n_running, sizeof(int), cudaMemcpyDeviceToHost, s));
    PDSB_CUDA_OK(cudaStreamSynchronize(s));
    if (n_iter) *n_iter = it + 1;
    if (running == 0) break;
  }
  return 0;
}

int grouped_glm(const double* X, int64_t ldx, const double* y, const double* mask, const int64_t* offsets,
                int64_t n_groups, int64_t n, int p, int add_bias, int family, double tol, int64_t max_iter, double* beta,
                int* status, int64_t* n_iter, cudaStream_t s) {
  if (n_groups <= 0) return 0;
  if (p < 1 || p > 64) { set_error("grouped GLM: p=%d not supported (1..64)", p); return 1; }
  if (max_iter < 1) { set_error("grouped GLM: max_iter=%lld must be >= 1", (long long)max_iter); return 1; }
  if (!X || !y || !offsets || !beta || !status || !n_iter) { set_error("grouped GLM: null argument"); return 1; }
  add_bias = add_bias ? 1 : 0;
  switch (family) {
    case PDSB_GLM_GAUSSIAN:
      return grouped_glm_family<glm::Gaussian>(X, ldx, y, mask, offsets, n_groups, n, p, add_bias, tol, max_iter, beta,
                                               status, n_iter, s);
    case PDSB_GLM_POISSON:
      return grouped_glm_family<glm::Poisson>(X, ldx, y, mask, offsets, n_groups, n, p, add_bias, tol, max_iter, beta,
                                              status, n_iter, s);
    case PDSB_GLM_BINOMIAL:
      return grouped_glm_family<glm::Binomial>(X, ldx, y, mask, offsets, n_groups, n, p, add_bias, tol, max_iter, beta,
                                               status, n_iter, s);
    case PDSB_GLM_GAMMA:
      return grouped_glm_family<glm::Gamma>(X, ldx, y, mask, offsets, n_groups, n, p, add_bias, tol, max_iter, beta,
                                            status, n_iter, s);
    default: set_error("grouped GLM: unknown family %d", family); return 1;
  }
}

}  // namespace pdsb
