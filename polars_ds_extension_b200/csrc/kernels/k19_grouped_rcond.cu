// K19 — group_by(key).agg(pds.lin_reg_w_rcond(...)): every group's rank-revealing least squares and singular values in
// one launch sequence.
//
// Polars' loop makes one pl_lr_w_rcond call per group (an upload, K2's moments, K3's one-CTA RCOND solve, a synchronise).
// Here the frame stays in HBM in key order, as for pl_lr_by:
//   pass 0 + 1  K5's work list and grouped moments (group_moments, k5_grouped.cu), unchanged: per item the packed moments
//               of [x | y | 1] over its kept rows (a row with a NaN / inf in x or y drops out);
//   pass 2      one 32-thread CTA per group: the item moments summed in item order (group_solve's order), A = X'X (+ l2 on
//               the feature diagonal, not the bias) and X'y in shared memory, jacobi.h's Jacobi, then rcond.h's RCOND
//               rule, the one K3 runs for a single call, with the group's own tolerance max(rcond, eps_T max(len_g, q)).
// A group's sums depend only on its own items, so its coefficients and singular values are bit for bit the same
// whatever the other groups hold.  HBM bytes per row: (p + 1) s in pass 1; pass 2 reads (p + 2)(p + 3) / 2 doubles per
// item.
//
// ptxas (-Xptxas -v, sm_90a, CUDA 12.9): grouped_rcond_kernel 64 registers, no spill, no stack frame; 16 bytes of static
// shared memory (jacobi.h's rotation flag) and rcond_smem(q) dynamic, 69 KB at q = 65.
#include "../common.h"
#include "kernels.h"
#include "../host/host.h"
#include "k5_solve.h"
#include <cfloat>

namespace pdsb {

namespace {

constexpr int NT = 32;          // jacobi.h's and rcond.h's CTA size: one warp per group

}  // namespace
}  // namespace pdsb

#include "jacobi.h"
#include "rcond.h"

namespace pdsb {
namespace {

constexpr int RC_MAXP = 64;     // group_moments' feature limit

// A and V [q x q], X'y and rcond.h's vec [q], Jacobi's rotation table, rcond.h's perm [q]
__host__ __device__ inline size_t rcond_smem(int q) {
  return (2 * (size_t)q * q + 2 * (size_t)q + 4 * (size_t)(q / 2 + 2)) * sizeof(double) + (size_t)q * sizeof(int);
}

// beta [n_groups][q], sv [n_groups][q] descending, status [n_groups]: PDSB_GATED (beta and sv NaN) for a group with fewer
// kept rows than coefficients.  rcond: already rounded to the data type; eps: that type's epsilon.
__global__ void __launch_bounds__(NT)
grouped_rcond_kernel(const double* __restrict__ part, const int64_t* __restrict__ item_start,
                     const int64_t* __restrict__ offsets, int64_t n_items, int p, int add_bias, double rcond, double eps,
                     double l2, double* __restrict__ beta, double* __restrict__ sv, int* __restrict__ status) {
  extern __shared__ __align__(16) double rsm[];
  const int64_t g = blockIdx.x;
  const int tid = threadIdx.x, q = p + add_bias, q1 = p + 2, nm = q1 * (q1 + 1) / 2;
  double* A = rsm;
  double* V = A + (size_t)q * q;
  double* b = V + (size_t)q * q;
  double* vec = b + q;
  double* cs = vec + q;
  int* perm = reinterpret_cast<int*>(cs + 4 * (size_t)(q / 2 + 2));
  const int64_t it0 = item_start[g], it1 = item_start[g + 1];
  // moment (i, j), i <= j, of Z = [x.., y, 1]: X'X, X'y, the column sums (the bias) and the kept-row count
  double count = 0.0;
  for (int k = tid; k < nm; k += NT) {
    double s = 0.0;
    for (int64_t it = it0; it < it1; ++it) s += part[(size_t)k * n_items + it];
    int i, j;
    packed_pair(k, q1, i, j);
    if (j < p) {
      const double v = (i == j && l2 > 0.0) ? s + l2 : s;    // K3's ridge: features only
      at(A, q, i, j) = v; at(A, q, j, i) = v;
    } else if (j == p) {
      if (i < p) b[i] = s;                                   // i == p: y'y, not needed
    } else if (i < p) {
      if (add_bias) { at(A, q, i, p) = s; at(A, q, p, i) = s; }
    } else if (i == p) {
      if (add_bias) b[p] = s;
    } else {
      count = s;
      if (add_bias) at(A, q, p, p) = s;
    }
  }
  count = __shfl_sync(0xffffffffu, count, (nm - 1) % NT);
  double* bg = beta + (size_t)g * q;
  double* sg = sv + (size_t)g * q;
  if ((int64_t)llround(count) < q) {       // "#Data < #features" would be an error for a single call; per group it is null
    for (int i = tid; i < q; i += NT) { bg[i] = nan(""); sg[i] = nan(""); }
    if (tid == 0) status[g] = PDSB_GATED;
    return;
  }
  if (tid == 0) status[g] = PDSB_OK;
  // host_lin_reg_t's tolerance on the group's rows: its length counts the rows the fit drops as well
  const double tol = fmax(rcond, eps * (double)max(offsets[g + 1] - offsets[g], (int64_t)q));
  jacobi_eigen(A, V, q, cs);               // its first __syncthreads publishes A and b
  rcond_from_eigen(A, V, q, b, tol, perm, vec, sg, bg);
}

}  // namespace

template <typename T>
int grouped_lin_reg_rcond(const T* X, int64_t ldx, const T* y, const int64_t* offsets, int64_t n_groups, int64_t n,
                          int p, const pdsb_solve_opts& o, double* beta, double* sv, int* status, cudaStream_t s) {
  if (n_groups <= 0) return 0;
  if (p < 1 || p > RC_MAXP) {
    set_error("grouped lin_reg_w_rcond: %d features; at most %d are supported", p, RC_MAXP);
    return 1;
  }
  if (!X || !y || !offsets || !beta || !sv || !status) { set_error("grouped lin_reg_w_rcond: null argument"); return 1; }
  const int add_bias = o.add_bias ? 1 : 0, q = p + add_bias;
  DevBag bag(s);
  GroupWork wl;
  double* part = nullptr;
  if (build_work_list(offsets, n_groups, n, ItemCount::EXACT, p <= 10 ? ItemMaps::ROWS : ItemMaps::NONE, bag, wl, s) ||
      group_moments<T>(X, ldx, y, offsets, n_groups, p, wl, bag, &part, s))
    return 1;
  // host_lin_reg_t's rule: the f32 twin rounds rcond to f32 and floors it with f32's epsilon
  const bool f32 = sizeof(T) == 4;
  const double rcond = f32 ? (double)(float)o.tol : o.tol;
  const double eps = f32 ? (double)FLT_EPSILON : DBL_EPSILON;
  const size_t smem = rcond_smem(q);
  if (smem_opt_in(grouped_rcond_kernel, smem)) return 1;
  grouped_rcond_kernel<<<(unsigned)n_groups, NT, smem, s>>>(part, wl.item_start, offsets, wl.n_items, p, add_bias, rcond,
                                                            eps, o.l2_reg, beta, sv, status);
  PDSB_LAUNCH_OK();
  count_launch();
  return 0;
}

template int grouped_lin_reg_rcond<float>(const float*, int64_t, const float*, const int64_t*, int64_t, int64_t, int,
                                          const pdsb_solve_opts&, double*, double*, int*, cudaStream_t);
template int grouped_lin_reg_rcond<double>(const double*, int64_t, const double*, const int64_t*, int64_t, int64_t, int,
                                           const pdsb_solve_opts&, double*, double*, int*, cudaStream_t);

}  // namespace pdsb
