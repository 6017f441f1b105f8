// The RCOND rule of lin_reg_w_rcond, shared by K3 (solve_kernel, PDSB_METHOD_RCOND: one call) and K19
// (k19_grouped_rcond.cu: one group per CTA).  Header-only for the reason jacobi.h is; the including file defines NT, its
// CTA size, and includes jacobi.h first.
#pragma once
#include <cuda_runtime.h>

namespace pdsb {

namespace {

// After jacobi_eigen(A, V, q, ...) on the (ridged) q x q Gram: the eigenvalues lambda (A's diagonal) in descending order
// (selection sort on thread 0; q is tiny), thr = tol * sqrt(max(lambda_max, 0)) (rcond times the largest singular value
// of X, lr_solvers.rs:230-232), then beta = V diag(lambda >= thr ? 1 / lambda : 0) V^T b.  Quirk kept (:236-240): the
// EIGENVALUE of X'X is compared against thr, not the singular value.  sv (nullable): sqrt(max(lambda, 0)) in the same
// descending order.  perm [q] ints and vec [q] doubles are scratch; every thread of the CTA takes part.
__device__ __forceinline__ void rcond_from_eigen(double* A, double* V, int q, double* b, double tol, int* perm,
                                                 double* vec, double* sv, double* beta) {
  const int tid = threadIdx.x;
  if (tid == 0) {
    for (int i = 0; i < q; ++i) perm[i] = i;
    for (int i = 0; i < q; ++i) {
      int best = i;
      for (int j = i + 1; j < q; ++j) if (at(A, q, perm[j], perm[j]) > at(A, q, perm[best], perm[best])) best = j;
      int x = perm[i]; perm[i] = perm[best]; perm[best] = x;
    }
  }
  __syncthreads();
  const double smax = fmax(at(A, q, perm[0], perm[0]), 0.0);
  const double thr = tol * sqrt(smax);
  for (int idx = tid; idx < q; idx += NT) {
    double lam = at(A, q, perm[idx], perm[idx]);
    if (sv) sv[idx] = sqrt(fmax(lam, 0.0));
    double s = 0.0;
    for (int r = 0; r < q; ++r) s += at(V, q, r, perm[idx]) * b[r];
    vec[idx] = (lam >= thr) ? s / lam : 0.0;
  }
  __syncthreads();
  for (int i = tid; i < q; i += NT) {
    double s = 0.0;
    for (int r = 0; r < q; ++r) s += at(V, q, i, perm[r]) * vec[r];
    beta[i] = s;
  }
}

}  // namespace

}  // namespace pdsb
