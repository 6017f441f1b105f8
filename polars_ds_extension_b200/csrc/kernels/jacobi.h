// Single-CTA symmetric eigen-solver shared by K3 (svd / rcond solves), K13 (PCA), K18 and K19 (their grouped forms).  Header-only because the library is
// built without relocatable device code: a __device__ function defined in one .cu file cannot be called from another.
// The including file defines NT, its CTA size, in pdsb's anonymous namespace before the include.
#pragma once
#include <cuda_runtime.h>

namespace pdsb {

namespace {

__device__ __forceinline__ double& at(double* A, int q, int i, int j) { return A[i + (size_t)j * q]; }

// ---- symmetric eigen-decomposition by parallel-ordered two-sided Jacobi:  A = V diag(lam) V^T ----
__device__ void jacobi_eigen(double* A, double* V, int q, double* cs) {
  __shared__ int sh_rot;
  const int tid = threadIdx.x;
  for (int i = tid; i < q * q; i += NT) V[i] = ((i % q) == (i / q)) ? 1.0 : 0.0;
  __syncthreads();
  const int ne = (q + 1) & ~1;       // even number of players
  const int m = ne - 1;
  const int npairs = ne / 2;
  if (q < 2) return;
  for (int sweep = 0; sweep < 60; ++sweep) {
    if (tid == 0) sh_rot = 0;
    __syncthreads();
    for (int r = 0; r < m; ++r) {
      for (int pi = tid; pi < npairs; pi += NT) {     // any q: pairs strided over the CTA
        int a, b;
        if (pi == 0) { a = m; b = r; }
        else { a = (r + pi) % m; b = (r - pi % m + m) % m; }
        if (a > b) { int x = a; a = b; b = x; }
        double c = 1.0, s = 0.0;
        if (b < q && a != b) {
          double apq = at(A, q, a, b), app = at(A, q, a, a), aqq = at(A, q, b, b);
          // negligible-off-diagonal test (classic cyclic Jacobi): skip when apq cannot change either diagonal
          const double g = 100.0 * fabs(apq);
          const bool negligible = (fabs(app) + g == fabs(app)) && (fabs(aqq) + g == fabs(aqq));
          if (apq != 0.0 && !negligible) {
            double theta = (aqq - app) / (2.0 * apq);
            double tt = (theta >= 0.0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
            if (!isfinite(theta)) tt = 0.0;
            c = 1.0 / sqrt(tt * tt + 1.0);
            s = tt * c;
            if (s != 0.0) sh_rot = 1;
          }
        } else { a = -1; }
        cs[4 * pi + 0] = c; cs[4 * pi + 1] = s;
        cs[4 * pi + 2] = (double)a; cs[4 * pi + 3] = (double)b;
      }
      __syncthreads();
      // column update A <- A J, V <- V J
      for (int wkk = tid; wkk < npairs * q; wkk += NT) {
        int pi = wkk / q, k = wkk - pi * q;
        int a = (int)cs[4 * pi + 2], b = (int)cs[4 * pi + 3];
        double c = cs[4 * pi], s = cs[4 * pi + 1];
        if (a < 0 || s == 0.0) continue;
        double x = at(A, q, k, a), y = at(A, q, k, b);
        at(A, q, k, a) = c * x - s * y; at(A, q, k, b) = s * x + c * y;
        x = at(V, q, k, a); y = at(V, q, k, b);
        at(V, q, k, a) = c * x - s * y; at(V, q, k, b) = s * x + c * y;
      }
      __syncthreads();
      // row update A <- J^T A
      for (int wkk = tid; wkk < npairs * q; wkk += NT) {
        int pi = wkk / q, k = wkk - pi * q;
        int a = (int)cs[4 * pi + 2], b = (int)cs[4 * pi + 3];
        double c = cs[4 * pi], s = cs[4 * pi + 1];
        if (a < 0 || s == 0.0) continue;
        double x = at(A, q, a, k), y = at(A, q, b, k);
        at(A, q, a, k) = c * x - s * y; at(A, q, b, k) = s * x + c * y;
      }
      __syncthreads();
    }
    if (!sh_rot) break;
    __syncthreads();
  }
}

}  // namespace

}  // namespace pdsb
