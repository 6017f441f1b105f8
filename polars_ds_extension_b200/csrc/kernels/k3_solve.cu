// K3 — single-CTA dense solve on the (q1 x q1) moments, all in f64.
//
// Restates on the GPU what the reference does on the p x p normal equations with faer
// (/root/reference/src/linear/lr/lr_solvers.rs):
//   solve_xtx_xty / faer_solve_lr           :282-308   col-piv QR | thin SVD | LLT(+QR fallback)
//   faer_solve_lr_gated + sum_ln            :313-382   ln|det| - sum ln diag <= ln tol  -> null
//   faer_solve_lr_rcond                     :216-258   eigen-decomposition of X'X, rcond cut (quirk kept)
//   faer_coordinate_descent                 :426-538   lasso / elastic net / positive
//   faer_nn_lr                              :542-600   projected coordinate NNLS
//   faer_qr_lr_with_inv                     lr_online_solvers.rs:120-143 and linear_regression.rs:854-858 (inverse)
// The matrices are tiny (q <= ~260) and live in an L1-resident global workspace; one CTA of 256 threads,
// column-parallel Householder QR with column pivoting, parallel-ordered two-sided Jacobi for the SVD of the
// symmetric Gram, right-looking Cholesky.  Time is microseconds; what matters is that the data pass (K2) is
// never repeated: every solver variant starts from the same moments.
#include "../common.h"
#include "kernels.h"
#include <cmath>

namespace pdsb {

namespace {

constexpr int NT = 256;

struct Ws {
  double* A;     // q x q  col-major
  double* V;     // q x q  col-major
  double* B;     // q x nb col-major (nb = max(t, q))
  double* G;     // q x q  pristine copy (row-major == col-major, symmetric)
  double* vec;   // 4q scratch
  int* perm;     // q
  double* cs;    // 4 * (q/2+1) rotation params
};

__device__ __forceinline__ double& at(double* A, int q, int i, int j);   // jacobi.h

// ---- Householder QR with column pivoting; applies Q^T to B (nb columns) ----
__device__ void qr_pivot(double* A, int q, double* B, int nb, int* perm, double* cn, double* tau_v0) {
  __shared__ int sh_piv;
  __shared__ double sh_v0, sh_beta, sh_alpha, sh_s;
  const int tid = threadIdx.x;
  for (int j = tid; j < q; j += NT) perm[j] = j;
  __syncthreads();
  for (int k = 0; k < q; ++k) {
    for (int j = k + tid; j < q; j += NT) {
      double s = 0.0;
      for (int i = k; i < q; ++i) { double v = at(A, q, i, j); s += v * v; }
      cn[j] = s;
    }
    __syncthreads();
    if (tid < 32) {   // warp 0: arg-max of the trailing column norms (ties -> lowest index, like a serial scan)
      int piv = k; double best = -1.0;
      for (int j = k + tid; j < q; j += 32) { const double c = cn[j]; if (c > best) { best = c; piv = j; } }
      for (int off = 16; off; off >>= 1) {
        const double ob = __shfl_xor_sync(0xffffffffu, best, off);
        const int op = __shfl_xor_sync(0xffffffffu, piv, off);
        if (ob > best || (ob == best && op < piv)) { best = ob; piv = op; }
      }
      if (tid == 0) { sh_piv = piv; sh_s = best < 0.0 ? 0.0 : best; }
    }
    __syncthreads();
    const int piv = sh_piv;
    if (piv != k) {
      for (int i = tid; i < q; i += NT) { double a = at(A, q, i, k); at(A, q, i, k) = at(A, q, i, piv); at(A, q, i, piv) = a; }
      if (tid == 0) { int a = perm[k]; perm[k] = perm[piv]; perm[piv] = a; }
    }
    __syncthreads();
    if (tid == 0) {
      const double s = sh_s;                       // = sum_{i>=k} A[i,k]^2 of the pivot column (computed above)
      double normx = sqrt(s);
      double x0 = at(A, q, k, k);
      double alpha = (x0 >= 0.0) ? -normx : normx;
      double v0 = x0 - alpha;
      double vtv = v0 * v0 + (s - x0 * x0);
      sh_alpha = alpha; sh_v0 = v0;
      sh_beta = (vtv > 0.0 && isfinite(vtv)) ? 2.0 / vtv : 0.0;
    }
    __syncthreads();
    const double v0 = sh_v0, beta = sh_beta;
    if (beta != 0.0) {
      const int ncols = (q - k - 1) + nb;
      for (int c = tid; c < ncols; c += NT) {
        double* C = (c < q - k - 1) ? (A + (size_t)(k + 1 + c) * q) : (B + (size_t)(c - (q - k - 1)) * q);
        double dot = v0 * C[k];
        for (int i = k + 1; i < q; ++i) dot += at(A, q, i, k) * C[i];
        double f = beta * dot;
        C[k] -= f * v0;
        for (int i = k + 1; i < q; ++i) C[i] -= f * at(A, q, i, k);
      }
    }
    __syncthreads();
    if (tid == 0) { at(A, q, k, k) = sh_alpha; tau_v0[k] = v0; }
    __syncthreads();
  }
}

// back-substitution R z = c for every column of B, then un-permute into X (q x nb col-major)
__device__ void qr_backsolve(const double* A, int q, double* B, int nb, const int* perm, double* X) {
  for (int c = threadIdx.x; c < nb; c += NT) {
    double* z = B + (size_t)c * q;
    for (int i = q - 1; i >= 0; --i) {
      double s = z[i];
      for (int j = i + 1; j < q; ++j) s -= A[i + (size_t)j * q] * z[j];
      double r = A[i + (size_t)i * q];
      z[i] = (r != 0.0) ? s / r : 0.0;
    }
    for (int i = 0; i < q; ++i) X[perm[i] + (size_t)c * q] = z[i];
  }
  __syncthreads();
}

// ---- Cholesky (lower, in place). returns false when not positive definite ----
__device__ bool cholesky(double* A, int q) {
  __shared__ int sh_fail;
  const int tid = threadIdx.x;
  if (tid == 0) sh_fail = 0;
  __syncthreads();
  for (int k = 0; k < q; ++k) {
    if (tid == 0) {
      double d = at(A, q, k, k);
      if (!(d > 0.0) || !isfinite(d)) sh_fail = 1; else at(A, q, k, k) = sqrt(d);
    }
    __syncthreads();
    if (sh_fail) return false;
    const double lkk = at(A, q, k, k);
    for (int i = k + 1 + tid; i < q; i += NT) at(A, q, i, k) /= lkk;
    __syncthreads();
    for (int j = k + 1 + tid; j < q; j += NT) {
      const double ljk = at(A, q, j, k);
      for (int i = j; i < q; ++i) at(A, q, i, j) -= at(A, q, i, k) * ljk;
    }
    __syncthreads();
  }
  return true;
}

__device__ void chol_solve(const double* L, int q, double* B, int nb) {
  for (int c = threadIdx.x; c < nb; c += NT) {
    double* z = B + (size_t)c * q;
    for (int i = 0; i < q; ++i) {
      double s = z[i];
      for (int j = 0; j < i; ++j) s -= L[i + (size_t)j * q] * z[j];
      z[i] = s / L[i + (size_t)i * q];
    }
    for (int i = q - 1; i >= 0; --i) {
      double s = z[i];
      for (int j = i + 1; j < q; ++j) s -= L[j + (size_t)i * q] * z[j];
      z[i] = s / L[i + (size_t)i * q];
    }
  }
  __syncthreads();
}

}  // namespace
}  // namespace pdsb

// Included here, after the routines above, rather than at the top: static __shared__ variables are laid out in the order
// of the functions that define them, so this place keeps solve_kernel's shared-memory layout (and its SASS) unchanged.
#include "jacobi.h"
#include "rcond.h"

namespace pdsb {
namespace {

struct SolveParams {
  const double* M; pdsb_solve_opts o; double* beta; int* status; double* aux; Ws ws; int use_smem;
};

__device__ __forceinline__ int fidx(int i, int p, int t) { return i < p ? i : p + t; }  // feature i -> moments index

__global__ void __launch_bounds__(NT) solve_kernel(SolveParams P) {
  const pdsb_solve_opts& o = P.o;
  const int p = o.p, t = o.t, q1 = p + t + 1;
  const int q = p + (o.add_bias ? 1 : 0);
  const double* M = P.M;
  extern __shared__ double solve_smem[];
  double* A = P.ws.A; double* V = P.ws.V; double* B = P.ws.B; double* G = P.ws.G;
  if (P.use_smem) { A = solve_smem; B = solve_smem + (size_t)(p + (o.add_bias ? 1 : 0)) * (p + (o.add_bias ? 1 : 0)); }   // hot matrices on chip
  double* vec = P.ws.vec; int* perm = P.ws.perm;
  const int tid = threadIdx.x;
  __shared__ int sh_gate;
  __shared__ double sh_lnden, sh_lndet;
  if (tid == 0) { sh_gate = 0; *P.status = PDSB_OK; }

  const bool ridge = (o.method == PDSB_METHOD_LSTSQ || o.method == PDSB_METHOD_RCOND || o.method == PDSB_METHOD_INV) &&
                     o.l2_reg > 0.0;
  for (int idx = tid; idx < q * q; idx += NT) {
    int i = idx % q, j = idx / q;
    double v = M[(size_t)fidx(i, p, t) * q1 + fidx(j, p, t)];
    if (ridge && i == j && i < p) v += o.l2_reg;
    A[idx] = v; G[idx] = v;
  }
  const int nrhs = (o.method == PDSB_METHOD_INV) ? (t + q) : t;
  for (int idx = tid; idx < q * t; idx += NT) {
    int i = idx % q, k = idx / q;
    B[idx] = M[(size_t)fidx(i, p, t) * q1 + (p + k)];
  }
  if (o.method == PDSB_METHOD_INV)
    for (int idx = tid; idx < q * q; idx += NT) B[(size_t)q * t + idx] = ((idx % q) == (idx / q)) ? 1.0 : 0.0;
  __syncthreads();
  const double count = M[(size_t)(q1 - 1) * q1 + (q1 - 1)];

  if (o.method == PDSB_METHOD_LSTSQ || o.method == PDSB_METHOD_INV) {
    const bool gated = (o.method == PDSB_METHOD_LSTSQ) && o.singular_x_tol > 0.0;
    if (gated && tid == 0) {
      double s = 0.0; int bad = 0;
      // faer_solve_lr_gated (lr_solvers.rs:341-347): `d <= 0` gates; a NaN diagonal (null_policy "ignore" with NaN data)
      // compares false, poisons ln_den, and every later `<= ln_tol` test is false too: the reference SOLVES and returns
      // NaN coefficients (QR / LLT); its SVD fails to converge on NaN and gates (:360).
      for (int i = 0; i < q; ++i) { double d = at(G, q, i, i); if (d <= 0.0) bad = 1; else s += log(d); }
      sh_lnden = s; if (bad) sh_gate = 1;
    }
    __syncthreads();
    if (sh_gate) { if (tid == 0) *P.status = PDSB_GATED; return; }
    if (gated && isnan(sh_lnden)) {
      if (o.solver == PDSB_SOLVER_SVD) { if (tid == 0) *P.status = PDSB_GATED; return; }
      for (int idx = tid; idx < q * t; idx += NT) P.beta[idx] = nan("");
      return;
    }
    const double ln_tol = gated ? log(o.singular_x_tol) : 0.0;
    int solver = o.solver;
    if (o.method == PDSB_METHOD_INV) solver = PDSB_SOLVER_QR;
    if (solver == PDSB_SOLVER_CHOLESKEY) {
      bool ok = cholesky(A, q);
      if (ok) {
        if (gated) {
          if (tid == 0) { double s = 0.0; for (int i = 0; i < q; ++i) s += log(at(A, q, i, i)); sh_lndet = s + s; }
          __syncthreads();
          if (sh_lndet - sh_lnden <= ln_tol) { if (tid == 0) *P.status = PDSB_GATED; return; }
        }
        chol_solve(A, q, B, nrhs);
        for (int idx = tid; idx < q * t; idx += NT) P.beta[idx] = B[idx];
        return;
      }
      if (gated) { if (tid == 0) *P.status = PDSB_GATED; return; }  // lr_solvers.rs:371
      // ungated LLT failure falls back to QR (lr_solvers.rs:288-291): restore A
      for (int idx = tid; idx < q * q; idx += NT) A[idx] = G[idx];
      __syncthreads();
      solver = PDSB_SOLVER_QR;
    }
    if (solver == PDSB_SOLVER_SVD) {
      jacobi_eigen(A, V, q, P.ws.cs);
      if (tid == 0) {
        double s = 0.0;
        for (int i = 0; i < q; ++i) s += log(fabs(at(A, q, i, i)));
        sh_lndet = s;
      }
      __syncthreads();
      if (gated && (sh_lndet - sh_lnden <= ln_tol || !isfinite(sh_lndet))) { if (tid == 0) *P.status = PDSB_GATED; return; }
      // beta = V diag(1/lam) V^T B
      for (int idx = tid; idx < q * t; idx += NT) {
        int i = idx % q, k = idx / q;
        double s = 0.0;
        for (int r = 0; r < q; ++r) s += at(V, q, r, i) * B[r + (size_t)k * q];
        vec[idx] = s / at(A, q, i, i);
      }
      __syncthreads();
      for (int idx = tid; idx < q * t; idx += NT) {
        int i = idx % q, k = idx / q;
        double s = 0.0;
        for (int r = 0; r < q; ++r) s += at(V, q, i, r) * vec[r + (size_t)k * q];
        P.beta[idx] = s;
      }
      return;
    }
    // QR (default; also every unknown solver string: lr/mod.rs:23)
    qr_pivot(A, q, B, nrhs, perm, vec, vec + q);
    if (gated) {
      if (tid == 0) { double s = 0.0; for (int i = 0; i < q; ++i) s += log(fabs(at(A, q, i, i))); sh_lndet = s; }
      __syncthreads();
      if (sh_lndet - sh_lnden <= ln_tol) { if (tid == 0) *P.status = PDSB_GATED; return; }
    }
    qr_backsolve(A, q, B, nrhs, perm, V /* reuse V as X (q x nrhs) */);
    for (int idx = tid; idx < q * t; idx += NT) P.beta[idx] = V[idx];
    if (o.method == PDSB_METHOD_INV && P.aux)
      for (int idx = tid; idx < q * q; idx += NT) {
        // V[(t + c) * q + r] = inverse[r][c]; symmetric; write row-major
        int r = idx / q, c = idx % q;
        P.aux[idx] = V[(size_t)(t + c) * q + r];
      }
    return;
  }

  if (o.method == PDSB_METHOD_RCOND) {
    jacobi_eigen(A, V, q, P.ws.cs);
    rcond_from_eigen(A, V, q, B, o.tol, perm, vec, P.aux, P.beta);
    return;
  }

  // ---- iterative methods on the Gram (sequential over coordinates by nature): one warp ----
  if (tid >= 32) return;
  const int lane = tid;
  const int n1 = p;                                   // coordinates that are regularised / constrained
  double* beta = vec;                                 // q
  double* mu = vec + q;                               // q (NNLS)
  for (int i = lane; i < q; i += 32) { beta[i] = 0.0; mu[i] = -B[i]; }
  __syncwarp();
  if (o.method == PDSB_METHOD_CD) {
    const double mcount = count;
    const double lambda_l1 = mcount * o.l1_reg;
    const double l2n = mcount * o.l2_reg;
    const double y_sum = M[(size_t)p * q1 + (q1 - 1)];
    for (int it = 0; it < o.max_iter; ++it) {
      double max_change = 0.0;
      for (int j = 0; j < n1; ++j) {
        double before = beta[j];
        double part = 0.0;
        for (int i = lane; i < q; i += 32) if (i != j) part += at(G, q, i, j) * beta[i];
        for (int off = 16; off; off >>= 1) part += __shfl_xor_sync(0xffffffffu, part, off);
        double main_update = B[j] - part;
        double after;
        if (o.positive && main_update < 0.0) after = 0.0;
        else {
          double sgn = (main_update > 0.0) ? 1.0 : ((main_update < 0.0) ? -1.0 : 0.0);
          after = sgn * fmax(fabs(main_update) - lambda_l1, 0.0) / (at(G, q, j, j) + l2n);
        }
        __syncwarp();
        if (lane == 0) beta[j] = after;
        __syncwarp();
        max_change = fmax(max_change, fabs(after - before));
      }
      if (o.add_bias) {
        double part = 0.0;
        for (int j = lane; j < n1; j += 32) part += beta[j] * M[(size_t)j * q1 + (q1 - 1)];
        for (int off = 16; off; off >>= 1) part += __shfl_xor_sync(0xffffffffu, part, off);
        if (lane == 0) beta[n1] = (y_sum - part) / mcount;
        __syncwarp();
      }
      if (max_change < o.tol) break;
    }
  } else {  // NNLS
    for (int it = 0; it < o.max_iter; ++it) {
      int ok = 1;
      for (int i = lane; i < q; i += 32) {
        if (!(mu[i] >= -o.tol)) ok = 0;
        if (beta[i] > 0.0 && !(mu[i] <= o.tol)) ok = 0;
      }
      ok = __all_sync(0xffffffffu, ok);
      if (ok) break;
      for (int k = 0; k < q; ++k) {
        double beta_k = beta[k];
        double update = beta_k - mu[k] / at(G, q, k, k);
        if (!o.add_bias || k < q - 1) update = fmax(update, 0.0);
        double diff = update - beta_k;
        __syncwarp();
        for (int i = lane; i < q; i += 32) mu[i] += diff * at(G, q, i, k);
        if (lane == 0) beta[k] = update;
        __syncwarp();
      }
    }
  }
  for (int i = lane; i < q; i += 32) P.beta[i] = beta[i];
}

}  // namespace

int solve_from_moments(const double* M, const pdsb_solve_opts& o, double* beta, int* status, double* aux,
                       cudaStream_t s) {
  const int q = o.p + (o.add_bias ? 1 : 0);
  if (q < 1) { set_error("solve: no features"); return 1; }
  if (o.t < 1) { set_error("solve: no target"); return 1; }
  if ((o.method == PDSB_METHOD_CD || o.method == PDSB_METHOD_NNLS || o.method == PDSB_METHOD_RCOND) && o.t != 1) {
    set_error("The method is not supported.");
    return 1;
  }
  const int nb = o.t + q;
  size_t nd = (size_t)q * q * 2 + 2 * (size_t)q * nb + 4 * (size_t)q + (size_t)q * o.t + 4 * (size_t)(q / 2 + 2) + 8;
  size_t bytes = nd * sizeof(double) + (size_t)q * sizeof(int) + 64;
  char* base = nullptr;
  if (dev_alloc((void**)&base, bytes, s)) return 1;
  SolveParams P;
  P.M = M; P.o = o; P.beta = beta; P.status = status; P.aux = aux;
  double* d = reinterpret_cast<double*>(base);
  P.ws.A = d; d += (size_t)q * q;
  P.ws.V = d; d += (size_t)q * std::max(q, nb);   // V doubles as the solution buffer (q x nrhs)
  P.ws.G = d; d += (size_t)q * q;
  P.ws.B = d; d += (size_t)q * nb;
  P.ws.vec = d; d += 4 * (size_t)q + (size_t)q * o.t;
  P.ws.cs = d; d += 4 * (size_t)(q / 2 + 2);
  P.ws.perm = reinterpret_cast<int*>(d);
  const size_t hot = ((size_t)q * q + (size_t)q * nb) * sizeof(double);
  P.use_smem = hot <= 200 * 1024;
  if (P.use_smem && hot > 48 * 1024) cudaFuncSetAttribute(solve_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)hot);
  solve_kernel<<<1, NT, P.use_smem ? hot : 0, s>>>(P);
  cudaError_t e = cudaGetLastError();
  count_launch();
  dev_free(base, s);
  if (e != cudaSuccess) { set_error("solve launch failed: %s", cudaGetErrorString(e)); return 1; }
  return 0;
}

}  // namespace pdsb
