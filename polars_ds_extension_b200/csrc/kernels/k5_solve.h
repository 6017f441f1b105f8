// K5's per-group solve (pass 2) and work-queue pop, shared by the grouped lin_reg fit (k5_grouped.cu) and the grouped
// logistic fit (k16_grouped_logistic.cu).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "../../../include/pdsb.h"

namespace pdsb {

// the warp's next item from the global counter: lane 0 takes it, every lane returns it
__device__ __forceinline__ int64_t pop_item(unsigned long long* __restrict__ queue) {
  unsigned long long v = 0;
  if ((threadIdx.x & 31) == 0) v = atomicAdd(queue, 1ULL);
  return (int64_t)__shfl_sync(0xffffffffu, v, 0);
}

// ---------------- pass 2: batched solve, one thread per group, interleaved workspace ----------------
struct GroupSolveArgs {
  const double* part; const int64_t* item_start; const int64_t* offsets;
  int64_t n_groups, n_items; int p, add_bias, solver; double l2, tol;
  int method, positive, max_iter; double l1, cd_tol;      // PDSB_METHOD_CD / _NNLS per group (lr_solvers.rs:426-600)
  double* ws;      // [(q*q + 2q) ][n_groups]  interleaved; nullptr: the workspace lives in shared memory, [(q*q + 2q)][blockDim.x]
  double* beta;    // [n_groups][q]
  int* status;
};

// The workspace of one group's solve: A, b, scratch and (in shared memory only) the gathered moments.  It goes in the
// shared memory of a 32-thread CTA when that holds it, else in global memory, [(q*q + 2q)][n_groups].
struct GroupSolveLaunch {
  bool shared;
  size_t smem;      // dynamic shared memory per CTA
  int threads;      // per CTA
};
inline GroupSolveLaunch group_solve_launch(int p, int q) {
  const size_t per_thread = ((size_t)q * q + 2 * q + (size_t)(p + 2) * (p + 3) / 2) * sizeof(double);   // A, b, scratch, moments
  if (per_thread * 32 <= (size_t)200 * 1024) return {true, per_thread * 32, 32};
  return {false, 0, 128};
}

// The solve of group g on the packed moments of [X | y | 1] summed over its items [it0, it1) of a.part, written to
// a.beta[g] and a.status[g].  l1, l2: the penalties (lin_reg passes a.l1 and a.l2).  irls: the moments are IRLS-weighted
// (K16), so the ones x ones entry is sum w, not a row count: no "fewer rows than coefficients" gate, and coordinate
// descent scales its penalties by that unrounded sum.  With irls = false this is the lin_reg solve, unchanged.
__device__ __forceinline__ void group_solve(const GroupSolveArgs& a, int64_t g, int64_t it0, int64_t it1, double l1,
                                            double l2, bool irls) {
  const int p = a.p, q = p + (a.add_bias ? 1 : 0), q1 = p + 2;
  // one thread per group walks dependent chains over its q x q system: in global memory every step pays a DRAM / L2 round
  // trip (0.113 ms for 1e4 groups of 9 coefficients, 14 % of the C3 step); up to ~20 coefficients the workspace of a
  // 32-thread CTA fits shared memory instead (same interleaved layout, stride = threads per CTA)
  extern __shared__ double gs_smem[];
  const int64_t NG = a.ws ? a.n_groups : (int64_t)blockDim.x;
  double* base = a.ws ? a.ws + g : gs_smem + threadIdx.x;
  double* A = base;                                      // A(i,j) = A[(i + j*q) * NG]
  double* b = base + (size_t)q * q * NG;                 // b(i)   = b[i * NG]
  double* cn = base + ((size_t)q * q + q) * NG;          // scratch q
#define AA(i, j) A[((size_t)(i) + (size_t)(j) * q) * NG]
#define BB(i) b[(size_t)(i) * NG]
#define CN(i) cn[(size_t)(i) * NG]
  // moment (i,j) of Z=[x.., y, 1], i<=j, packed index
  auto midx = [&](int i, int j) { if (i > j) { int t = i; i = j; j = t; } return i * q1 - i * (i - 1) / 2 + (j - i); };
  auto fz = [&](int i) { return i < p ? i : p + 1; };    // coefficient index -> Z column (bias -> ones)
  const double* __restrict__ part = a.part;
  const int nm = q1 * (q1 + 1) / 2;
  // the group's moments, summed over its items in a fixed order.  With the shared-memory workspace they are gathered
  // first, eight independent loads at a time (a load followed at once by its consumer serialises on the in-order issue:
  // 64 dependent round trips were 40 of the kernel's 97 microseconds at 9 coefficients)
  double* ms = a.ws ? nullptr : base + ((size_t)q * q + 2 * q) * NG;     // ms(k) = ms[k * NG]
  if (ms) {
    for (int k0 = 0; k0 < nm; k0 += 8) {
      double v[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const int k = k0 + u < nm ? k0 + u : nm - 1;
        v[u] = part[(size_t)k * a.n_items + it0];
      }
      for (int64_t it = it0 + 1; it < it1; ++it) {
#pragma unroll
        for (int u = 0; u < 8; ++u) {
          const int k = k0 + u < nm ? k0 + u : nm - 1;
          v[u] += part[(size_t)k * a.n_items + it];
        }
      }
#pragma unroll
      for (int u = 0; u < 8; ++u)
        if (k0 + u < nm) ms[(size_t)(k0 + u) * NG] = v[u];
    }
  }
  auto mom = [&](int k) {
    if (ms) return ms[(size_t)k * NG];
    double s = 0.0;
    for (int64_t it = it0; it < it1; ++it) s += part[(size_t)k * a.n_items + it];
    return s;
  };
  const double count = mom(midx(p + 1, p + 1));
  const int64_t nrows = (int64_t)llround(count);   // valid rows of the group (lin_reg)
  double* out = a.beta + (size_t)g * q;
  if (!irls && nrows < q) {  // "#Data < #features" would be an error for a single call; per group it yields null
    a.status[g] = PDSB_GATED;
    for (int i = 0; i < q; ++i) out[i] = nan("");
    return;
  }
  for (int j = 0; j < q; ++j)
    for (int i = 0; i <= j; ++i) {
      double v = mom(midx(fz(i), fz(j)));
      if (a.method == PDSB_METHOD_LSTSQ && i == j && i < p && l2 > 0.0) v += l2;   // ridge; CD scales l2 by n itself
      AA(i, j) = v; AA(j, i) = v;
    }
  for (int i = 0; i < q; ++i) BB(i) = mom(midx(fz(i), p));
  if (a.method == PDSB_METHOD_CD || a.method == PDSB_METHOD_NNLS) {
    // Iterative solvers on the group's Gram, one thread per group (same recurrences as the single-problem kernel,
    // k3_solve.cu; faer_coordinate_descent lr_solvers.rs:426-538, faer_nn_lr :542-600).  The ridge term l2 was added to
    // the diagonal above only for LSTSQ callers: CD scales its penalties by the row count itself.
    for (int i = 0; i < q; ++i) CN(i) = 0.0;                      // beta
    if (a.method == PDSB_METHOD_CD) {
      const double mcount = irls ? count : (double)nrows, lambda_l1 = mcount * l1, l2n = mcount * l2;
      const double y_sum = mom(midx(p, p + 1));
      for (int it = 0; it < a.max_iter; ++it) {
        double max_change = 0.0;
        for (int j = 0; j < p; ++j) {
          const double before = CN(j);
          double part = 0.0;
          for (int i = 0; i < q; ++i) if (i != j) part += AA(i, j) * CN(i);
          const double mu = BB(j) - part;
          double after;
          if (a.positive && mu < 0.0) after = 0.0;
          else {
            const double sgn = (mu > 0.0) ? 1.0 : ((mu < 0.0) ? -1.0 : 0.0);
            after = sgn * fmax(fabs(mu) - lambda_l1, 0.0) / (AA(j, j) + l2n);
          }
          CN(j) = after;
          max_change = fmax(max_change, fabs(after - before));
        }
        if (a.add_bias) {
          double part = 0.0;
          for (int j = 0; j < p; ++j) part += CN(j) * mom(midx(j, p + 1));
          CN(p) = (y_sum - part) / mcount;
        }
        if (max_change < a.cd_tol) break;
      }
    } else {
      // mu = G beta - X'y lives in the b slots (negated X'y to start with)
      for (int i = 0; i < q; ++i) BB(i) = -BB(i);
      for (int it = 0; it < a.max_iter; ++it) {
        bool ok = true;
        for (int i = 0; i < q; ++i) {
          const double mu = BB(i);
          if (!(mu >= -a.cd_tol)) ok = false;
          if (CN(i) > 0.0 && !(mu <= a.cd_tol)) ok = false;
        }
        if (ok) break;
        for (int k = 0; k < q; ++k) {
          const double bk = CN(k);
          double upd = bk - BB(k) / AA(k, k);
          if (!a.add_bias || k < q - 1) upd = fmax(upd, 0.0);
          const double diff = upd - bk;
          for (int i = 0; i < q; ++i) BB(i) += diff * AA(i, k);
          CN(k) = upd;
        }
      }
    }
    for (int i = 0; i < q; ++i) out[i] = CN(i);
    a.status[g] = PDSB_OK;
    return;
  }
  const bool gated = a.tol > 0.0;
  double ln_den = 0.0;
  if (gated) {
    for (int i = 0; i < q; ++i) {
      double d = AA(i, i);
      if (d <= 0.0) { a.status[g] = PDSB_GATED; for (int k = 0; k < q; ++k) out[k] = nan(""); return; }
      ln_den += log(d);
    }
    // NaN diagonal: the reference's comparisons are all false -> it solves and returns NaN coefficients (k3_solve.cu)
    if (isnan(ln_den)) { a.status[g] = PDSB_OK; for (int k = 0; k < q; ++k) out[k] = nan(""); return; }
  }
  const double ln_tol = gated ? log(a.tol) : 0.0;
  int perm[66];
  bool done = false;
  if (a.solver == PDSB_SOLVER_CHOLESKEY) {
    bool ok = true;
    double ln_det = 0.0;
    for (int k = 0; k < q && ok; ++k) {
      double d = AA(k, k);
      if (!(d > 0.0) || !isfinite(d)) { ok = false; break; }
      d = sqrt(d); AA(k, k) = d; ln_det += 2.0 * log(d);
      for (int i = k + 1; i < q; ++i) AA(i, k) = AA(i, k) / d;
      for (int j = k + 1; j < q; ++j) { double ljk = AA(j, k); for (int i = j; i < q; ++i) AA(i, j) -= AA(i, k) * ljk; }
    }
    if (ok) {
      if (gated && ln_det - ln_den <= ln_tol) { a.status[g] = PDSB_GATED; for (int k = 0; k < q; ++k) out[k] = nan(""); return; }
      for (int i = 0; i < q; ++i) { double s = BB(i); for (int j = 0; j < i; ++j) s -= AA(i, j) * BB(j); BB(i) = s / AA(i, i); }
      for (int i = q - 1; i >= 0; --i) { double s = BB(i); for (int j = i + 1; j < q; ++j) s -= AA(j, i) * BB(j); BB(i) = s / AA(i, i); }
      for (int i = 0; i < q; ++i) out[i] = BB(i);
      done = true;
    } else if (gated) {
      a.status[g] = PDSB_GATED; for (int k = 0; k < q; ++k) out[k] = nan(""); return;
    } else {  // restore and fall through to QR (lr_solvers.rs:288-291)
      for (int j = 0; j < q; ++j)
        for (int i = 0; i <= j; ++i) {
          double v = mom(midx(fz(i), fz(j)));
          if (a.method == PDSB_METHOD_LSTSQ && i == j && i < p && l2 > 0.0) v += l2;   // ridge; CD scales l2 by n itself
          AA(i, j) = v; AA(j, i) = v;
        }
      for (int i = 0; i < q; ++i) BB(i) = mom(midx(fz(i), p));
    }
  }
  if (!done) {
    // Householder QR with column pivoting
    for (int j = 0; j < q; ++j) perm[j] = j;
    double ln_det = 0.0;
    for (int k = 0; k < q; ++k) {
      int piv = k; double best = -1.0;
      for (int j = k; j < q; ++j) {
        double s = 0.0;
        for (int i = k; i < q; ++i) { double v = AA(i, j); s += v * v; }
        CN(j) = s;
        if (s > best) { best = s; piv = j; }
      }
      if (piv != k) {
        for (int i = 0; i < q; ++i) { double t = AA(i, k); AA(i, k) = AA(i, piv); AA(i, piv) = t; }
        int t = perm[k]; perm[k] = perm[piv]; perm[piv] = t;
      }
      double s = CN(piv);
      double normx = sqrt(s), x0 = AA(k, k);
      double alpha = (x0 >= 0.0) ? -normx : normx;
      double v0 = x0 - alpha;
      double vtv = v0 * v0 + (s - x0 * x0);
      double hb = (vtv > 0.0 && isfinite(vtv)) ? 2.0 / vtv : 0.0;
      if (hb != 0.0) {
        for (int j = k + 1; j < q; ++j) {
          double dot = v0 * AA(k, j);
          for (int i = k + 1; i < q; ++i) dot += AA(i, k) * AA(i, j);
          double f = hb * dot;
          AA(k, j) -= f * v0;
          for (int i = k + 1; i < q; ++i) AA(i, j) -= f * AA(i, k);
        }
        double dot = v0 * BB(k);
        for (int i = k + 1; i < q; ++i) dot += AA(i, k) * BB(i);
        double f = hb * dot;
        BB(k) -= f * v0;
        for (int i = k + 1; i < q; ++i) BB(i) -= f * AA(i, k);
      }
      AA(k, k) = alpha;
      ln_det += log(fabs(alpha));
    }
    if (gated && ln_det - ln_den <= ln_tol) {
      a.status[g] = PDSB_GATED; for (int k = 0; k < q; ++k) out[k] = nan(""); return;
    }
    for (int i = q - 1; i >= 0; --i) {
      double s = BB(i);
      for (int j = i + 1; j < q; ++j) s -= AA(i, j) * BB(j);
      double r = AA(i, i);
      BB(i) = (r != 0.0) ? s / r : 0.0;
    }
    for (int i = 0; i < q; ++i) out[perm[i]] = BB(i);
  }
  a.status[g] = PDSB_OK;
#undef AA
#undef BB
#undef CN
}

}  // namespace pdsb
