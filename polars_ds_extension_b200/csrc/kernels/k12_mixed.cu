// K12 — MixedModel: the random-intercept linear mixed model fitted by REML (reference: fit_reml and profile,
// /root/reference/src/linear/mixed/mod.rs:121-272).
//
// With C = [X | y] (q = p + 1 columns), H^-1 = (I + gamma Z Z')^-1, group g of n_g rows with mean row m_g, and the
// within-group scatter W = sum_g sum_{i in g} (c_i - m_g)(c_i - m_g)', exactly
//     C' H^-1 C = W + sum_c c / (1 + gamma c) B_c,   B_c = sum_{g : n_g = c} m_g m_g',
//     ln det H  = sum_c N_c ln(1 + gamma c)                                   (N_c groups of size c).
// Every term is positive semi-definite, so nothing cancels, and one pass over the rows gives everything REML needs.
//   order        stable radix sort of (code, row) -> the row map the upload's gather uses, and the group offsets
//   group pass   K5's work list and item moments with every row shifted by its group's first row (exact zeros for a
//                column constant within a group); group_summary -> m_g and W in a fixed order
//   centring     when column 0 of X is the ones column, every other column and y are centred on their global mean
//                before the buckets: X -> X T with T unit-triangular, so the deviance is unchanged, and the offsets
//                that would cancel in the Cholesky (a feature or target far from zero next to its spread) are gone
//   buckets      groups sorted by size (radix sort), one run per distinct size -> (c, N_c, B_c), each run summed in
//                segments of at most SEG groups by many blocks, then the segments in order
//   search       one CTA runs the reference's golden-section loop; each evaluation assembles C'H^-1C from W and the
//                buckets (O(D q^2), D distinct sizes) and takes its Cholesky: ln det X'HiX from L_XX, r'Hir = L_yy^2,
//                beta by back-substitution.  Then the standard errors and the containment degrees of freedom.
// f64 throughout, as the reference.  Bit-reproducible: every sum has a fixed order that depends only on the data.
#include <cfloat>
#include <cmath>
#include <cub/cub.cuh>

#include "../common.h"
#include "../host/host.h"
#include "kernels.h"

namespace pdsb {

namespace {

constexpr int NT = 256;            // threads of the summary / bucket kernels
constexpr int RT = 256;            // threads of the search CTA
constexpr int SUM_BLOCKS = 512;    // groups are dealt to at most this many blocks for W: the order depends on n_groups only
constexpr int64_t SEG = 256;       // groups per bucket segment (a segment never crosses a run)

// packed upper-triangular (i <= j) index tables over q columns, in shared memory
__device__ __forceinline__ void pack_tables(int q, unsigned char* ti, unsigned char* tj) {
  const int nq = q * (q + 1) / 2;
  for (int k = threadIdx.x; k < nq; k += blockDim.x) {
    int i = 0, rem = k;
    while (rem >= q - i) { rem -= q - i; ++i; }
    ti[k] = (unsigned char)i;
    tj[k] = (unsigned char)(i + rem);
  }
}

__global__ void iota_kernel(int64_t* __restrict__ v, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) v[i] = i;
}

// offsets[g] = first position of code g in the sorted codes (lower bound), offsets[n_groups] = n
__global__ void offsets_kernel(const int64_t* __restrict__ sorted, int64_t n, int64_t n_groups, int64_t* __restrict__ offsets) {
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g <= n_groups; g += (int64_t)gridDim.x * blockDim.x) {
    int64_t lo = 0, hi = n;
    while (lo < hi) { const int64_t mid = (lo + hi) >> 1; if (sorted[mid] < g) lo = mid + 1; else hi = mid; }
    offsets[g] = lo;
  }
}

// Block b takes groups [b per_block, (b+1) per_block) in order.  Per group: S_c (shifted sums) and the count from the item
// partials, m_g = first row + S / n_g, and W_g = Q_g - S S' / n_g added to the block's partial W.  An empty group has
// m_g = 0 and adds nothing.  The block also adds up n_g m_g (for the column means; its partial is [nq + q] wide) and
// clears *ones when a group's mean of column 0 is not exactly 1 (column 0 is then not the intercept).
__global__ void __launch_bounds__(NT)
group_summary_kernel(const double* __restrict__ part, int64_t n_items, const int64_t* __restrict__ item_start,
                     const int64_t* __restrict__ offsets, const double* __restrict__ Z, int64_t ld, int64_t n_groups, int p,
                     int64_t per_block, double* __restrict__ mg, int64_t* __restrict__ sz, double* __restrict__ wpart,
                     int* __restrict__ ones) {
  extern __shared__ __align__(16) unsigned char k12_smem[];
  const int q = p + 1, q1 = p + 2, nq = q * (q + 1) / 2;
  double* Wb = reinterpret_cast<double*>(k12_smem);      // [nq]
  double* S = Wb + nq;                                   // [q]
  double* Mb = S + q;                                    // [q]
  unsigned char* ti = reinterpret_cast<unsigned char*>(Mb + q);
  unsigned char* tj = ti + nq;
  pack_tables(q, ti, tj);
  for (int k = threadIdx.x; k < nq; k += blockDim.x) Wb[k] = 0.0;
  for (int c = threadIdx.x; c < q; c += blockDim.x) Mb[c] = 0.0;
  auto midx = [&](int i, int j) { return i * q1 - i * (i - 1) / 2 + (j - i); };   // K5's packing over [X, y, 1]
  const int64_t g0 = (int64_t)blockIdx.x * per_block, g1 = min(g0 + per_block, n_groups);
  __syncthreads();
  for (int64_t g = g0; g < g1; ++g) {
    const int64_t f = offsets[g], len = offsets[g + 1] - f;
    if (threadIdx.x == 0) sz[g] = len;
    if (len == 0) {
      for (int c = threadIdx.x; c < q; c += blockDim.x) mg[g * q + c] = 0.0;
      continue;
    }
    const int64_t it0 = item_start[g], it1 = item_start[g + 1];
    const double nd = (double)len;
    for (int c = threadIdx.x; c < q; c += blockDim.x) {
      double s = 0.0;
      for (int64_t it = it0; it < it1; ++it) s += part[(size_t)midx(c, p + 1) * n_items + it];
      S[c] = s;
      const double m = Z[(int64_t)c * ld + f] + s / nd;
      mg[g * q + c] = m;
      Mb[c] += nd * m;
      if (c == 0 && m != 1.0) *ones = 0;
    }
    __syncthreads();
    for (int k = threadIdx.x; k < nq; k += blockDim.x) {
      const int i = ti[k], j = tj[k];
      double Q = 0.0;
      for (int64_t it = it0; it < it1; ++it) Q += part[(size_t)midx(i, j) * n_items + it];
      Wb[k] += Q - S[i] * S[j] / nd;
    }
    __syncthreads();
  }
  for (int k = threadIdx.x; k < nq; k += blockDim.x) wpart[(size_t)blockIdx.x * (nq + q) + k] = Wb[k];
  for (int c = threadIdx.x; c < q; c += blockDim.x) wpart[(size_t)blockIdx.x * (nq + q) + nq + c] = Mb[c];
}

// W = the block partials added in block order; mu = W + nq: the centring shift, the column means of [X | y] except
// column 0 (0 there, and everywhere when column 0 is not the ones column)
__global__ void w_reduce_kernel(const double* __restrict__ wpart, int nb, int nq, int q, int64_t n,
                                const int* __restrict__ ones, double* __restrict__ W) {
  for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < nq + q; k += gridDim.x * blockDim.x) {
    double v = 0.0;
    for (int b = 0; b < nb; ++b) v += wpart[(size_t)b * (nq + q) + k];
    if (k >= nq) v = (k == nq || !*ones) ? 0.0 : v / (double)n;
    W[k] = v;
  }
}

// segments: run r (groups [t0, t1) of the size-sorted list) is cut at multiples of SEG, nseg[r] pieces
__global__ void seg_count_kernel(const int64_t* __restrict__ run_start, const int64_t* __restrict__ run_cnt,
                                 const int64_t* __restrict__ num_runs, int64_t* __restrict__ nseg) {
  const int64_t D = *num_runs;
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < D; r += (int64_t)gridDim.x * blockDim.x) {
    const int64_t t0 = run_start[r], t1 = t0 + run_cnt[r];
    nseg[r] = (t1 - 1) / SEG - t0 / SEG + 1;
  }
}

// segment partials: P_s = sum over the segment's groups, in group order, of (m_g - mu)(m_g - mu)'
__global__ void __launch_bounds__(NT)
seg_sum_kernel(const int64_t* __restrict__ run_start, const int64_t* __restrict__ run_cnt, const int64_t* __restrict__ num_runs,
               const int64_t* __restrict__ nseg, const int64_t* __restrict__ seg_base, const int64_t* __restrict__ gid,
               const double* __restrict__ mg, const double* __restrict__ mu, int q, double* __restrict__ P) {
  extern __shared__ __align__(16) unsigned char k12_smem[];
  const int nq = q * (q + 1) / 2;
  unsigned char* ti = k12_smem;
  unsigned char* tj = ti + nq;
  pack_tables(q, ti, tj);
  __syncthreads();
  const int64_t D = *num_runs, S = seg_base[D - 1] + nseg[D - 1];
  for (int64_t sg = blockIdx.x; sg < S; sg += gridDim.x) {
    int64_t lo = 0, hi = D;                              // the run of segment sg: seg_base[r] <= sg < seg_base[r + 1]
    while (hi - lo > 1) { const int64_t mid = (lo + hi) >> 1; if (seg_base[mid] <= sg) lo = mid; else hi = mid; }
    const int64_t t0 = run_start[lo], t1 = t0 + run_cnt[lo], j = sg - seg_base[lo];
    const int64_t a = max(t0, (t0 / SEG + j) * SEG), b = min(t1, (t0 / SEG + j + 1) * SEG);
    for (int k = threadIdx.x; k < nq; k += blockDim.x) {
      const int i = ti[k], jj = tj[k];
      const double mi = mu[i], mj = mu[jj];
      double v = 0.0;
      for (int64_t t = a; t < b; ++t) {
        const double* m = mg + gid[t] * q;
        v += (m[i] - mi) * (m[jj] - mj);
      }
      P[(size_t)sg * nq + k] = v;
    }
  }
}

// B_r = the segments of run r added in order
__global__ void run_reduce_kernel(const int64_t* __restrict__ num_runs, const int64_t* __restrict__ nseg,
                                  const int64_t* __restrict__ seg_base, const double* __restrict__ P, int nq,
                                  double* __restrict__ B) {
  const int64_t D = *num_runs;
  for (int64_t r = blockIdx.x; r < D; r += gridDim.x)
    for (int k = threadIdx.x; k < nq; k += blockDim.x) {
      double v = 0.0;
      for (int64_t sg = seg_base[r]; sg < seg_base[r] + nseg[r]; ++sg) v += P[(size_t)sg * nq + k];
      B[(size_t)r * nq + k] = v;
    }
}

struct RemlArgs {
  const double* W;          // [nq] packed over [X | y], then mu [q] (the centring shift)
  const double* B;          // [D][nq]
  const int64_t* run_size;  // [D] distinct group sizes, ascending
  const int64_t* run_cnt;   // [D] groups of that size
  const int64_t* num_runs;  // D
  int64_t n, n_groups, max_iter;
  int p;
  double tol;
  const uint8_t* between;   // [p]
  double* wts;              // [D] scratch: c / (1 + gamma c) of the evaluation in progress
  double* out;
};

struct Golden;

struct RemlShared {
  double* A;     // [q][q] row-major, lower triangle used
  double* M;     // [p][p] scratch (inverse columns, rank blocks)
  double* d0;    // [p]
  double* red;   // [RT]
  unsigned char *ti, *tj;
  int* flag;
  Golden* gs;
};

// the golden-section state; phase = what x is: 0 fc and 1 fe of the start, 2 fc / 3 fe of a step, 4 the optimum
struct Golden {
  double lo, hi, c, e, fc, fe, x;
  int64_t it, evals;
  int phase;
  __device__ static double phi() { return (sqrt(5.0) - 1.0) / 2.0; }
  // record f = deviance(x) and choose the next x (fit_reml's loop: `for _ in 0..max_iter { if hi - lo < tol break; ...}`)
  __device__ void step(double f, int64_t max_iter, double tol) {
    ++evals;
    if (phase == 4) return;
    if (phase == 0) { fc = f; phase = 1; x = e; return; }
    if (phase == 2) fc = f; else fe = f;
    if (it < max_iter && !(hi - lo < tol)) {
      ++it;
      if (fc < fe) {
        hi = e; e = c; fe = fc;
        c = __dsub_rn(hi, __dmul_rn(phi(), __dsub_rn(hi, lo)));
        x = c; phase = 2;
      } else {
        lo = c; c = e; fc = fe;
        e = __dadd_rn(lo, __dmul_rn(phi(), __dsub_rn(hi, lo)));
        x = e; phase = 3;
      }
    } else {
      x = __dmul_rn(__dadd_rn(lo, hi), 0.5);
      phase = 4;
    }
  }
};

__device__ __forceinline__ double block_sum(double v, double* red) {
  red[threadIdx.x] = v;
  __syncthreads();
  for (int off = RT / 2; off; off >>= 1) {
    if ((int)threadIdx.x < off) red[threadIdx.x] += red[threadIdx.x + off];
    __syncthreads();
  }
  const double r = red[0];
  __syncthreads();
  return r;
}

// profile(gamma) of the reference: returns PDSB_MIXED_* and leaves the Cholesky factor of C'H^-1C in A
// (L_XX, the y row L_yX, and r'Hir in A(p, p)); *dev = the REML deviance
__device__ __forceinline__ int reml_profile(const RemlArgs& a, const RemlShared& sh, double gamma, double* dev) {
  const int p = a.p, q = p + 1, nq = q * (q + 1) / 2;
  const int64_t D = *a.num_runs;
  double* A = sh.A;
  double part = 0.0;
  for (int64_t r = threadIdx.x; r < D; r += blockDim.x) {
    const double c = (double)a.run_size[r], h = __dadd_rn(1.0, __dmul_rn(gamma, c));
    a.wts[r] = c / h;
    part += (double)a.run_cnt[r] * log(h);
  }
  const double ln_det_h = block_sum(part, sh.red);     // its barriers also publish the weights
  for (int k = threadIdx.x; k < nq; k += blockDim.x) {
    double v = a.W[k];
    for (int64_t r = 0; r < D; ++r) v += a.wts[r] * a.B[(size_t)r * nq + k];
    A[sh.tj[k] * q + sh.ti[k]] = v;
  }
  __syncthreads();
  for (int k = 0; k < p; ++k) {
    if (threadIdx.x == 0) {
      const double d = A[k * q + k];
      *sh.flag = d > 0.0;                              // faer's LLT fails on a pivot that is not > 0 (NaN included)
      if (d > 0.0) A[k * q + k] = sqrt(d);
    }
    __syncthreads();
    if (!*sh.flag) return PDSB_MIXED_NOT_PD;
    const double piv = A[k * q + k];
    for (int i = k + 1 + threadIdx.x; i < q; i += blockDim.x) A[i * q + k] /= piv;
    __syncthreads();
    const int m = q - k - 1;
    for (int t = threadIdx.x; t < m * m; t += blockDim.x) {
      const int i = k + 1 + t / m, j = k + 1 + t % m;
      if (j <= i) A[i * q + j] -= A[i * q + k] * A[j * q + k];
    }
    __syncthreads();
  }
  const double rv = A[p * q + p] / (double)(a.n - p);
  if (!(rv > 0.0)) return PDSB_MIXED_RESID_VAR;
  double ld = 0.0;
  for (int k = 0; k < p; ++k) ld += log(fabs(A[k * q + k]));
  *dev = (double)(a.n - p) * log(rv) + ln_det_h + 2.0 * ld;
  return PDSB_MIXED_OK;
}

// rank of the symmetric m x m matrix in M (row-major, overwritten) by Cholesky with diagonal pivoting: a pivot at or
// below abs_tol, or at or below rel * its column's starting diagonal, ends the count
__device__ __forceinline__ int pivoted_rank(const RemlShared& sh, double* M, int m, double abs_tol, double rel) {
  for (int i = threadIdx.x; i < m; i += blockDim.x) sh.d0[i] = M[i * m + i];
  __syncthreads();
  int rank = 0;
  for (int k = 0; k < m; ++k) {
    if (threadIdx.x == 0) {
      int piv = k;
      for (int t = k + 1; t < m; ++t) if (M[t * m + t] > M[piv * m + piv]) piv = t;
      const double d = M[piv * m + piv];
      *sh.flag = d > abs_tol && d > rel * sh.d0[piv];
      if (*sh.flag && piv != k) {
        for (int t = 0; t < m; ++t) { const double x = M[k * m + t]; M[k * m + t] = M[piv * m + t]; M[piv * m + t] = x; }
        for (int t = 0; t < m; ++t) { const double x = M[t * m + k]; M[t * m + k] = M[t * m + piv]; M[t * m + piv] = x; }
        const double x = sh.d0[k]; sh.d0[k] = sh.d0[piv]; sh.d0[piv] = x;
      }
      if (*sh.flag) M[k * m + k] = sqrt(M[k * m + k]);
    }
    __syncthreads();
    if (!*sh.flag) break;
    ++rank;
    const double piv = M[k * m + k];
    for (int i = k + 1 + threadIdx.x; i < m; i += blockDim.x) M[i * m + k] /= piv;
    __syncthreads();
    const int r = m - k - 1;
    for (int t = threadIdx.x; t < r * r; t += blockDim.x) {
      const int i = k + 1 + t / r, j = k + 1 + t % r;
      M[i * m + j] -= M[i * m + k] * M[j * m + k];
    }
    __syncthreads();
  }
  __syncthreads();
  return rank;
}

__global__ void __launch_bounds__(RT) reml_kernel(RemlArgs a) {
  extern __shared__ __align__(16) unsigned char k12_smem[];
  const int p = a.p, q = p + 1, nq = q * (q + 1) / 2;
  RemlShared sh;
  sh.red = reinterpret_cast<double*>(k12_smem);      // the fixed-size parts first: constant addresses
  sh.gs = reinterpret_cast<Golden*>(sh.red + RT);
  sh.flag = reinterpret_cast<int*>(sh.gs + 1);
  sh.A = reinterpret_cast<double*>(sh.flag + 2);
  sh.M = sh.A + q * q;
  sh.d0 = sh.M + p * p;
  sh.ti = reinterpret_cast<unsigned char*>(sh.d0 + p);
  sh.tj = sh.ti + nq;
  pack_tables(q, sh.ti, sh.tj);
  __syncthreads();
  double* out = a.out;
  // golden section exactly as fit_reml (mod.rs:196-222).  Thread 0 keeps the state in shared memory (so that it is
  // not live in registers across the evaluations); the explicit roundings keep the compiler from fusing these products
  // and sums, so lo / hi / c / e follow the reference's arithmetic.
  Golden& gs = *sh.gs;
  if (threadIdx.x == 0) {
    gs.lo = 0.0; gs.hi = 1e6;
    gs.c = __dsub_rn(gs.hi, __dmul_rn(gs.phi(), __dsub_rn(gs.hi, gs.lo)));
    gs.e = __dadd_rn(gs.lo, __dmul_rn(gs.phi(), __dsub_rn(gs.hi, gs.lo)));
    gs.x = gs.c; gs.it = 0; gs.evals = 0; gs.phase = 0;
  }
  __syncthreads();
  int st;
  for (;;) {           // one call site keeps a single copy of the profile code
    double f = 0.0;
    st = reml_profile(a, sh, gs.x, &f);
    const int phase = gs.phase;
    __syncthreads();
    if (threadIdx.x == 0) gs.step(f, a.max_iter, a.tol);
    __syncthreads();
    if (st || phase == 4) break;
  }
  const double gamma = gs.x;
  const int64_t evals = gs.evals;
  if (threadIdx.x == 0) { out[3 * p] = gamma; out[3 * p + 2] = (double)evals; out[3 * p + 3] = (double)st; }
  if (st) return;
  const double* A = sh.A;
  const double* mu = a.W + nq;
  const double rv = A[p * q + p] / (double)(a.n - p);
  if (threadIdx.x == 0) {
    out[3 * p + 1] = rv;
    // beta of the centred design: L_XX' beta = L_yX'; then the intercept of the original one,
    // beta_0 = beta'_0 - sum_j mu_j beta_j + mu_y (mu_0 = 0)
    for (int i = p - 1; i >= 0; --i) {
      double s = A[p * q + i];
      for (int j = i + 1; j < p; ++j) s -= A[j * q + i] * out[j];
      out[i] = s / A[i * q + i];
    }
    double b0 = out[0];
    for (int j = 1; j < p; ++j) b0 -= mu[j] * out[j];
    out[0] = b0 + mu[p];
  }
  // diag((X'HiX)^-1)_j = |column j of L_XX^-1|^2: thread j solves L x = e_j into column j of M
  for (int j = threadIdx.x; j < p; j += blockDim.x) {
    double* x = sh.M;
    double ss = 0.0;
    for (int i = j; i < p; ++i) {
      double s = i == j ? 1.0 : 0.0;
      for (int k = j; k < i; ++k) s -= A[i * q + k] * x[k * p + j];
      const double v = s / A[i * q + i];
      x[i * p + j] = v;
      ss += v * v;
    }
    out[p + j] = sqrt(rv * ss);
  }
  // the intercept's variance a' (X'HiX)^-1 a with a = (1, -mu_1, .., -mu_{p-1}): |L^-1 a|^2
  if (threadIdx.x == 0) {
    double ss = 0.0;
    for (int i = 0; i < p; ++i) {
      double s = i == 0 ? 1.0 : -mu[i];
      for (int k = 0; k < i; ++k) s -= A[i * q + k] * sh.d0[k];
      const double v = s / A[i * q + i];
      sh.d0[i] = v;
      ss += v * v;
    }
    out[p] = sqrt(rv * ss);
  }
  __syncthreads();

  // containment degrees of freedom (mod.rs:239-259) without Z: the Gram of the centred X is W + sum_c c B_c, and of X
  // itself G(i,j) + mu_i s_j + mu_j s_i + mu_i mu_j n with s_j = G(0,j) (row 0 of the ones column); rank([X | Z]) =
  // non-empty groups + rank(W_XX).  Pivot thresholds: (1e-9 R00)^2 with R00 the largest column norm of the matrix whose
  // QR the reference ranks, and q eps times the column's starting diagonal.
  const int64_t D = *a.num_runs;
  double* G = sh.A;                                          // full Gram of [X | y], row-major q x q
  for (int k = threadIdx.x; k < nq; k += blockDim.x) {
    double v = a.W[k];
    for (int64_t r = 0; r < D; ++r) v += (double)a.run_size[r] * a.B[(size_t)r * nq + k];
    G[sh.ti[k] * q + sh.tj[k]] = v;
    G[sh.tj[k] * q + sh.ti[k]] = v;
  }
  __syncthreads();
  for (int j = threadIdx.x; j < p; j += blockDim.x) sh.d0[j] = G[j];
  __syncthreads();
  for (int k = threadIdx.x; k < nq; k += blockDim.x) {
    const int i = sh.ti[k], j = sh.tj[k];
    if (j >= p) continue;
    const double v = G[i * q + j] + mu[i] * sh.d0[j] + mu[j] * sh.d0[i] + mu[i] * mu[j] * sh.d0[0];
    G[i * q + j] = v;
    G[j * q + i] = v;
  }
  __syncthreads();
  const double rel = (double)q * DBL_EPSILON;
  // between columns
  int mb = 0;
  for (int j = 0; j < p; ++j) mb += a.between[j] ? 1 : 0;
  double r00b = 0.0;
  for (int i = 0, bi = 0; i < p; ++i) {
    if (!a.between[i]) continue;
    r00b = fmax(r00b, G[i * q + i]);
    for (int t = threadIdx.x; t < p; t += blockDim.x)
      if (a.between[t]) {
        int bj = 0;
        for (int u = 0; u < t; ++u) bj += a.between[u] ? 1 : 0;
        sh.M[bi * mb + bj] = G[i * q + t];
      }
    ++bi;
  }
  __syncthreads();
  const int rank_b = (mb == 0 || !(r00b > 0.0)) ? 0 : pivoted_rank(sh, sh.M, mb, 1e-18 * r00b, rel);
  // within block of W, and the largest column norm of [X | Z]
  const int64_t nonempty = a.n_groups - (a.run_size[0] == 0 ? a.run_cnt[0] : 0);
  double r00c = (double)a.run_size[D - 1];
  for (int i = 0; i < p; ++i) r00c = fmax(r00c, G[i * q + i]);
  for (int k = threadIdx.x; k < nq; k += blockDim.x) {
    const int i = sh.ti[k], j = sh.tj[k];
    if (j < p) { sh.M[i * p + j] = a.W[k]; sh.M[j * p + i] = a.W[k]; }
  }
  __syncthreads();
  const int rank_w = !(r00c > 0.0) ? 0 : pivoted_rank(sh, sh.M, p, 1e-18 * r00c, rel);
  if (threadIdx.x == 0)
    for (int j = 0; j < p; ++j)
      out[2 * p + j] = a.between[j] ? (double)(a.n_groups - rank_b) : (double)(a.n - (nonempty + rank_w));
}

int64_t key_bits(int64_t max_key) {
  int b = 1;
  while (b < 63 && (max_key >> b) != 0) ++b;
  return b;
}

}  // namespace

int mixed_order_rows(const int64_t* codes, int64_t n, int64_t n_groups, int64_t* rows, int64_t* offsets, cudaStream_t s) {
  DevBag bag(s);
  int64_t* idx = bag.alloc<int64_t>((size_t)n);
  int64_t* sorted = bag.alloc<int64_t>((size_t)n);
  if (!idx || !sorted) return 1;
  iota_kernel<<<(unsigned)std::max<int64_t>(1, std::min<int64_t>(ceil_div(n, 256), 4096)), 256, 0, s>>>(idx, n);
  PDSB_LAUNCH_OK();
  count_launch();
  const int bits = (int)key_bits(n_groups - 1);
  size_t tb = 0;
  PDSB_CUDA_OK(cub::DeviceRadixSort::SortPairs(nullptr, tb, codes, sorted, idx, rows, n, 0, bits, s));
  void* tmp = bag.alloc<unsigned char>(tb);
  if (!tmp) return 1;
  PDSB_CUDA_OK(cub::DeviceRadixSort::SortPairs(tmp, tb, codes, sorted, idx, rows, n, 0, bits, s));
  offsets_kernel<<<(unsigned)std::max<int64_t>(1, std::min<int64_t>(ceil_div(n_groups + 1, 256), 4096)), 256, 0, s>>>(
      sorted, n, n_groups, offsets);
  PDSB_LAUNCH_OK();
  count_launch();
  return 0;
}

int mixed_reml(const double* Z, int64_t ld, const int64_t* offsets, int64_t G, int64_t n, int p, const uint8_t* between,
               int64_t max_iter, double tol, double* out, cudaStream_t s) {
  const int q = p + 1, q1 = p + 2, nq = q * (q + 1) / 2, nm = q1 * (q1 + 1) / 2;
  const int64_t n_items = group_items_bound(n, G);
  const int64_t per_block = ceil_div(G, SUM_BLOCKS);
  const int nb = (int)ceil_div(G, per_block);
  // distinct positive sizes sum to at most n, so D (D + 1) / 2 <= n; one more for the empty groups
  const int64_t dmax = std::min<int64_t>(G, (int64_t)std::sqrt(2.0 * (double)n) + 2);
  DevBag bag(s);
  double* part = bag.alloc<double>((size_t)nm * n_items);
  double* mg = bag.alloc<double>((size_t)G * q);
  int64_t* sz = bag.alloc<int64_t>((size_t)G);
  int64_t* sz_sorted = bag.alloc<int64_t>((size_t)G);
  int64_t* gid = bag.alloc<int64_t>((size_t)G);
  int64_t* gid_sorted = bag.alloc<int64_t>((size_t)G);
  int64_t* runs = bag.alloc<int64_t>((size_t)3 * G + 1);    // run_size, run_cnt, run_start, num_runs
  const int64_t smax = dmax + ceil_div(G, SEG);                  // segments: at most one per run plus one per SEG cut
  double* wpart = bag.alloc<double>((size_t)nb * (nq + q));
  double* W = bag.alloc<double>((size_t)nq + q);
  double* B = bag.alloc<double>((size_t)dmax * nq);
  double* P = bag.alloc<double>((size_t)smax * nq);
  double* wts = bag.alloc<double>((size_t)dmax);
  int64_t* segs = bag.alloc<int64_t>((size_t)2 * dmax);          // nseg, seg_base
  int* ones = bag.alloc<int>(1);
  if (!part || !mg || !sz || !sz_sorted || !gid || !gid_sorted || !runs || !wpart || !W || !B || !P || !wts ||
      !segs || !ones)
    return 1;
  int64_t *nseg = segs, *seg_base = segs + dmax;
  int64_t *run_size = runs, *run_cnt = runs + G, *run_start = runs + 2 * G, *num_runs = runs + 3 * G;

  GroupWork wl;
  if (build_work_list(offsets, G, n, ItemCount::BOUND, ItemMaps::NONE, bag, wl, s) ||
      group_moments_shifted(Z, ld, Z + (size_t)p * ld, offsets, G, p, wl, part, s))
    return 1;
  const int one = 1;
  PDSB_CUDA_OK(cudaMemcpyAsync(ones, &one, sizeof(int), cudaMemcpyHostToDevice, s));
  const size_t sm_sum = ((size_t)nq + 2 * q) * sizeof(double) + 2 * (size_t)nq;
  if (sm_sum > 48 * 1024) PDSB_CUDA_OK(cudaFuncSetAttribute(group_summary_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm_sum));
  group_summary_kernel<<<nb, NT, sm_sum, s>>>(part, n_items, wl.item_start, offsets, Z, ld, G, p, per_block, mg, sz, wpart, ones);
  PDSB_LAUNCH_OK();
  count_launch();
  w_reduce_kernel<<<(unsigned)ceil_div(nq + q, 256), 256, 0, s>>>(wpart, nb, nq, q, n, ones, W);
  PDSB_LAUNCH_OK();
  count_launch();

  // size buckets: groups sorted by size (stable: group order within a size), one run per distinct size
  iota_kernel<<<(unsigned)std::max<int64_t>(1, std::min<int64_t>(ceil_div(G, 256), 4096)), 256, 0, s>>>(gid, G);
  PDSB_LAUNCH_OK();
  count_launch();
  PDSB_CUDA_OK(cudaMemsetAsync(run_cnt, 0, (size_t)G * sizeof(int64_t), s));
  const int bits = (int)key_bits(n);
  PDSB_CUDA_OK(cudaMemsetAsync(nseg, 0, (size_t)dmax * sizeof(int64_t), s));
  size_t tb_sort = 0, tb_rle = 0, tb_scan = 0, tb_seg = 0;
  PDSB_CUDA_OK(cub::DeviceRadixSort::SortPairs(nullptr, tb_sort, sz, sz_sorted, gid, gid_sorted, G, 0, bits, s));
  PDSB_CUDA_OK(cub::DeviceRunLengthEncode::Encode(nullptr, tb_rle, sz_sorted, run_size, run_cnt, num_runs, (int)G, s));
  PDSB_CUDA_OK(cub::DeviceScan::ExclusiveSum(nullptr, tb_scan, run_cnt, run_start, G, s));
  PDSB_CUDA_OK(cub::DeviceScan::ExclusiveSum(nullptr, tb_seg, nseg, seg_base, dmax, s));
  void* tmp = bag.alloc<unsigned char>(std::max(std::max(tb_sort, tb_seg), std::max(tb_rle, tb_scan)));
  if (!tmp) return 1;
  PDSB_CUDA_OK(cub::DeviceRadixSort::SortPairs(tmp, tb_sort, sz, sz_sorted, gid, gid_sorted, G, 0, bits, s));
  PDSB_CUDA_OK(cub::DeviceRunLengthEncode::Encode(tmp, tb_rle, sz_sorted, run_size, run_cnt, num_runs, (int)G, s));
  PDSB_CUDA_OK(cub::DeviceScan::ExclusiveSum(tmp, tb_scan, run_cnt, run_start, G, s));
  seg_count_kernel<<<(unsigned)ceil_div(dmax, 256), 256, 0, s>>>(run_start, run_cnt, num_runs, nseg);
  PDSB_LAUNCH_OK();
  count_launch();
  PDSB_CUDA_OK(cub::DeviceScan::ExclusiveSum(tmp, tb_seg, nseg, seg_base, dmax, s));
  seg_sum_kernel<<<(unsigned)std::min<int64_t>(smax, 4096), NT, 2 * (size_t)nq, s>>>(run_start, run_cnt, num_runs, nseg, seg_base,
                                                                                     gid_sorted, mg, W + nq, q, P);
  PDSB_LAUNCH_OK();
  count_launch();
  run_reduce_kernel<<<(unsigned)std::min<int64_t>(dmax, 1024), NT, 0, s>>>(num_runs, nseg, seg_base, P, nq, B);
  PDSB_LAUNCH_OK();
  count_launch();

  RemlArgs a;
  a.W = W; a.B = B; a.run_size = run_size; a.run_cnt = run_cnt; a.num_runs = num_runs;
  a.n = n; a.n_groups = G; a.max_iter = max_iter; a.p = p; a.tol = tol; a.between = between; a.wts = wts; a.out = out;
  const size_t sm_reml = ((size_t)q * q + (size_t)p * p + p + RT + 1) * sizeof(double) + sizeof(Golden) + 2 * (size_t)nq;
  if (sm_reml > 48 * 1024) PDSB_CUDA_OK(cudaFuncSetAttribute(reml_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm_reml));
  reml_kernel<<<1, RT, sm_reml, s>>>(a);
  PDSB_LAUNCH_OK();
  count_launch();
  return 0;
}

}  // namespace pdsb
