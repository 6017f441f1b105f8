// K14 — smooth_spline: the cubic smoothing spline of pl_smooth_spline as an O(n) partitioned band solve.
//
// The reference (src/num_ext/splines.rs:33-97) builds dense Q (n x n-2), R^-1 Q' and M = I + lambda Q R^-1 Q' and runs a
// dense Cholesky of M: O(n^2) memory, O(n^3) time.  Here the same g comes from the Reinsch form
//   (R + lambda Q'Q) gamma = Q'y,   g = y - lambda Q gamma,
// whose matrix A (m = n - 2 unknowns) is SPD and pentadiagonal, every band a closed form of four consecutive x.
// A pentadiagonal matrix is block tridiagonal with 2 x 2 blocks (unknowns 2i, 2i+1 form block i; an odd m gets one
// decoupled unknown with A = 1, rhs = 0, gamma = 0), and the whole solve works on that form:
//   * the blocks are cut into partitions of LB blocks; the last block of every partition but the last one is a
//     separator, the others are its interior;
//   * pass 1 (one thread per partition): one forward block-LDL' sweep over the interior, carrying the fill towards the
//     left separator, gives the partition's Schur complement contribution on its two separators (14 doubles);
//   * the separators form a block-tridiagonal SPD system of P - 1 blocks, solved by the same two passes one level up
//     (the level's blocks are read from the partition outputs below it) until one partition is left;
//   * pass 2 (one thread per partition): with both separator values known the interior is a standalone block
//     tridiagonal system: forward sweep (G r and G C kept in shared memory), backward sweep, then the output — at level
//     0 g itself through the stencil g_k = y_k - lambda (a_k gamma_k + b_{k-1} gamma_{k-1} + c_{k-2} gamma_{k-2}).
// Every sum has a fixed order and no atomics touch data, so a repeated call is bit-identical.  DESIGN.md "K14 in detail"
// has the byte count and the choices.
//
// ptxas (-Xptxas -v, sm_90a, CUDA 12.9): see DESIGN.md "K14 in detail"; no stack frame and no spill in any kernel.
#include "../common.h"
#include "kernels.h"
#include <cmath>
#include <vector>

namespace pdsb {
namespace {

constexpr int LB = 16;     // 2 x 2 blocks per partition (32 unknowns at level 0)
constexpr int NT = 64;     // threads (= partitions) per CTA
constexpr int NF = 14;     // doubles per partition output (see pass 1)
constexpr int NS = 6;      // shared-memory doubles per block in pass 2: u = G r (2), Z = G C (4)

// Partition output fields (structure of arrays, stride = number of partitions):
//   0-2 DR  D of the right separator + this partition's Schur term (sym: 00, 01, 11)    3-4 rR  its rhs
//   5-7 DL  this partition's Schur term on its left separator (sym)                    8-9 rL  its rhs term
//   10-13 CLR  coupling left separator -> right separator (row-major 2 x 2)
enum { F_DR = 0, F_RR = 3, F_DL = 5, F_RL = 8, F_C = 10 };

// Level 0: block i of A and its rhs straight from x, y (h_j = x_{j+1} - x_j, r_j = 1 / h_j; row j of Q' is
// a_j = r_j, b_j = -(r_j + r_{j+1}), c_j = r_{j+1} at columns j, j+1, j+2).
// D = A[2i..2i+1, 2i..2i+1] (sym), C = A[2i..2i+1, 2i+2..2i+3] (row-major), r = (Q'y)[2i..2i+1].
struct Src0 {
  const double* __restrict__ x;
  const double* __restrict__ y;
  int64_t n, m;
  double lam;
  __device__ __forceinline__ void get(int64_t i, double D[3], double C[4], double r[2]) const {
    const int64_t j0 = 2 * i;
    double hh[4], rr[4];
    double xp = __ldg(x + min(j0, n - 1));
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      if (j0 + t <= n - 2) {
        const double xn = __ldg(x + j0 + t + 1);
        hh[t] = xn - xp;
        rr[t] = __drcp_rn(hh[t]);
        xp = xn;
      } else {
        hh[t] = 0.0; rr[t] = 0.0;
      }
    }
    double dd[2], ee[2], ff[2], bb[2];
#pragma unroll
    for (int t = 0; t < 2; ++t) {
      const int64_t j = j0 + t;
      if (j < m) {
        const double a = rr[t], b = -(rr[t] + rr[t + 1]), c = rr[t + 1];
        dd[t] = (hh[t] + hh[t + 1]) * (1.0 / 3.0) + lam * (a * a + b * b + c * c);
        ee[t] = j + 1 < m ? hh[t + 1] * (1.0 / 6.0) + lam * (b * rr[t + 1] + c * -(rr[t + 1] + rr[t + 2])) : 0.0;
        ff[t] = j + 2 < m ? lam * (c * rr[t + 2]) : 0.0;
        bb[t] = a * __ldg(y + j) + b * __ldg(y + j + 1) + c * __ldg(y + j + 2);
      } else {
        dd[t] = 1.0; ee[t] = 0.0; ff[t] = 0.0; bb[t] = 0.0;
      }
    }
    D[0] = dd[0]; D[1] = ee[0]; D[2] = dd[1];
    C[0] = ff[0]; C[1] = 0.0; C[2] = ee[1]; C[3] = ff[1];
    r[0] = bb[0]; r[1] = bb[1];
  }
};

// Level >= 1: block k is separator k of the level below, assembled from the partition outputs there (stride S).
struct SrcR {
  const double* __restrict__ po;
  int64_t S;
  __device__ __forceinline__ void get(int64_t k, double D[3], double C[4], double r[2]) const {
#pragma unroll
    for (int f = 0; f < 3; ++f) D[f] = po[(F_DR + f) * S + k] + po[(F_DL + f) * S + k + 1];
#pragma unroll
    for (int f = 0; f < 2; ++f) r[f] = po[(F_RR + f) * S + k] + po[(F_RL + f) * S + k + 1];
#pragma unroll
    for (int f = 0; f < 4; ++f) C[f] = po[(F_C + f) * S + k + 1];
  }
};

// 2 x 2 SPD block: D = L diag(d0, d1) L', L = [[1, 0], [l, 1]]; f = (1/d0, l, 1/d1)
struct Fac { double i0, l, i1; };
__device__ __forceinline__ Fac factor(const double D[3]) {
  Fac f;
  f.i0 = __drcp_rn(D[0]);
  f.l = D[1] * f.i0;
  f.i1 = __drcp_rn(D[2] - f.l * D[1]);
  return f;
}
// w = D^-1 v
__device__ __forceinline__ void gsolve(const Fac& f, double v0, double v1, double& w0, double& w1) {
  const double z1 = v1 - f.l * v0;
  w1 = z1 * f.i1;
  w0 = v0 * f.i0 - f.l * w1;
}

// x and y finite, x strictly increasing (h <= 0 is "not increasing"; a NaN gap is not, as in the reference)
__device__ __forceinline__ int check_rows(const double* x, const double* y, int64_t n, int64_t lo, int64_t hi) {
  int bad = 0;
  for (int64_t j = lo; j < hi; ++j) {
    const double xj = __ldg(x + j);
    if (!isfinite(xj) || !isfinite(__ldg(y + j))) bad |= PDSB_SPLINE_NONFINITE;
    if (j + 1 < n && __ldg(x + j + 1) - xj <= 0.0) bad |= PDSB_SPLINE_NOT_INCREASING;
  }
  return bad;
}

// rows [lo, hi) of level 0 belong to partition k: 2 LB k .. 2 LB (k + 1), the last partition up to n
__device__ __forceinline__ void part_rows(int64_t k, int64_t P, int64_t n, int64_t& lo, int64_t& hi) {
  lo = 2 * (int64_t)LB * k;
  hi = k == P - 1 ? n : min(n, lo + 2 * (int64_t)LB);
}

template <class Src>
__global__ void __launch_bounds__(NT)
spline_pass1(Src src, int64_t M, int64_t P, double* __restrict__ po, const double* __restrict__ x,
             const double* __restrict__ y, int64_t n, int* status) {
  const int64_t k = (int64_t)blockIdx.x * NT + threadIdx.x;
  if (k >= P) return;
  if (x) {                                         // level 0 checks its input rows
    int64_t lo, hi;
    part_rows(k, P, n, lo, hi);
    const int bad = check_rows(x, y, n, lo, hi);
    if (bad) atomicOr(status, bad);
  }
  if (P == 1) return;
  const int64_t b0 = k * LB;
  const bool has_l = k > 0, has_r = k < P - 1;
  const int ni = has_r ? LB - 1 : (int)(M - b0);
  double D[3], C[4], r[2];
  double W[4] = {0.0, 0.0, 0.0, 0.0};             // fill: A'[interior block i, left separator], row-major
  double DL[3] = {0.0, 0.0, 0.0}, rL[2] = {0.0, 0.0};
  double out[NF];
#pragma unroll
  for (int f = 0; f < NF; ++f) out[f] = 0.0;
  if (has_l) {
    src.get(b0 - 1, D, C, r);
    W[0] = C[0]; W[1] = C[2]; W[2] = C[1]; W[3] = C[3];     // A[I_0, S_L] = C_sep'
  }
  src.get(b0, D, C, r);
  double Dt[3] = {D[0], D[1], D[2]}, rt[2] = {r[0], r[1]};
  for (int i = 0; i < ni; ++i) {
    const Fac f = factor(Dt);
    double u0, u1;
    gsolve(f, rt[0], rt[1], u0, u1);
    double Y[4] = {0.0, 0.0, 0.0, 0.0};           // G W
    if (has_l) {
      gsolve(f, W[0], W[2], Y[0], Y[2]);
      gsolve(f, W[1], W[3], Y[1], Y[3]);
      DL[0] -= W[0] * Y[0] + W[2] * Y[2];
      DL[1] -= W[0] * Y[1] + W[2] * Y[3];
      DL[2] -= W[1] * Y[1] + W[3] * Y[3];
      rL[0] -= W[0] * u0 + W[2] * u1;
      rL[1] -= W[1] * u0 + W[3] * u1;
    }
    const bool last = i + 1 == ni;
    if (last && !has_r) break;
    const double Cc[4] = {C[0], C[1], C[2], C[3]};
    double Z[4];                                   // G C
    gsolve(f, Cc[0], Cc[2], Z[0], Z[2]);
    gsolve(f, Cc[1], Cc[3], Z[1], Z[3]);
    src.get(b0 + i + 1, D, C, r);                  // next interior block, or the right separator
    Dt[0] = D[0] - (Cc[0] * Z[0] + Cc[2] * Z[2]);
    Dt[1] = D[1] - (Cc[0] * Z[1] + Cc[2] * Z[3]);
    Dt[2] = D[2] - (Cc[1] * Z[1] + Cc[3] * Z[3]);
    rt[0] = r[0] - (Cc[0] * u0 + Cc[2] * u1);
    rt[1] = r[1] - (Cc[1] * u0 + Cc[3] * u1);
    if (!last) {
      if (has_l) {                                 // W <- -C' G W
        W[0] = -(Cc[0] * Y[0] + Cc[2] * Y[2]);
        W[1] = -(Cc[0] * Y[1] + Cc[2] * Y[3]);
        W[2] = -(Cc[1] * Y[0] + Cc[3] * Y[2]);
        W[3] = -(Cc[1] * Y[1] + Cc[3] * Y[3]);
      }
      continue;
    }
    out[F_DR + 0] = Dt[0]; out[F_DR + 1] = Dt[1]; out[F_DR + 2] = Dt[2];
    out[F_RR + 0] = rt[0]; out[F_RR + 1] = rt[1];
    if (has_l) {                                   // -(G W)' C
      out[F_C + 0] = -(Y[0] * Cc[0] + Y[2] * Cc[2]);
      out[F_C + 1] = -(Y[0] * Cc[1] + Y[2] * Cc[3]);
      out[F_C + 2] = -(Y[1] * Cc[0] + Y[3] * Cc[2]);
      out[F_C + 3] = -(Y[1] * Cc[1] + Y[3] * Cc[3]);
    }
  }
  out[F_DL + 0] = DL[0]; out[F_DL + 1] = DL[1]; out[F_DL + 2] = DL[2];
  out[F_RL + 0] = rL[0]; out[F_RL + 1] = rL[1];
#pragma unroll
  for (int f = 0; f < NF; ++f) po[f * P + k] = out[f];
}

// gnext: the level above's solution (2 per separator); level > 0 writes its own solution to gout, level 0 writes g.
template <class Src, bool L0>
__global__ void __launch_bounds__(NT)
spline_pass2(Src src, int64_t M, int64_t P, const double* __restrict__ gnext, double* __restrict__ gout,
             const double* __restrict__ x, const double* __restrict__ y, int64_t n, double lam,
             const int* __restrict__ status) {
  extern __shared__ double sm[];
  const int64_t k = (int64_t)blockIdx.x * NT + threadIdx.x;
  if (k >= P) return;
  double* slot = sm + threadIdx.x;                 // slot[(s * LB + i) * NT]
  auto S = [&](int s, int i) -> double& { return slot[(s * LB + i) * NT]; };
  if (L0 && *status != 0) {                        // invalid input: g is all NaN (the host reports the error)
    int64_t lo, hi;
    part_rows(k, P, n, lo, hi);
    for (int64_t j = lo; j < hi; ++j) gout[j] = NAN;
    return;
  }
  const int64_t b0 = k * LB;
  const bool has_l = k > 0, has_r = k < P - 1;
  const int ni = has_r ? LB - 1 : (int)(M - b0);
  double gl0 = 0.0, gl1 = 0.0, gr0 = 0.0, gr1 = 0.0;
  if (has_l) { gl0 = gnext[2 * (k - 1)]; gl1 = gnext[2 * (k - 1) + 1]; }
  if (has_r) { gr0 = gnext[2 * k]; gr1 = gnext[2 * k + 1]; }
  double D[3], C[4], r[2];
  double cl[4] = {0.0, 0.0, 0.0, 0.0};
  if (has_l) src.get(b0 - 1, D, cl, r);
  src.get(b0, D, C, r);
  double Dt[3] = {D[0], D[1], D[2]};
  double rt[2] = {r[0] - (cl[0] * gl0 + cl[2] * gl1), r[1] - (cl[1] * gl0 + cl[3] * gl1)};
  for (int i = 0; i < ni; ++i) {
    const bool last = i + 1 == ni;
    if (last && has_r) {                           // coupling to the known right separator
      rt[0] -= C[0] * gr0 + C[1] * gr1;
      rt[1] -= C[2] * gr0 + C[3] * gr1;
    }
    const Fac f = factor(Dt);
    double u0, u1;
    gsolve(f, rt[0], rt[1], u0, u1);
    S(0, i) = u0; S(1, i) = u1;
    if (last) break;
    const double Cc[4] = {C[0], C[1], C[2], C[3]};
    double Z[4];
    gsolve(f, Cc[0], Cc[2], Z[0], Z[2]);
    gsolve(f, Cc[1], Cc[3], Z[1], Z[3]);
    S(2, i) = Z[0]; S(3, i) = Z[1]; S(4, i) = Z[2]; S(5, i) = Z[3];
    src.get(b0 + i + 1, D, C, r);
    Dt[0] = D[0] - (Cc[0] * Z[0] + Cc[2] * Z[2]);
    Dt[1] = D[1] - (Cc[0] * Z[1] + Cc[2] * Z[3]);
    Dt[2] = D[2] - (Cc[1] * Z[1] + Cc[3] * Z[3]);
    rt[0] = r[0] - (Cc[0] * u0 + Cc[2] * u1);
    rt[1] = r[1] - (Cc[1] * u0 + Cc[3] * u1);
  }
  // backward: gamma_i = G r~_i - (G C_i) gamma_{i+1}; gamma overwrites u
  double n0 = S(0, ni - 1), n1 = S(1, ni - 1);
  for (int i = ni - 2; i >= 0; --i) {
    const double g0 = S(0, i) - (S(2, i) * n0 + S(3, i) * n1);
    const double g1 = S(1, i) - (S(4, i) * n0 + S(5, i) * n1);
    S(0, i) = g0; S(1, i) = g1;
    n0 = g0; n1 = g1;
  }
  if (!L0) {
    for (int i = 0; i < ni; ++i) { gout[2 * (b0 + i)] = S(0, i); gout[2 * (b0 + i) + 1] = S(1, i); }
    if (has_r) { gout[2 * (b0 + ni)] = gr0; gout[2 * (b0 + ni) + 1] = gr1; }
    return;
  }
  // g_j = y_j - lambda (a_j gamma_j + b_{j-1} gamma_{j-1} + c_{j-2} gamma_{j-2}), gamma_q = 0 outside [0, m)
  const int64_t m = n - 2, q0 = 2 * b0, q1 = 2 * (b0 + ni);
  auto gam = [&](int64_t q) -> double {
    if (q < 0 || q >= m) return 0.0;
    if (q < q0) return q == q0 - 2 ? gl0 : gl1;
    if (q >= q1) return q == q1 ? gr0 : gr1;
    return S((int)((q - q0) & 1), (int)((q - q0) >> 1));
  };
  int64_t lo, hi;
  part_rows(k, P, n, lo, hi);
  double rm1 = lo >= 1 ? __drcp_rn(__ldg(x + lo) - __ldg(x + lo - 1)) : 0.0;
  for (int64_t j = lo; j < hi; ++j) {
    const double r0 = j <= n - 2 ? __drcp_rn(__ldg(x + j + 1) - __ldg(x + j)) : 0.0;
    const double s = r0 * gam(j) + (-(rm1 + r0)) * gam(j - 1) + rm1 * gam(j - 2);
    gout[j] = __ldg(y + j) - lam * s;
    rm1 = r0;
  }
}

__global__ void spline_check_kernel(const double* __restrict__ x, const double* __restrict__ y, int64_t n, int mask,
                                    int* status) {
  int bad = 0;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += stride)
    bad |= check_rows(x, y, n, j, j + 1);
  bad &= mask;
  if (bad) atomicOr(status, bad);
}

int64_t parts_of(int64_t M) { return (M + LB - 1) / LB; }
int grid_of(int64_t P) { return (int)((P + NT - 1) / NT); }

}  // namespace

int smooth_spline_solve(const double* x, const double* y, int64_t n, double lam, double* g, int* status,
                        int64_t* reduced_blocks, cudaStream_t s) {
  PDSB_CUDA_OK(cudaMemsetAsync(status, 0, sizeof(int), s));
  if (lam == 0.0) {                                // I g = y: checks, then a copy
    const int grid = (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div(n, 256), (int64_t)sm_count() * 8));
    spline_check_kernel<<<grid, 256, 0, s>>>(x, y, n, PDSB_SPLINE_NOT_INCREASING, status);
    PDSB_LAUNCH_OK();
    count_launch();
    PDSB_CUDA_OK(cudaMemcpyAsync(g, y, (size_t)n * sizeof(double), cudaMemcpyDeviceToDevice, s));
    if (reduced_blocks) *reduced_blocks = 0;
    return 0;
  }
  // levels: M_0 = ceil(m / 2) blocks; P_l = ceil(M_l / LB) partitions; M_{l+1} = P_l - 1, until one partition
  std::vector<int64_t> Ms, Ps;
  for (int64_t M = (n - 2 + 1) / 2;;) {
    const int64_t P = parts_of(M);
    Ms.push_back(M); Ps.push_back(P);
    if (P == 1) break;
    M = P - 1;
  }
  const int L = (int)Ms.size();
  size_t total = 0;
  for (int l = 0; l + 1 < L; ++l) total += (size_t)NF * Ps[l] + 2 * (size_t)Ms[l + 1];
  if (reduced_blocks) { *reduced_blocks = 0; for (int l = 1; l < L; ++l) *reduced_blocks += Ms[l]; }
  double* base = nullptr;
  if (total && dev_alloc((void**)&base, total * sizeof(double), s)) return 1;
  std::vector<double*> po(L, nullptr), gam(L, nullptr);   // po[l]: partition outputs of level l; gam[l]: level l's solution
  for (size_t l = 0, off = 0; l + 1 < (size_t)L; ++l) {
    po[l] = base + off; off += (size_t)NF * Ps[l];
    gam[l + 1] = base + off; off += 2 * (size_t)Ms[l + 1];
  }
  const Src0 s0{x, y, n, n - 2, lam};
  const size_t smem = (size_t)NS * LB * NT * sizeof(double);
  int rc = 0;
  auto launched = [&]() { cudaError_t e = cudaGetLastError(); count_launch();
                          if (e != cudaSuccess) { set_error("smooth_spline launch failed: %s", cudaGetErrorString(e)); rc = 1; }
                          return rc == 0; };
  spline_pass1<Src0><<<grid_of(Ps[0]), NT, 0, s>>>(s0, Ms[0], Ps[0], po[0], x, y, n, status);
  if (!launched()) goto done;
  for (int l = 1; l < L; ++l) {
    if (Ps[l] == 1) break;
    spline_pass1<SrcR><<<grid_of(Ps[l]), NT, 0, s>>>(SrcR{po[l - 1], Ps[l - 1]}, Ms[l], Ps[l], po[l], nullptr, nullptr,
                                                      0, status);
    if (!launched()) goto done;
  }
  for (int l = L - 1; l >= 1; --l) {
    spline_pass2<SrcR, false><<<grid_of(Ps[l]), NT, smem, s>>>(SrcR{po[l - 1], Ps[l - 1]}, Ms[l], Ps[l],
                                                                l + 1 < L ? gam[l + 1] : nullptr, gam[l], nullptr,
                                                                nullptr, 0, 0.0, status);
    if (!launched()) goto done;
  }
  spline_pass2<Src0, true><<<grid_of(Ps[0]), NT, smem, s>>>(s0, Ms[0], Ps[0], L > 1 ? gam[1] : nullptr, g, x, y, n,
                                                             lam, status);
  launched();
done:
  if (base) dev_free(base, s);
  return rc;
}

}  // namespace pdsb
