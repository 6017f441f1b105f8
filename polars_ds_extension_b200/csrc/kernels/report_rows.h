// The two rules of lin_reg_report that K9 (k9_report.cu, one frame) and K17 (k17_grouped_report.cu, every group of a
// frame) share, so that each is stated once:
//   hc_weight       the per-row HC weight  omega = e^2 * {1, 1/(1-h), 1/(1-h)^2},  h = x G^-1 x^T, all in T;
//   report_column   column i of the 8 x q report block from n, SSR, var(y), beta, G^-1 and (HC) the meat.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "special.h"

namespace pdsb {

// se_type: 0 se, 1..4 hc0..hc3.  x(a): the row's value of coefficient a (1 for the bias); g(a, b): G^-1[a][b] as T.
// hc0 / hc1 (and se) read neither.
template <typename T, typename XF, typename GF>
__device__ __forceinline__ T hc_weight(T e, int q, int se_type, XF x, GF g) {
  T wgt = e * e;
  if (se_type >= 3) {   // hc2, hc3 need the leverage
    T h = T(0);
    for (int a = 0; a < q; ++a) {
      const T xa = x(a);
      T inner = T(0);
      for (int b = 0; b < q; ++b) inner = fma(g(a, b), x(b), inner);
      h = fma(xa, inner, h);
    }
    T d = T(1) - h;
    wgt = (se_type == 4) ? wgt / (d * d) : wgt / d;
  }
  return wgt;
}

// Column i of the report of a fit of q coefficients on n rows: out[r * q + i] for the rows beta, se, t, p>|t|, 0.025,
// 0.975, r2, adj_r2.  se_type 0 (or a weighted fit): se = sqrt(mse G^-1[i][i]) with mse = mse_ssr / (n - q); hc0..hc3:
// the sandwich G^-1 meat G^-1, meat(r, c) = sum omega z_r z_c over coefficients r, c, times n / (n - q) for hc1.
// r2 = 1 - ssr / (y_var n) (the reference multiplies the ddof = 1 variance by n, linear_regression.rs:867).
// t_alpha = student_t_ppf(0.975, n - q), computed once per fit by the caller.
template <typename Meat>
__device__ __forceinline__ void report_column(int i, int q, int se_type, double n, double ssr, double mse_ssr,
                                              double y_var, double t_alpha, const double* __restrict__ beta,
                                              const double* __restrict__ ginv, Meat meat, double* __restrict__ o) {
  const double dof = n - (double)q;
  const double ratio = ssr / (y_var * n);
  const double r2 = 1.0 - ratio;
  const double adj_r2 = 1.0 - ratio * ((n - 1.0) / (dof - 1.0));
  double se;
  if (se_type == 0) {
    const double mse = mse_ssr / dof;
    se = sqrt(mse * ginv[(size_t)i * q + i]);
  } else {
    double v = 0.0;
    for (int r = 0; r < q; ++r) {
      double inner = 0.0;
      for (int c = 0; c < q; ++c) inner += meat(r, c) * ginv[(size_t)c * q + i];
      v += ginv[(size_t)i * q + r] * inner;
    }
    if (se_type == 2) v *= n / (n - (double)q);
    se = sqrt(v);
  }
  const double b = beta[i];
  const double t = b / se;
  const double pval = 2.0 * student_t_sf(fabs(t), dof);
  o[0 * q + i] = b;
  o[1 * q + i] = se;
  o[2 * q + i] = t;
  o[3 * q + i] = pval;
  o[4 * q + i] = b - t_alpha * se;
  o[5 * q + i] = b + t_alpha * se;
  o[6 * q + i] = r2;
  o[7 * q + i] = adj_r2;
}

}  // namespace pdsb
