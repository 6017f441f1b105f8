// Device layer of the C ABI (pdsb_dev_*): thin, typed wrappers over the kernel launchers.
#include "../common.h"
#include "../kernels/kernels.h"
#include "../kernels/special.h"
#include "host.h"

using namespace pdsb;

// PCA: Gram of X (f64 products and sums) then K13's eigen kernel.  With p >= 2 the last feature goes in as the one
// target: the moments of [X[:, :p-1] | x_p | 1] hold all of G in the same order, and the single-target DMMA kernel needs
// fewer tensor-core block pairs than [X | 1] (10 instead of 15 at p = 32).
template <typename T>
static int pca_gram_eigen(const T* X, int64_t ldx, const T* mask, int64_t n, int p, double* sigma, double* V, int* status,
                          cudaStream_t s) {
  const int q1 = p + 1, t = p >= 2 ? 1 : 0;
  DevBag bag(s);
  double* M = bag.alloc<double>((size_t)q1 * q1);
  if (!M) return 1;
  const T* last = t ? X + (size_t)(p - 1) * ldx : nullptr;
  if (moments<T>(MomentsPrecision::F64_PRODUCTS, X, ldx, last, ldx, nullptr, mask, n, p - t, t, M, s)) return 1;
  return pca_eigen(M, q1, p, sigma, V, status, s);
}

static int pca_check(int64_t n, int p, const void* sigma, const void* V, const void* status) {
  if (p < 1 || p > 259) { set_error("pca: %d features; between 1 and 259 are supported", p); return 1; }
  if (n < 0 || !sigma || !V || !status) { set_error("pca: invalid arguments"); return 1; }
  return 0;
}

static int project_check(int64_t n, int64_t ldo, int p, int k) {
  if (p < 1 || p > 259) { set_error("project: %d features; between 1 and 259 are supported", p); return 1; }
  if (k < 1 || k > p || n < 0 || ldo < n) { set_error("project: invalid arguments"); return 1; }
  return 0;
}

extern "C" {

const char* pdsb_last_error(void) { return get_error(); }
int pdsb_version(void) { return PDSB_VERSION; }
int64_t pdsb_kernel_launch_count(void) { return g_kernel_launches.load(); }
int pdsb_last_moments_path(void) { return last_moments_path(); }
int pdsb_last_online_path(void) { return last_online_path(); }
void pdsb_set_moments_path(int path) { force_moments_path(path); }
void pdsb_set_tc_variant(int v) { set_tc_mode(v); }
int pdsb_set_device(int device) {
  if (require_device()) return 1;
  PDSB_CUDA_OK(cudaSetDevice(device));
  return 0;
}

// host-callable special functions (unit-tested against scipy on the CPU; the same code runs in K9)
double pdsb_student_t_sf(double x, double df) { return student_t_sf(x, df); }
double pdsb_student_t_ppf(double p, double df) { return student_t_ppf(p, df); }

int pdsb_dev_moments_f32(const float* X, int64_t ldx, const float* Y, int64_t ldy, const float* w,
                         const float* mask, int64_t n, int p, int t, double* M, void* stream) {
  if (require_device()) return 1;
  return moments<float>(MomentsPrecision::TF32_ALLOWED, X, ldx, Y, ldy, w, mask, n, p, t, M, (cudaStream_t)stream);
}

int pdsb_dev_moments_f64(const double* X, int64_t ldx, const double* Y, int64_t ldy, const double* w,
                         const double* mask, int64_t n, int p, int t, double* M, void* stream) {
  if (require_device()) return 1;
  return moments<double>(MomentsPrecision::F64_ACCUM, X, ldx, Y, ldy, w, mask, n, p, t, M, (cudaStream_t)stream);
}

// ---- row-blocked frames ("native" layout of the f32 headline path): [block][column][PDSB_FRAME_ROWS] ----
size_t pdsb_frame_elems(int64_t n, int ncols) { return (size_t)((n + FRAME_ROWS - 1) / FRAME_ROWS) * FRAME_ROWS * (size_t)ncols; }

int pdsb_dev_frame_from_colmajor_f32(const float* src, int64_t ld, int64_t n, int ncols, float* frame, void* stream) {
  if (require_device()) return 1;
  return to_frame<float>(src, ld, n, ncols, frame, (cudaStream_t)stream);
}

int pdsb_dev_moments_frame_f32(const float* frame, int64_t n, int ncols, int xcol, int p, int ycol, int t,
                               const float* mask, double* M, void* stream) {
  if (require_device()) return 1;
  if (xcol < 0 || ycol < 0 || xcol + p > ncols || ycol + t > ncols) { set_error("moments_frame: columns out of range"); return 1; }
  return moments<float>(MomentsPrecision::TF32_ALLOWED, frame + (size_t)xcol * FRAME_ROWS, 0, frame + (size_t)ycol * FRAME_ROWS,
                        0, nullptr, mask, n, p, t, M, (cudaStream_t)stream, (int64_t)ncols * FRAME_ROWS);
}

int pdsb_dev_predict_frame_f32(const float* frame, int64_t n, int ncols, int xcol, int p, int ycol, int t, int add_bias,
                               const float* mask, const double* beta, const int* status, float* pred, float* resid,
                               int64_t ldo, uint8_t* valid, double* ssr, void* stream) {
  if (require_device()) return 1;
  if (xcol < 0 || ycol < 0 || xcol + p > ncols || ycol + t > ncols) { set_error("predict_frame: columns out of range"); return 1; }
  return predict_frame_f32(frame, n, ncols, xcol, p, ycol, t, add_bias, mask, beta, status, pred, resid, ldo, valid, ssr,
                           (cudaStream_t)stream);
}

int pdsb_dev_solve(const double* M, const pdsb_solve_opts* opts, double* beta, int* status, double* aux,
                   void* stream) {
  if (require_device()) return 1;
  if (!opts) { set_error("solve: null options"); return 1; }
  return solve_from_moments(M, *opts, beta, status, aux, (cudaStream_t)stream);
}

int pdsb_dev_predict_f32(const float* X, int64_t ldx, const float* Y, int64_t ldy, const float* w,
                         const float* mask, int64_t n, int p, int t, int add_bias, const double* beta,
                         const int* status, float* pred, float* resid, int64_t ldo, uint8_t* valid,
                         double* ssr, void* stream) {
  if (require_device()) return 1;
  return predict_resid<float>(X, ldx, Y, ldy, w, mask, n, p, t, add_bias, beta, status, pred, resid, ldo, valid,
                              ssr, (cudaStream_t)stream);
}
int pdsb_dev_predict_f64(const double* X, int64_t ldx, const double* Y, int64_t ldy, const double* w,
                         const double* mask, int64_t n, int p, int t, int add_bias, const double* beta,
                         const int* status, double* pred, double* resid, int64_t ldo, uint8_t* valid,
                         double* ssr, void* stream) {
  if (require_device()) return 1;
  return predict_resid<double>(X, ldx, Y, ldy, w, mask, n, p, t, add_bias, beta, status, pred, resid, ldo, valid,
                               ssr, (cudaStream_t)stream);
}

int pdsb_dev_grouped_lin_reg_f32(const float* X, int64_t ldx, const float* y, const int64_t* offsets,
                                 int64_t n_groups, int64_t n, int p, const pdsb_solve_opts* opts,
                                 double* beta, int* status, void* stream) {
  if (require_device()) return 1;
  return grouped_lin_reg<float>(X, ldx, y, offsets, n_groups, n, p, *opts, beta, status, (cudaStream_t)stream);
}
int pdsb_dev_grouped_lin_reg_f64(const double* X, int64_t ldx, const double* y, const int64_t* offsets,
                                 int64_t n_groups, int64_t n, int p, const pdsb_solve_opts* opts,
                                 double* beta, int* status, void* stream) {
  if (require_device()) return 1;
  return grouped_lin_reg<double>(X, ldx, y, offsets, n_groups, n, p, *opts, beta, status, (cudaStream_t)stream);
}

// group_by().agg(lin_reg(weights=w)): every group's weighted least squares
int pdsb_dev_grouped_wls_lin_reg_f32(const float* X, int64_t ldx, const float* y, const float* w, const int64_t* offsets,
                                     int64_t n_groups, int64_t n, int p, const pdsb_solve_opts* opts, double* beta,
                                     int* status, void* stream) {
  if (require_device()) return 1;
  return grouped_wls_lin_reg<float>(X, ldx, y, w, offsets, n_groups, n, p, *opts, beta, status, (cudaStream_t)stream);
}
int pdsb_dev_grouped_wls_lin_reg_f64(const double* X, int64_t ldx, const double* y, const double* w,
                                     const int64_t* offsets, int64_t n_groups, int64_t n, int p,
                                     const pdsb_solve_opts* opts, double* beta, int* status, void* stream) {
  if (require_device()) return 1;
  return grouped_wls_lin_reg<double>(X, ldx, y, w, offsets, n_groups, n, p, *opts, beta, status, (cudaStream_t)stream);
}

// group_by().agg(lin_reg(target=[...])): every group's multi-target fit from one read of [Y | X]
int pdsb_dev_grouped_lin_reg_multi_f32(const float* Z, int64_t ld, int t, int p, const int64_t* offsets,
                                       int64_t n_groups, int64_t n, const pdsb_solve_opts* opts, double* beta,
                                       int* status, void* stream) {
  if (require_device()) return 1;
  return grouped_lin_reg_multi<float>(Z, ld, t, p, offsets, n_groups, n, *opts, beta, status, (cudaStream_t)stream);
}
int pdsb_dev_grouped_lin_reg_multi_f64(const double* Z, int64_t ld, int t, int p, const int64_t* offsets,
                                       int64_t n_groups, int64_t n, const pdsb_solve_opts* opts, double* beta,
                                       int* status, void* stream) {
  if (require_device()) return 1;
  return grouped_lin_reg_multi<double>(Z, ld, t, p, offsets, n_groups, n, *opts, beta, status, (cudaStream_t)stream);
}

// group_by().agg(query_ar_coeffs(x, lag)): the lagged design of every group formed on chip from the one column
int pdsb_dev_grouped_ar_lin_reg_f32(const float* x, const float* mask, const int64_t* offsets, int64_t n_groups,
                                    int64_t n, int lag, const pdsb_solve_opts* opts, double* beta, int* status,
                                    void* stream) {
  if (require_device()) return 1;
  return grouped_ar_lin_reg<float>(x, mask, offsets, n_groups, n, lag, *opts, beta, status, (cudaStream_t)stream);
}
int pdsb_dev_grouped_ar_lin_reg_f64(const double* x, const double* mask, const int64_t* offsets, int64_t n_groups,
                                    int64_t n, int lag, const pdsb_solve_opts* opts, double* beta, int* status,
                                    void* stream) {
  if (require_device()) return 1;
  return grouped_ar_lin_reg<double>(x, mask, offsets, n_groups, n, lag, *opts, beta, status, (cudaStream_t)stream);
}

int pdsb_dev_grouped_predict_f32(const float* X, int64_t ldx, const float* y, const int64_t* offsets, int64_t n_groups,
                                 int64_t n, int p, int add_bias, const double* beta, const int* status, const float* mask,
                                 float* pred, float* resid, uint8_t* valid, void* stream) {
  if (require_device()) return 1;
  return grouped_predict<float>(X, ldx, y, offsets, n_groups, n, p, add_bias, beta, status, mask, pred, resid, valid,
                                (cudaStream_t)stream);
}
int pdsb_dev_grouped_predict_f64(const double* X, int64_t ldx, const double* y, const int64_t* offsets, int64_t n_groups,
                                 int64_t n, int p, int add_bias, const double* beta, const int* status, const double* mask,
                                 double* pred, double* resid, uint8_t* valid, void* stream) {
  if (require_device()) return 1;
  return grouped_predict<double>(X, ldx, y, offsets, n_groups, n, p, add_bias, beta, status, mask, pred, resid, valid,
                                 (cudaStream_t)stream);
}

int pdsb_dev_grouped_report_f32(const float* X, int64_t ldx, const float* y, const float* ymask, const int64_t* offsets,
                                int64_t n_groups, int64_t n, int p, int add_bias, int se_type, double* out, int* status,
                                void* stream) {
  if (require_device()) return 1;
  return grouped_report<float>(X, ldx, y, ymask, offsets, n_groups, n, p, add_bias, se_type, out, status,
                               (cudaStream_t)stream);
}
int pdsb_dev_grouped_report_f64(const double* X, int64_t ldx, const double* y, const double* ymask,
                                const int64_t* offsets, int64_t n_groups, int64_t n, int p, int add_bias, int se_type,
                                double* out, int* status, void* stream) {
  if (require_device()) return 1;
  return grouped_report<double>(X, ldx, y, ymask, offsets, n_groups, n, p, add_bias, se_type, out, status,
                                (cudaStream_t)stream);
}

int pdsb_dev_grouped_lin_reg_rcond_f32(const float* X, int64_t ldx, const float* y, const int64_t* offsets,
                                       int64_t n_groups, int64_t n, int p, const pdsb_solve_opts* opts, double* beta,
                                       double* sv, int* status, void* stream) {
  if (require_device()) return 1;
  return grouped_lin_reg_rcond<float>(X, ldx, y, offsets, n_groups, n, p, *opts, beta, sv, status,
                                      (cudaStream_t)stream);
}
int pdsb_dev_grouped_lin_reg_rcond_f64(const double* X, int64_t ldx, const double* y, const int64_t* offsets,
                                       int64_t n_groups, int64_t n, int p, const pdsb_solve_opts* opts, double* beta,
                                       double* sv, int* status, void* stream) {
  if (require_device()) return 1;
  return grouped_lin_reg_rcond<double>(X, ldx, y, offsets, n_groups, n, p, *opts, beta, sv, status,
                                       (cudaStream_t)stream);
}

int pdsb_dev_grouped_logistic_f64(const double* X, int64_t ldx, const double* y, const double* mask,
                                  const int64_t* offsets, int64_t n_groups, int64_t n, int p, int add_bias, double l1,
                                  double l2, double tol, int64_t max_iter, double* beta, int* status, int64_t* n_iter,
                                  void* stream) {
  if (require_device()) return 1;
  return grouped_logistic(X, ldx, y, mask, offsets, n_groups, n, p, add_bias, l1, l2, tol, max_iter, beta, status,
                          n_iter, (cudaStream_t)stream);
}

int pdsb_dev_grouped_glm_f64(const double* X, int64_t ldx, const double* y, const double* mask, const int64_t* offsets,
                             int64_t n_groups, int64_t n, int p, int add_bias, int family, double tol, int64_t max_iter,
                             double* beta, int* status, int64_t* n_iter, void* stream) {
  if (require_device()) return 1;
  return grouped_glm(X, ldx, y, mask, offsets, n_groups, n, p, add_bias, family, tol, max_iter, beta, status, n_iter,
                     (cudaStream_t)stream);
}

int pdsb_dev_online_lin_reg_f32(const float* X, int64_t ldx, const float* y, int64_t n, int p, int add_bias,
                                int64_t window, int64_t min_rows, int skip, double lambda, float* coeffs,
                                float* pred, uint8_t* valid, void* stream) {
  if (require_device()) return 1;
  return online_lin_reg<float>(X, ldx, y, n, p, add_bias, window, min_rows, skip, lambda, nullptr, 0, coeffs, pred, valid,
                               (cudaStream_t)stream);
}
int pdsb_dev_online_lin_reg_f64(const double* X, int64_t ldx, const double* y, int64_t n, int p, int add_bias,
                                int64_t window, int64_t min_rows, int skip, double lambda, double* coeffs,
                                double* pred, uint8_t* valid, void* stream) {
  if (require_device()) return 1;
  return online_lin_reg<double>(X, ldx, y, n, p, add_bias, window, min_rows, skip, lambda, nullptr, 0, coeffs, pred, valid,
                                (cudaStream_t)stream);
}

// recursive_lin_reg(...).over(key): every group's K6 passes in one launch sequence
int pdsb_dev_grouped_recursive_lin_reg_f32(const float* X, int64_t ldx, const float* y, int64_t n, int p, int add_bias,
                                           int64_t min_rows, double lambda, const int64_t* offsets, int64_t n_groups,
                                           const uint8_t* skip, float* coeffs, float* pred, uint8_t* valid,
                                           void* stream) {
  if (require_device()) return 1;
  return grouped_recursive_lin_reg<float>(X, ldx, y, offsets, skip, n_groups, n, p, add_bias, min_rows, lambda, coeffs,
                                          pred, valid, (cudaStream_t)stream);
}
int pdsb_dev_grouped_recursive_lin_reg_f64(const double* X, int64_t ldx, const double* y, int64_t n, int p, int add_bias,
                                           int64_t min_rows, double lambda, const int64_t* offsets, int64_t n_groups,
                                           const uint8_t* skip, double* coeffs, double* pred, uint8_t* valid,
                                           void* stream) {
  if (require_device()) return 1;
  return grouped_recursive_lin_reg<double>(X, ldx, y, offsets, skip, n_groups, n, p, add_bias, min_rows, lambda, coeffs,
                                           pred, valid, (cudaStream_t)stream);
}

// rolling_lin_reg over groups: every group's K6 passes in one launch sequence.  grouped_rolling_lin_reg refuses window < 1
// before any device work, so that message does not wait for the device check.
int pdsb_dev_grouped_rolling_lin_reg_f32(const float* X, int64_t ldx, const float* y, int64_t n, int p, int add_bias,
                                         int64_t window, int64_t min_rows, double lambda, const int64_t* offsets,
                                         int64_t n_groups, const uint8_t* skip, float* coeffs, float* pred,
                                         uint8_t* valid, void* stream) {
  if (window >= 1 && require_device()) return 1;
  return grouped_rolling_lin_reg<float>(X, ldx, y, offsets, skip, n_groups, n, p, add_bias, window, min_rows, lambda,
                                        coeffs, pred, valid, (cudaStream_t)stream);
}
int pdsb_dev_grouped_rolling_lin_reg_f64(const double* X, int64_t ldx, const double* y, int64_t n, int p, int add_bias,
                                         int64_t window, int64_t min_rows, double lambda, const int64_t* offsets,
                                         int64_t n_groups, const uint8_t* skip, double* coeffs, double* pred,
                                         uint8_t* valid, void* stream) {
  if (window >= 1 && require_device()) return 1;
  return grouped_rolling_lin_reg<double>(X, ldx, y, offsets, skip, n_groups, n, p, add_bias, window, min_rows, lambda,
                                         coeffs, pred, valid, (cudaStream_t)stream);
}

int pdsb_dev_recursive_shard_f32(const float* X, int64_t ldx, const float* y, int64_t n, int p, int add_bias,
                                 int64_t min_rows, int skip, double lambda, const double* m0, int64_t row0,
                                 float* coeffs, float* pred, uint8_t* valid, void* stream) {
  if (require_device()) return 1;
  return online_lin_reg<float>(X, ldx, y, n, p, add_bias, 0, min_rows, skip, lambda, m0, row0, coeffs, pred, valid,
                               (cudaStream_t)stream);
}
int pdsb_dev_recursive_shard_f64(const double* X, int64_t ldx, const double* y, int64_t n, int p, int add_bias,
                                 int64_t min_rows, int skip, double lambda, const double* m0, int64_t row0,
                                 double* coeffs, double* pred, uint8_t* valid, void* stream) {
  if (require_device()) return 1;
  return online_lin_reg<double>(X, ldx, y, n, p, add_bias, 0, min_rows, skip, lambda, m0, row0, coeffs, pred, valid,
                                (cudaStream_t)stream);
}

// pl_singular_values / pl_pca (pca.rs:39-78, 126-182): the SVD of X from the eigen-decomposition of X'X
int pdsb_dev_pca_f32(const float* X, int64_t ldx, const float* mask, int64_t n, int p, double* sigma, double* V,
                     int* status, void* stream) {
  if (require_device()) return 1;
  if (pca_check(n, p, sigma, V, status)) return 1;
  return pca_gram_eigen<float>(X, ldx, mask, n, p, sigma, V, status, (cudaStream_t)stream);
}
int pdsb_dev_pca_f64(const double* X, int64_t ldx, const double* mask, int64_t n, int p, double* sigma, double* V,
                     int* status, void* stream) {
  if (require_device()) return 1;
  if (pca_check(n, p, sigma, V, status)) return 1;
  return pca_gram_eigen<double>(X, ldx, mask, n, p, sigma, V, status, (cudaStream_t)stream);
}

// pl_principal_components (pca.rs:80-124): `mat * v`, first k columns
int pdsb_dev_project_f32(const float* X, int64_t ldx, int64_t n, int p, const double* V, int k, double* out,
                         int64_t ldo, void* stream) {
  if (require_device()) return 1;
  if (project_check(n, ldo, p, k)) return 1;
  return pca_project<float>(X, ldx, n, p, V, k, out, ldo, (cudaStream_t)stream);
}
int pdsb_dev_project_f64(const double* X, int64_t ldx, int64_t n, int p, const double* V, int k, double* out,
                         int64_t ldo, void* stream) {
  if (require_device()) return 1;
  if (project_check(n, ldo, p, k)) return 1;
  return pca_project<double>(X, ldx, n, p, V, k, out, ldo, (cudaStream_t)stream);
}

// group_by(key).agg(singular_values / pca), principal_components(...).over(key): K18
int pdsb_dev_grouped_pca_f32(const float* X, int64_t ldx, const float* mask, const int64_t* offsets, int64_t n_groups,
                             int64_t n, int p, int center, double* mean, double* sigma, double* V, int* status,
                             void* stream) {
  if (require_device()) return 1;
  return grouped_pca<float>(X, ldx, mask, offsets, n_groups, n, p, center, mean, sigma, V, status, (cudaStream_t)stream);
}
int pdsb_dev_grouped_pca_f64(const double* X, int64_t ldx, const double* mask, const int64_t* offsets, int64_t n_groups,
                             int64_t n, int p, int center, double* mean, double* sigma, double* V, int* status,
                             void* stream) {
  if (require_device()) return 1;
  return grouped_pca<double>(X, ldx, mask, offsets, n_groups, n, p, center, mean, sigma, V, status, (cudaStream_t)stream);
}
int pdsb_dev_grouped_project_f32(const float* X, int64_t ldx, const int64_t* offsets, int64_t n_groups, int64_t n,
                                 int p, const double* mean, const double* V, int k, double* out, int64_t ldo,
                                 void* stream) {
  if (require_device()) return 1;
  return grouped_project<float>(X, ldx, offsets, n_groups, n, p, mean, V, k, out, ldo, (cudaStream_t)stream);
}
int pdsb_dev_grouped_project_f64(const double* X, int64_t ldx, const int64_t* offsets, int64_t n_groups, int64_t n,
                                 int p, const double* mean, const double* V, int k, double* out, int64_t ldo,
                                 void* stream) {
  if (require_device()) return 1;
  return grouped_project<double>(X, ldx, offsets, n_groups, n, p, mean, V, k, out, ldo, (cudaStream_t)stream);
}

// pl_smooth_spline (splines.rs:33-97): the Reinsch band system instead of the dense n x n solve (K14)
int pdsb_dev_smooth_spline_f64(const double* x, const double* y, int64_t n, double lambda, double* g, int* status,
                               void* stream) {
  if (require_device()) return 1;
  if (n < 3 || !x || !y || !g || !status || !(lambda >= 0.0)) { set_error("smooth_spline: invalid arguments"); return 1; }
  return smooth_spline_solve(x, y, n, lambda, g, status, nullptr, (cudaStream_t)stream);
}

// pl_isotonic_regression (isotonic_regression.rs): PAVA over partitions, joined by a tree of bridge merges (K15)
int pdsb_dev_isotonic_f64(const double* y, const double* w, int64_t n, int increasing, double* out, int* status,
                          void* stream) {
  if (require_device()) return 1;
  if (n < 0 || (n > 0 && (!y || !out)) || !status) { set_error("isotonic_regression: invalid arguments"); return 1; }
  return isotonic_fit(y, w, n, increasing, out, status, (cudaStream_t)stream);
}

// isotonic_regression(...).over(key): every group's K15 fit in one launch sequence
int pdsb_dev_grouped_isotonic_f64(const double* y, const double* w, const int64_t* offsets, int64_t n_groups, int64_t n,
                                  int increasing, double* out, int* status, void* stream) {
  if (require_device()) return 1;
  if (n < 0 || n_groups < 0 || (n_groups > 0 && (!offsets || !status)) || (n > 0 && (!y || !out || n_groups < 1))) {
    set_error("isotonic_regression: invalid arguments"); return 1;
  }
  return grouped_isotonic_fit(y, w, offsets, n_groups, n, increasing, out, status, (cudaStream_t)stream);
}

int pdsb_dev_report_f32(const float* X, int64_t ldx, const float* y, const float* w, const float* mask,
                        int64_t n, int p, int add_bias, int se_type, double y_var, double* out, void* stream) {
  if (require_device()) return 1;
  return report_stats<float>(X, ldx, y, w, mask, n, p, add_bias, se_type, y_var, out, (cudaStream_t)stream);
}
int pdsb_dev_report_f64(const double* X, int64_t ldx, const double* y, const double* w, const double* mask,
                        int64_t n, int p, int add_bias, int se_type, double y_var, double* out, void* stream) {
  if (require_device()) return 1;
  return report_stats<double>(X, ldx, y, w, mask, n, p, add_bias, se_type, y_var, out, (cudaStream_t)stream);
}

}  // extern "C"
