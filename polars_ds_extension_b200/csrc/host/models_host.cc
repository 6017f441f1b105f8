// Dense-matrix host layer: the second caller of the solvers (SURVEY.md §8f rank 1).
//
// Reference: PyLR / PyElasticNet / PyOnlineLR (/root/reference/src/pymodels/py_lr.rs:21-224) wrap
// LR::fit -> faer_solve_lr (src/linear/lr/lr_solvers.rs:64-73, 296-308; ungated, ridge on the non-bias diagonal),
// ElasticNet::fit -> faer_coordinate_descent (:140-176), OnlineLR::fit -> faer_qr_lr_with_inv
// (src/linear/online_lr/lr_online_solvers.rs:100-143), OnlineLR::update -> woodbury_step (:62-90, 307-332) and
// LinearModel::predict (src/linear/lr/mod.rs:146-174), and PyGLM (src/pymodels/py_glm.rs:12-102) -> faer_irls
// (src/linear/glm/glm_solvers.rs:249-359); the error strings are LinalgErrors::to_string
// (src/linear/mod.rs:20-31).  Inputs are numpy float64 matrices (numpy_faer.rs:10-66).
//
// Everything numeric runs on the device: upload -> (transpose to the column-major frame) -> K2a moments -> K3 solve,
// K10 strided predict, K10 Woodbury update on device-resident state, and for GLM the K11 row pass + K2a + K3 per IRLS
// iteration; for MixedModel (src/linear/mixed/mod.rs:121-272) the group-ordered upload, the K5 group pass and the K12
// REML search.  No CPU arithmetic beyond the GLM stopping test on q coefficients, no fallback.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>

#include "../common.h"
#include "../kernels/kernels.h"
#include "host.h"
#include <mutex>

namespace pdsb {
namespace {

int check_matrix(const pdsb_matrix* m) {
  if (!m || m->n_rows < 0 || m->n_cols < 0 || (m->n_rows > 0 && m->n_cols > 0 && !m->data)) {
    set_error("Input is not contiguous or is empty");
    return 1;
  }
  return 0;
}

// Host matrix -> device.  C order (col_stride 1) lands row-major and is transposed by K10 into the column-major
// destination; F order (row_stride 1) is copied column by column with one strided DMA.  Returns the device view
// actually usable by a strided reader in (*view, *vrs, *vcs) when `colmajor_dst` is null (predict path).
int upload(const pdsb_matrix& m, double* colmajor_dst, int64_t ld, DevBag& bag, cudaStream_t s, const double** view,
           int64_t* vrs, int64_t* vcs) {
  const int64_t n = m.n_rows, p = m.n_cols;
  if (n == 0 || p == 0) return 0;
  if (m.col_stride == 1 && m.row_stride >= p) {
    double* raw = bag.alloc<double>((size_t)n * p);
    if (!raw) return 1;
    PDSB_CUDA_OK(cudaMemcpy2DAsync(raw, (size_t)p * 8, m.data, (size_t)m.row_stride * 8, (size_t)p * 8, (size_t)n,
                                   cudaMemcpyHostToDevice, s));
    if (colmajor_dst) return gather_colmajor(raw, p, 1, n, (int)p, nullptr, colmajor_dst, ld, s);
    *view = raw; *vrs = p; *vcs = 1;
    return 0;
  }
  if (m.row_stride == 1 && m.col_stride >= n) {
    double* dst = colmajor_dst;
    int64_t dld = ld;
    if (!dst) { dld = pad_ld(n); dst = bag.alloc<double>((size_t)dld * p); if (!dst) return 1; }
    PDSB_CUDA_OK(cudaMemcpy2DAsync(dst, (size_t)dld * 8, m.data, (size_t)m.col_stride * 8, (size_t)n * 8, (size_t)p,
                                   cudaMemcpyHostToDevice, s));
    if (!colmajor_dst) { *view = dst; *vrs = 1; *vcs = dld; }
    return 0;
  }
  if (p == 1 && m.row_stride >= 1) {   // a strided vector (a column of a C-order matrix)
    double* dst = colmajor_dst ? colmajor_dst : bag.alloc<double>((size_t)n);
    if (!dst) return 1;
    PDSB_CUDA_OK(cudaMemcpy2DAsync(dst, 8, m.data, (size_t)m.row_stride * 8, 8, (size_t)n, cudaMemcpyHostToDevice, s));
    if (!colmajor_dst) { *view = dst; *vrs = 1; *vcs = n; }
    return 0;
  }
  set_error("Input array is not contiguous.");
  return 1;
}

// The shape checks of LinearModel::fit (lr/mod.rs:122-126; ElasticNet also fits n < p, lr_solvers.rs:168-175) and the
// upload of X and y into one column-major block [X | y] with leading dimension pad_ld(n).  Returns it, or nullptr.
double* upload_xy(const pdsb_matrix& X, const pdsb_matrix& y, bool wide_ok, DevBag& bag, cudaStream_t s) {
  const int64_t n = X.n_rows, ld = pad_ld(n);
  const int p = (int)X.n_cols;
  if (n != y.n_rows || y.n_cols != 1) { set_error("Dimension mismatch."); return nullptr; }
  if (n == 0 || p == 0 || (!wide_ok && n < p)) { set_error("Not enough rows / columns."); return nullptr; }
  double* dZ = bag.alloc<double>((size_t)ld * (p + 1));
  const double* v; int64_t a, b;
  if (!dZ || upload(X, dZ, ld, bag, s, &v, &a, &b) || upload(y, dZ + (size_t)ld * p, ld, bag, s, &v, &a, &b)) return nullptr;
  return dZ;
}

// LinearModel::predict and GLM::predict after their checks: out = g^-1(X coeffs (+ bias, last)) with the canonical
// link of `family` (PDSB_GLM_GAUSSIAN: the identity).
int predict_rows(const pdsb_matrix& X, const double* coeffs, int n_coef, int has_bias, int family, double* out) {
  const int64_t n = X.n_rows;
  const int p = (int)X.n_cols;
  if (n == 0) return 0;
  cudaStream_t s;
  if (thread_stream(&s)) return 1;
  DevBag bag(s);
  double* dbeta = bag.alloc<double>((size_t)n_coef);
  double* dout = bag.alloc<double>((size_t)n);
  if (!dbeta || !dout) return 1;
  PDSB_CUDA_OK(cudaMemcpyAsync(dbeta, coeffs, (size_t)n_coef * sizeof(double), cudaMemcpyHostToDevice, s));
  const double* view = nullptr; int64_t rs = 0, cs = 0;
  if (p > 0 && upload(X, nullptr, 0, bag, s, &view, &rs, &cs)) return 1;
  if (predict_strided(view, rs, cs, n, p, dbeta, has_bias ? 1 : 0, dout, s, family)) return 1;
  PDSB_CUDA_OK(cudaMemcpyAsync(out, dout, (size_t)n * sizeof(double), cudaMemcpyDeviceToHost, s));
  PDSB_CUDA_OK(cudaStreamSynchronize(s));
  return 0;
}

}  // namespace
}  // namespace pdsb

using namespace pdsb;

struct pdsb_online_lr {
  int q, has_bias, device;
  double* inv;   // [q][q]
  double* w;     // [q]  (bias last)
  double* x;     // [q]  staging for one row
  bool fit;
  // the handle owns its stream and a lock: update / get / set from ANY thread are ordered on this one stream and never
  // race on inv / w / the single staging row (the Python OnlineLR object carries no thread affinity)
  cudaStream_t stream = nullptr;
  std::mutex mu;
};

extern "C" {

int pdsb_model_fit(int model, const pdsb_matrix* X, const pdsb_matrix* y, int add_bias, const char* solver,
                   double l1_reg, double l2_reg, double tol, int64_t max_iter, double* coeffs, double* inv) {
  if (require_device()) return 1;
  if (check_matrix(X) || check_matrix(y)) return 1;
  if (!coeffs || (model == PDSB_MODEL_ONLINE_LR && !inv)) { set_error("pdsb_model_fit: null output"); return 1; }
  cudaStream_t s;
  if (thread_stream(&s)) return 1;
  DevBag bag(s);
  double* dZ = upload_xy(*X, *y, model == PDSB_MODEL_ELASTIC_NET, bag, s);
  if (!dZ) return 1;
  const int64_t n = X->n_rows, ld = pad_ld(n);
  const int p = (int)X->n_cols, q = p + (add_bias ? 1 : 0);
  double* dM = bag.alloc<double>((size_t)(p + 2) * (p + 2));
  double* dbeta = bag.alloc<double>((size_t)q);
  double* daux = bag.alloc<double>((size_t)q * q + q);
  int* dstatus = bag.alloc<int>(2);
  if (!dM || !dbeta || !daux || !dstatus) return 1;
  if (moments<double>(MomentsPrecision::F64_ACCUM, dZ, ld, dZ + (size_t)ld * p, ld, nullptr, nullptr, n, p, 1, dM, s)) return 1;

  pdsb_solve_opts o{};
  o.p = p; o.t = 1; o.add_bias = add_bias ? 1 : 0; o.solver = solver_from_string(solver ? solver : "qr");
  o.singular_x_tol = 0.0;                       // the model classes never gate (faer_solve_lr, not _gated)
  if (model == PDSB_MODEL_LR) { o.method = PDSB_METHOD_LSTSQ; o.l2_reg = l2_reg; }
  else if (model == PDSB_MODEL_ELASTIC_NET) {
    o.method = PDSB_METHOD_CD; o.l1_reg = l1_reg; o.l2_reg = l2_reg; o.tol = tol; o.max_iter = (int)max_iter; o.positive = 0;
  } else if (model == PDSB_MODEL_ONLINE_LR) { o.method = PDSB_METHOD_INV; o.l2_reg = l2_reg; }
  else { set_error("pdsb_model_fit: unknown model %d", model); return 1; }
  if (solve_from_moments(dM, o, dbeta, dstatus, model == PDSB_MODEL_ONLINE_LR ? daux : nullptr, s)) return 1;
  PDSB_CUDA_OK(cudaMemcpyAsync(coeffs, dbeta, (size_t)q * sizeof(double), cudaMemcpyDeviceToHost, s));
  if (model == PDSB_MODEL_ONLINE_LR)
    PDSB_CUDA_OK(cudaMemcpyAsync(inv, daux, (size_t)q * q * sizeof(double), cudaMemcpyDeviceToHost, s));
  PDSB_CUDA_OK(cudaStreamSynchronize(s));
  return 0;
}

int pdsb_model_predict(const pdsb_matrix* X, const double* coeffs, int n_coef, int has_bias, double* out) {
  if (require_device()) return 1;
  if (check_matrix(X)) return 1;
  if (n_coef < 1 || !coeffs) { set_error("Matrix is not learned yet."); return 1; }      // lr/mod.rs:149-150
  const int p = n_coef - (has_bias ? 1 : 0);
  if (X->n_cols != p) { set_error("Dimension mismatch."); return 1; }                  // :147-148
  return predict_rows(*X, coeffs, n_coef, has_bias, PDSB_GLM_GAUSSIAN, out);
}

// GLM::fit -> faer_irls (glm_solvers.rs:196-216, 249-359).  Per iteration: the K11 row pass (weights and working
// response; the first one starts from y), the weighted moments [X | z | 1]' W [X | z | 1] (K2a), the QR solve on them
// (K3; the bias is the ones column) and a D2H copy of beta and the moments for the host-side stopping test.
int pdsb_glm_fit(const pdsb_matrix* X, const pdsb_matrix* y, int add_bias, int family, int64_t max_iter, double tol,
                 double* coeffs, int64_t* n_iter) {
  if (require_device()) return 1;
  if (check_matrix(X) || check_matrix(y)) return 1;
  if (!coeffs) { set_error("pdsb_glm_fit: null output"); return 1; }
  if (family < PDSB_GLM_GAUSSIAN || family > PDSB_GLM_GAMMA) { set_error("pdsb_glm_fit: unknown family %d", family); return 1; }
  cudaStream_t s;
  if (thread_stream(&s)) return 1;
  DevBag bag(s);
  double* dZ = upload_xy(*X, *y, false, bag, s);
  if (!dZ) return 1;
  const int64_t n = X->n_rows, ld = pad_ld(n);
  const int p = (int)X->n_cols, q = p + (add_bias ? 1 : 0), q1 = p + 2;
  const double* dy = dZ + (size_t)ld * p;
  double* dw = bag.alloc<double>((size_t)ld);
  double* dz = bag.alloc<double>((size_t)ld);
  double* dM = bag.alloc<double>((size_t)q1 * q1);
  double* dbeta = bag.alloc<double>((size_t)q);
  double* dmean = bag.alloc<double>(1);
  int* dstatus = bag.alloc<int>(2);
  if (!dw || !dz || !dM || !dbeta || !dmean || !dstatus) return 1;
  if (mean_values<double>(dy, n, dmean, s)) return 1;         // mean(y) of the start (glm_solvers.rs:272-277)

  pdsb_solve_opts o{};
  o.p = p; o.t = 1; o.add_bias = add_bias ? 1 : 0; o.method = PDSB_METHOD_LSTSQ; o.solver = PDSB_SOLVER_QR;
  o.singular_x_tol = 0.0;                                       // faer_weighted_lr: col_piv_qr, no ridge, no gate
  std::vector<double> hb(q, 0.0), hb_new(q), hM((size_t)q1 * q1);
  // coefficient / target index -> moments index (the ones column is the last one)
  auto mi = [&](int j) { return j < p ? j : (j == p ? p : p + 1); };
  int64_t it = 0;
  while (it < max_iter) {
    if (irls_rows(family, dZ, ld, dy, nullptr, n, p, o.add_bias, dbeta, it == 0 ? dmean : nullptr, dw, dz, nullptr,
                  nullptr, s)) return 1;
    ++it;
    if (moments<double>(MomentsPrecision::F64_ACCUM, dZ, ld, dz, ld, dw, nullptr, n, p, 1, dM, s)) return 1;
    if (solve_from_moments(dM, o, dbeta, dstatus, nullptr, s)) return 1;
    PDSB_CUDA_OK(cudaMemcpyAsync(hb_new.data(), dbeta, (size_t)q * sizeof(double), cudaMemcpyDeviceToHost, s));
    PDSB_CUDA_OK(cudaMemcpyAsync(hM.data(), dM, hM.size() * sizeof(double), cudaMemcpyDeviceToHost, s));
    PDSB_CUDA_OK(cudaStreamSynchronize(s));
    // faer's QR propagates a NaN in X'WX or X'Wz into the solution; K3 zeroes a zero pivot instead, so a non-finite
    // moment is mapped to NaN coefficients here (q + 1 rows / columns used: features, z, and the ones when biased)
    bool finite = true;
    for (int j = 0; j <= q; ++j)
      for (int k = 0; k <= q; ++k) finite &= std::isfinite(hM[(size_t)mi(j) * q1 + mi(k)]);
    if (!finite) {
      for (int j = 0; j < q; ++j) hb_new[j] = NAN;
      PDSB_CUDA_OK(cudaMemcpyAsync(dbeta, hb_new.data(), (size_t)q * sizeof(double), cudaMemcpyHostToDevice, s));
    }
    double max_diff = 0.0;                                      // f64::max ignores a NaN operand, as fmax does
    for (int j = 0; j < q; ++j) max_diff = std::fmax(max_diff, std::fabs(hb[j] - hb_new[j]));
    hb = hb_new;
    if (max_diff < tol) break;
  }
  PDSB_CUDA_OK(cudaStreamSynchronize(s));
  std::memcpy(coeffs, hb.data(), (size_t)q * sizeof(double));
  if (n_iter) *n_iter = it;
  return 0;
}

// GLM.fit_by: pdsb_glm_fit on every group at once.  [X | y] is uploaded once, in the caller's (group) order, then K16
// runs every group's IRLS with the family's row rule; one copy back of the coefficients, statuses and iteration counts.
int pdsb_glm_fit_by(const pdsb_matrix* X, const pdsb_matrix* y, const int64_t* offsets, int64_t n_groups, int add_bias,
                    int family, int64_t max_iter, double tol, double* coeffs, int64_t* n_iter, int* status) {
  if (require_device()) return 1;
  if (check_matrix(X) || check_matrix(y)) return 1;
  if (!coeffs || !offsets) { set_error("pdsb_glm_fit_by: null argument"); return 1; }
  if (family < PDSB_GLM_GAUSSIAN || family > PDSB_GLM_GAMMA) { set_error("GLM.fit_by: unknown family %d", family); return 1; }
  const int64_t n = X->n_rows;
  if (n != y->n_rows || y->n_cols != 1) { set_error("Dimension mismatch."); return 1; }
  if (X->n_cols < 1 || X->n_cols > 64) {
    set_error("GLM.fit_by: %lld features not supported (1..64)", (long long)X->n_cols);
    return 1;
  }
  if (max_iter < 1) { set_error("GLM.fit_by: max_iter=%lld must be >= 1", (long long)max_iter); return 1; }
  if (check_group_offsets(offsets, n_groups, n, "GLM.fit_by")) return 1;
  const int p = (int)X->n_cols, q = p + (add_bias ? 1 : 0);
  std::vector<int> hs((size_t)n_groups, PDSB_GLM_EMPTY);
  std::vector<int64_t> hit((size_t)n_groups, 0);
  if (n == 0) {                                 // every group is empty
    for (int64_t k = 0; k < n_groups * q; ++k) coeffs[k] = NAN;
  } else {
    cudaStream_t s;
    if (thread_stream(&s)) return 1;
    DevBag bag(s);
    double* dZ = upload_xy(*X, *y, true, bag, s);
    double* dbeta = bag.alloc<double>((size_t)n_groups * q);
    int* dst = bag.alloc<int>((size_t)n_groups);
    int64_t* dit = bag.alloc<int64_t>((size_t)n_groups);
    int64_t* doff = nullptr;
    if (!dZ || !dbeta || !dst || !dit || upload_offsets(offsets, n_groups, doff, bag, s)) return 1;
    const int64_t ld = pad_ld(n);
    if (grouped_glm(dZ, ld, dZ + (size_t)ld * p, nullptr, doff, n_groups, n, p, add_bias ? 1 : 0, family, tol, max_iter,
                    dbeta, dst, dit, s)) return 1;
    PDSB_CUDA_OK(cudaMemcpyAsync(coeffs, dbeta, (size_t)n_groups * q * sizeof(double), cudaMemcpyDeviceToHost, s));
    PDSB_CUDA_OK(cudaMemcpyAsync(hit.data(), dit, (size_t)n_groups * sizeof(int64_t), cudaMemcpyDeviceToHost, s));
    if (download_status(dst, (size_t)n_groups, hs, s)) return 1;
  }
  if (status) std::memcpy(status, hs.data(), hs.size() * sizeof(int));
  if (n_iter) std::memcpy(n_iter, hit.data(), hit.size() * sizeof(int64_t));
  return 0;
}

int pdsb_glm_predict(const pdsb_matrix* X, const double* coeffs, int n_coef, int has_bias, int family, int linear,
                     double* out) {
  if (require_device()) return 1;
  if (check_matrix(X)) return 1;
  if (n_coef < 1 || !coeffs) { set_error("Matrix is not learned yet."); return 1; }      // lr/mod.rs:149-150
  if (family < PDSB_GLM_GAUSSIAN || family > PDSB_GLM_GAMMA) { set_error("pdsb_glm_predict: unknown family %d", family); return 1; }
  const int p = n_coef - (has_bias ? 1 : 0);
  if (X->n_cols != p) { set_error("Dimension mismatch."); return 1; }                  // :147-148
  return predict_rows(*X, coeffs, n_coef, has_bias, linear ? PDSB_GLM_GAUSSIAN : family, out);
}

// MixedModel.fit -> fit_reml (mixed/mod.rs:173-272): group codes -> row order (radix sort), [X | y] uploaded in group
// order through the permuted gather, then the K5 group pass, the size buckets and the REML search of K12 on the device.
// One D2H at the end carries the results and the status of the search.
int pdsb_mixed_fit(const pdsb_matrix* X, const pdsb_matrix* y, const int64_t* group_codes, int64_t n_groups,
                   const int64_t* between_idx, int n_between, int64_t max_iter, double tol, double* coeffs,
                   double* std_errors, double* dfs, double* gamma, double* resid_variance, int64_t* n_evals) {
  if (require_device()) return 1;
  if (check_matrix(X) || check_matrix(y)) return 1;
  if (!coeffs || !std_errors || !dfs || !gamma || !resid_variance) { set_error("pdsb_mixed_fit: null output"); return 1; }
  const int64_t n = X->n_rows;
  if (n != y->n_rows || y->n_cols != 1) { set_error("X, y, and group must have the same number of rows."); return 1; }
  if (n <= X->n_cols) { set_error("Not enough rows to fit a mixed model with this many fixed effects."); return 1; }
  if (X->n_cols < 1 || X->n_cols > 64) {
    set_error("MixedModel supports 1 to 64 fixed effects (intercept included), got %lld.", (long long)X->n_cols);
    return 1;
  }
  const int p = (int)X->n_cols;
  if (!group_codes || n_groups < 1) { set_error("Group codes must lie in [0, n_groups)."); return 1; }
  int64_t lo = group_codes[0], hi = group_codes[0];
  for (int64_t i = 1; i < n; ++i) { lo = std::min(lo, group_codes[i]); hi = std::max(hi, group_codes[i]); }
  if (lo < 0 || hi >= n_groups) { set_error("Group codes must lie in [0, n_groups)."); return 1; }
  std::vector<uint8_t> between(p, 0);
  if (n_between < 0 || (n_between > 0 && !between_idx)) { set_error("pdsb_mixed_fit: bad between_idx"); return 1; }
  for (int i = 0; i < n_between; ++i) {
    if (between_idx[i] < 0 || between_idx[i] >= p) { set_error("between_idx must lie in [0, %d).", p); return 1; }
    between[between_idx[i]] = 1;
  }
  cudaStream_t s;
  if (thread_stream(&s)) return 1;
  DevBag bag(s);
  const int64_t ld = pad_ld(n);
  int64_t* dcodes = bag.alloc<int64_t>((size_t)n);
  int64_t* rows = bag.alloc<int64_t>((size_t)n);
  int64_t* offsets = bag.alloc<int64_t>((size_t)n_groups + 1);
  double* dZ = bag.alloc<double>((size_t)ld * (p + 1));
  uint8_t* dbetween = bag.alloc<uint8_t>((size_t)p);
  double* dout = bag.alloc<double>((size_t)3 * p + 4);
  if (!dcodes || !rows || !offsets || !dZ || !dbetween || !dout) return 1;
  PDSB_CUDA_OK(cudaMemcpyAsync(dcodes, group_codes, (size_t)n * sizeof(int64_t), cudaMemcpyHostToDevice, s));
  PDSB_CUDA_OK(cudaMemcpyAsync(dbetween, between.data(), (size_t)p, cudaMemcpyHostToDevice, s));
  if (mixed_order_rows(dcodes, n, n_groups, rows, offsets, s)) return 1;
  const double* v; int64_t rs, cs;
  if (upload(*X, nullptr, 0, bag, s, &v, &rs, &cs) || gather_colmajor(v, rs, cs, n, p, rows, dZ, ld, s)) return 1;
  if (upload(*y, nullptr, 0, bag, s, &v, &rs, &cs) || gather_colmajor(v, rs, cs, n, 1, rows, dZ + (size_t)ld * p, ld, s))
    return 1;
  if (mixed_reml(dZ, ld, offsets, n_groups, n, p, dbetween, max_iter < 0 ? 0 : max_iter, tol, dout, s)) return 1;
  std::vector<double> h((size_t)3 * p + 4);
  PDSB_CUDA_OK(cudaMemcpyAsync(h.data(), dout, h.size() * sizeof(double), cudaMemcpyDeviceToHost, s));
  PDSB_CUDA_OK(cudaStreamSynchronize(s));
  const int st = (int)h[3 * p + 3];
  if (st == PDSB_MIXED_NOT_PD) { set_error("X'HiX is not positive definite; design may be rank-deficient."); return 1; }
  if (st == PDSB_MIXED_RESID_VAR) { set_error("Residual variance estimate is non-positive."); return 1; }
  std::memcpy(coeffs, h.data(), (size_t)p * sizeof(double));
  std::memcpy(std_errors, h.data() + p, (size_t)p * sizeof(double));
  std::memcpy(dfs, h.data() + 2 * p, (size_t)p * sizeof(double));
  *gamma = h[3 * p];
  *resid_variance = h[3 * p + 1];
  if (n_evals) *n_evals = (int64_t)h[3 * p + 2];
  return 0;
}

pdsb_online_lr* pdsb_online_lr_new(int n_coef, int has_bias) {
  if (require_device()) return nullptr;
  if (n_coef < 1 || n_coef > 512) { set_error("online lin_reg state: %d coefficients not supported (1..512)", n_coef); return nullptr; }
  pdsb_online_lr* h = new pdsb_online_lr{n_coef, has_bias ? 1 : 0, 0, nullptr, nullptr, nullptr, false};
  cudaGetDevice(&h->device);
  double* blk = nullptr;
  if (cudaMalloc(&blk, ((size_t)n_coef * n_coef + 2 * (size_t)n_coef) * sizeof(double)) != cudaSuccess) {
    set_error("online lin_reg state: cudaMalloc failed");
    delete h;
    return nullptr;
  }
  h->inv = blk; h->w = blk + (size_t)n_coef * n_coef; h->x = h->w + n_coef;
  if (cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking) != cudaSuccess) {
    set_error("pdsb_online_lr_new: stream creation failed");
    cudaFree(blk);
    delete h;
    return nullptr;
  }
  return h;
}

void pdsb_online_lr_free(pdsb_online_lr* h) {
  if (!h) return;
  if (h->stream) { cudaStreamSynchronize(h->stream); cudaStreamDestroy(h->stream); }
  cudaFree(h->inv);
  delete h;
}

/* coeffs: n_coef values (bias last), inv: n_coef^2 row-major  (OnlineLR::set_coeffs_bias_inverse, :29-52) */
int pdsb_online_lr_set(pdsb_online_lr* h, const double* coeffs, const double* inv) {
  if (!h || !coeffs || !inv) { set_error("pdsb_online_lr_set: null argument"); return 1; }
  std::lock_guard<std::mutex> lk(h->mu);
  cudaStream_t s = h->stream;
  PDSB_CUDA_OK(cudaMemcpyAsync(h->w, coeffs, (size_t)h->q * sizeof(double), cudaMemcpyHostToDevice, s));
  PDSB_CUDA_OK(cudaMemcpyAsync(h->inv, inv, (size_t)h->q * h->q * sizeof(double), cudaMemcpyHostToDevice, s));
  PDSB_CUDA_OK(cudaStreamSynchronize(s));
  h->fit = true;
  return 0;
}

/* x_row: the n_coef - has_bias feature values of ONE row; non-finite rows are ignored (OnlineLR::update :85-89) */
int pdsb_online_lr_update(pdsb_online_lr* h, const double* x_row, double y, double c) {
  if (!h || !x_row) { set_error("pdsb_online_lr_update: null argument"); return 1; }
  if (!h->fit) { set_error("Matrix is not learned yet."); return 1; }
  std::lock_guard<std::mutex> lk(h->mu);
  cudaStream_t s = h->stream;
  const int pf = h->q - h->has_bias;
  if (pf > 0) PDSB_CUDA_OK(cudaMemcpyAsync(h->x, x_row, (size_t)pf * sizeof(double), cudaMemcpyHostToDevice, s));
  if (woodbury_update(h->inv, h->w, h->q, h->has_bias, h->x, y, c, s)) return 1;
  return 0;   // stream-ordered on the handle's stream: the next update / get (from any thread) sees the new state
}

int pdsb_online_lr_get(pdsb_online_lr* h, double* coeffs, double* inv) {
  if (!h) { set_error("pdsb_online_lr_get: null handle"); return 1; }
  if (!h->fit) { set_error("Matrix is not learned yet."); return 1; }
  std::lock_guard<std::mutex> lk(h->mu);
  cudaStream_t s = h->stream;
  if (coeffs) PDSB_CUDA_OK(cudaMemcpyAsync(coeffs, h->w, (size_t)h->q * sizeof(double), cudaMemcpyDeviceToHost, s));
  if (inv) PDSB_CUDA_OK(cudaMemcpyAsync(inv, h->inv, (size_t)h->q * h->q * sizeof(double), cudaMemcpyDeviceToHost, s));
  PDSB_CUDA_OK(cudaStreamSynchronize(s));
  return 0;
}

}  // extern "C"
