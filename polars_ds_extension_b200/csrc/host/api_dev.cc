// Device layer of the C ABI (pdsb_dev_*): thin, typed wrappers over the kernel launchers.
#include "../common.h"
#include "../kernels/kernels.h"
#include "../kernels/special.h"
#include "host.h"

using namespace pdsb;

static thread_local int t_last_moments_path = 0;
static std::atomic<int> g_forced_path{0};

extern "C" {

const char* pdsb_last_error(void) { return get_error(); }
int pdsb_version(void) { return PDSB_VERSION; }
int64_t pdsb_kernel_launch_count(void) { return g_kernel_launches.load(); }
int pdsb_last_moments_path(void) { return t_last_moments_path; }
void pdsb_set_moments_path(int path) { g_forced_path.store(path); }
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
  cudaStream_t s = (cudaStream_t)stream;
  const int forced = g_forced_path.load();
  t_last_moments_path = 0;
  // few features, one target, no mask / weights: the register-moments kernel is HBM-bound where the tensor-core kernel
  // is bound by its per-stage cost (path 3 in pdsb_last_moments_path)
  if (!w && !mask && forced == 0 && t == 1 && p <= 10 && n >= 65536) {
    int rc = moments_small<float>(X, ldx, Y, n, p, M, s);
    if (rc == 0) { t_last_moments_path = 3; return 0; }
    if (rc > 0) return rc;
  }
  if (!w && forced != 1 && moments_wgmma_supported(X, ldx, Y, ldy, n, p, t)) {
    int rc = moments_wgmma_f32(X, ldx, Y, ldy, mask, n, p, t, M, s);
    if (rc == 0) { t_last_moments_path = 1; return 0; }
    if (rc > 0) return rc;
  }
  if (forced == 2) { set_error("moments: tensor-core path forced but shape/alignment unsupported"); return 1; }
  return moments_simt<float>(X, ldx, Y, ldy, w, mask, n, p, t, M, s);
}

int pdsb_dev_moments_f64(const double* X, int64_t ldx, const double* Y, int64_t ldy, const double* w,
                         const double* mask, int64_t n, int p, int t, double* M, void* stream) {
  if (require_device()) return 1;
  return moments_simt<double>(X, ldx, Y, ldy, w, mask, n, p, t, M, (cudaStream_t)stream);
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
  cudaStream_t s = (cudaStream_t)stream;
  if (xcol < 0 || ycol < 0 || xcol + p > ncols || ycol + t > ncols) { set_error("moments_frame: columns out of range"); return 1; }
  t_last_moments_path = 0;
  if (g_forced_path.load() != 1) {
    int rc = moments_wgmma_frame_f32(frame, n, ncols, xcol, p, ycol, t, mask, M, s);
    if (rc == 0) { t_last_moments_path = 1; return 0; }
    if (rc > 0) return rc;
  }
  if (g_forced_path.load() == 2) { set_error("moments_frame: tensor-core path forced but shape unsupported"); return 1; }
  const int64_t bstride = (int64_t)ncols * FRAME_ROWS;
  return moments_simt<float>(frame + (size_t)xcol * FRAME_ROWS, 0, frame + (size_t)ycol * FRAME_ROWS, 0, nullptr, mask, n, p, t,
                             M, s, bstride);
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
