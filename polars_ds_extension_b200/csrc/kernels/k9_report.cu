// K9 — lin_reg_report / wls_report statistics, all on the device.
//
// Reference: pl_lin_reg_report / pl_wls_report (/root/reference/src/num_ext/linear_regression.rs:822-1117).
// The reference materialises the p x N matrix (X'X)^-1 X' (:857) and N x N diagonal products for HC0-HC3
// (:880-909).  Here:   moments (K2) -> explicit inverse + beta (K3, method INV) -> residual pass (K4, SSR) ->
// [HC only] per-row weight  omega_i = e_i^2 * {1, 1/(1-h_i), 1/(1-h_i)^2},  h_i = x_i G^-1 x_i^T  (this file) ->
// "meat" X' diag(omega) X as a weighted moments pass (K2a) -> p-length epilogue: G^-1 meat G^-1, SE, t,
// p = 2 sf(|t|, dof), CI = beta -/+ t_{0.975,dof} SE, r2 = 1 - SSR/(var_y * n) (the reference multiplies the
// ddof=1 variance by n, :867 — kept), adj_r2.  The per-row weight and the epilogue's per-coefficient rule live in
// report_rows.h, shared with the grouped report (K17).
#include "../common.h"
#include "kernels.h"
#include "report_rows.h"

namespace pdsb {

namespace {

// STAGED: G^-1 is copied to shared memory as T (q^2 elements) when that fits the block's opt-in limit, which holds
// q <= 170 in f64 and q <= 241 in f32; wider fits read it from global memory, where at most 259^2 doubles (537 KB) stay
// cache-resident.  Both read the same (T) G^-1 values, so the weights do not depend on where they were read.
template <typename T, bool STAGED>
__global__ void __launch_bounds__(256)
hc_weights_kernel(const T* __restrict__ X, int64_t ldx, const T* __restrict__ resid, const T* __restrict__ mask,
                  int64_t n, int p, int add_bias, int se_type, const double* __restrict__ ginv /* q x q */,
                  T* __restrict__ omega) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  T* gi = reinterpret_cast<T*>(smem_raw);
  const int q = p + (add_bias ? 1 : 0);
  if (STAGED) {
    for (int i = threadIdx.x; i < q * q; i += blockDim.x) gi[i] = (T)ginv[i];
    __syncthreads();
  }
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x) {
    T wgt = hc_weight<T>(resid[r], q, se_type, [&](int a) { return (a < p) ? X[(int64_t)a * ldx + r] : T(1); },
                         [&](int a, int b) { return STAGED ? gi[a * q + b] : (T)ginv[a * q + b]; });
    if (mask && mask[r] == T(0)) wgt = T(0);
    omega[r] = wgt;
  }
}

struct FinalizeArgs {
  const double* nvalid;  // number of rows that entered the fit
  const double* beta;    // q
  const double* ginv;    // q x q
  const double* ssr;     // [0] unweighted, [4] weighted (layout of predict's ssr buffer: 8 doubles)
  const double* meat;    // moments with omega weights (q1 x q1) or null
  int p, add_bias, se_type, weighted;
  double y_var;
  double* out;           // 8 x q
};

__global__ void report_finalize_kernel(FinalizeArgs a) {
  const int p = a.p, q = p + (a.add_bias ? 1 : 0), q1 = p + 2;
  const int i = threadIdx.x;
  __shared__ double t_alpha;
  const double n = *a.nvalid;
  if (i == 0) t_alpha = student_t_ppf(0.975, n - (double)q);
  __syncthreads();
  if (i >= q) return;
  auto fz = [&](int c) { return c < p ? c : p + 1; };
  report_column(i, q, a.weighted ? 0 : a.se_type, n, a.ssr[0], a.weighted ? a.ssr[4] : a.ssr[0], a.y_var, t_alpha,
                a.beta, a.ginv, [&](int r, int c) { return a.meat[(size_t)fz(r) * q1 + fz(c)]; }, a.out);
}

}  // namespace

template <typename T>
int report_stats(const T* X, int64_t ldx, const T* y, const T* w, const T* mask, int64_t n, int p, int add_bias,
                 int se_type, double y_var, double* out, cudaStream_t s) {
  const int q = p + (add_bias ? 1 : 0), q1 = p + 2;
  char* base = nullptr;
  // M (q1^2) | meat (q1^2) | beta (q) | ginv (q^2) | ssr (8) | status
  size_t nd = 2 * (size_t)q1 * q1 + q + (size_t)q * q + 8 + 4;
  if (dev_alloc((void**)&base, nd * sizeof(double), s)) return 1;
  double* M = reinterpret_cast<double*>(base);
  double* meat = M + (size_t)q1 * q1;
  double* beta = meat + (size_t)q1 * q1;
  double* ginv = beta + q;
  double* ssr = ginv + (size_t)q * q;
  double* nvalid = ssr + 8;
  int* status = reinterpret_cast<int*>(ssr + 10);
  T* pred = nullptr; T* resid = nullptr; T* omega = nullptr;
  const int64_t ldo = (n + 3) & ~int64_t(3);
  int rc = 0;
  auto cleanup = [&]() {
    if (pred) dev_free(pred, s);
    if (resid) dev_free(resid, s);
    if (omega) dev_free(omega, s);
    dev_free(base, s);
  };
  if (dev_alloc((void**)&pred, (size_t)ldo * sizeof(T), s) || dev_alloc((void**)&resid, (size_t)ldo * sizeof(T), s)) { cleanup(); return 1; }
  rc = mask ? count_mask<T>(mask, n, nvalid, s) : fill_value<double>(nvalid, 1, (double)n, s);
  if (!rc) rc = moments<T>(MomentsPrecision::F64_ACCUM, X, ldx, y, n, w, mask, n, p, 1, M, s);
  pdsb_solve_opts o{};
  o.p = p; o.t = 1; o.add_bias = add_bias; o.method = PDSB_METHOD_INV; o.solver = PDSB_SOLVER_QR;
  if (!rc) rc = solve_from_moments(M, o, beta, status, ginv, s);
  if (!rc) rc = predict_resid<T>(X, ldx, y, n, w, mask, n, p, 1, add_bias, beta, status, pred, resid, ldo, nullptr, ssr, s);
  const bool hc = (se_type >= 1) && !w;
  if (!rc && hc) {
    if (dev_alloc((void**)&omega, (size_t)ldo * sizeof(T), s)) { cleanup(); return 1; }
    // hc0 / hc1 do not read G^-1; hc2 / hc3 stage it in shared memory when it fits
    int dev = 0, optin = 48 * 1024;
    cudaError_t e = cudaGetDevice(&dev);
    if (e == cudaSuccess) e = cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
    const size_t staged = (size_t)q * q * sizeof(T);
    const bool stage = se_type >= 3 && staged <= (size_t)optin;
    const size_t smem = stage ? staged : 0;
    auto k = stage ? hc_weights_kernel<T, true> : hc_weights_kernel<T, false>;
    if (e == cudaSuccess && smem > 48 * 1024) e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e == cudaSuccess) {
      int grid = (int)std::min<int64_t>(ceil_div(n, 256), (int64_t)sm_count() * 8);
      k<<<grid, 256, smem, s>>>(X, ldx, resid, mask, n, p, add_bias, se_type, ginv, omega);
      e = cudaGetLastError(); count_launch();
    }
    if (e != cudaSuccess) { set_error("hc_weights launch failed: %s", cudaGetErrorString(e)); rc = 1; }
    if (!rc) rc = moments<T>(MomentsPrecision::F64_ACCUM, X, ldx, y, n, omega, mask, n, p, 1, meat, s);
  }
  if (!rc) {
    FinalizeArgs a;
    a.nvalid = nvalid; a.beta = beta; a.ginv = ginv; a.ssr = ssr; a.meat = hc ? meat : nullptr;
    a.p = p; a.add_bias = add_bias; a.se_type = hc ? se_type : 0; a.weighted = w ? 1 : 0; a.y_var = y_var; a.out = out;
    int threads = ((q + 31) / 32) * 32;
    report_finalize_kernel<<<1, threads, 0, s>>>(a);
    cudaError_t e = cudaGetLastError(); count_launch();
    if (e != cudaSuccess) { set_error("report finalize launch failed: %s", cudaGetErrorString(e)); rc = 1; }
  }
  cleanup();
  return rc;
}

template int report_stats<float>(const float*, int64_t, const float*, const float*, const float*, int64_t, int, int,
                                 int, double, double*, cudaStream_t);
template int report_stats<double>(const double*, int64_t, const double*, const double*, const double*, int64_t, int,
                                  int, int, double, double*, cudaStream_t);

}  // namespace pdsb
