// Grouped host entries of the C ABI (pdsb_host_grouped_*, pdsb_host_pca_by, pdsb_host_grouped_isotonic): per group, the
// single call of lr_host.cc on that group's rows, for every group in one launch sequence.  The frame is uploaded once in
// group order (rows [offsets[g], offsets[g+1]) are group g), the checked offsets go to the device, and the grouped
// kernels (K5, K6 over groups, K15-K19) write per-group results that come back in one copy each.
#include "../common.h"
#include "../kernels/kernels.h"
#include "host.h"
#include <cstring>
#include <cmath>

namespace pdsb {

// The offsets are user data (an Int64 column): every group must be a row range inside the frame of n rows, or the
// kernels would read outside X / y.  Every grouped host entry shares these checks; `what` names the expression in the
// message.
int check_group_offsets(const int64_t* offsets, int64_t n_groups, int64_t n, const char* what) {
  if (n_groups < 1 || offsets[0] != 0 || offsets[n_groups] != n) { set_error("%s: bad group offsets", what); return 1; }
  for (int64_t g = 0; g < n_groups; ++g)
    if (offsets[g] < 0 || offsets[g] > offsets[g + 1] || offsets[g + 1] > n) {
      set_error("%s: group offsets must be non-decreasing and within [0, n] (group %lld)", what, (long long)g);
      return 1;
    }
  return 0;
}

int upload_offsets(const int64_t* offsets, int64_t n_groups, int64_t*& doff, DevBag& bag, cudaStream_t s) {
  if (!(doff = bag.alloc<int64_t>((size_t)n_groups + 1))) return 1;
  PDSB_CUDA_OK(cudaMemcpyAsync(doff, offsets, (size_t)(n_groups + 1) * sizeof(int64_t), cudaMemcpyHostToDevice, s));
  return 0;
}

int download_status(const int* dst, size_t count, std::vector<int>& h, cudaStream_t s) {
  h.resize(count);
  PDSB_CUDA_OK(cudaMemcpyAsync(h.data(), dst, count * sizeof(int), cudaMemcpyDeviceToHost, s));
  PDSB_CUDA_OK(cudaStreamSynchronize(s));
  return 0;
}

namespace {

// the validity bytes of a per-group result: a group is valid when its status is PDSB_OK
uint8_t* valid_from_status(pdsb_host_result* out, const std::vector<int>& hs) {
  uint8_t* v = reinterpret_cast<uint8_t*>(result_buf(out, hs.size()));
  if (v) for (size_t g = 0; g < hs.size(); ++g) v[g] = hs[g] == PDSB_OK;
  return v;
}

// The frame of a grouped call: build_frame's upload of [targets | features] in group order (no weights), then the offset
// checks (`what` names the expression in their message) and the offsets on the device (doff, n_groups + 1).
template <typename T>
int grouped_frame(const pdsb_column* cols, int n_cols, int n_targets, const NullPolicy& pol, bool multi, bool online,
                  const int64_t* offsets, int64_t n_groups, const char* what, Frame<T>& F, int64_t*& doff, DevBag& bag,
                  cudaStream_t s) {
  if (build_frame<T>(cols, n_cols, n_targets, nullptr, pol, multi, online, F, bag, s)) return 1;
  if (check_group_offsets(offsets, n_groups, F.n, what)) return 1;
  return upload_offsets(offsets, n_groups, doff, bag, s);
}

// grouped_frame for pl_lr_by, pl_lr_pred_by, pl_lin_reg_report_by and pl_lr_w_rcond_by: nulls only with "skip" (a null
// row becomes NaN and drops out of its group), and no weights.
template <typename T>
int lr_by_frame(const pdsb_column* cols, int n_cols, const int64_t* offsets, int64_t n_groups, const pdsb_lr_kwargs* kw,
                const NullPolicy& pol, Frame<T>& F, int64_t*& doff, DevBag& bag, cudaStream_t s) {
  for (int c = 0; c < n_cols; ++c)
    if (col_nulls(cols[c]) > 0 && pol.kind != NullKind::SKIP) {
      if (pol.kind == NullKind::RAISE) set_error("Nulls found in data");
      else set_error("grouped lin_reg: only null_policy='skip' is supported with nulls");
      return 1;
    }
  NullPolicy nanpol{NullKind::IGNORE, 0.0};
  if (grouped_frame<T>(cols, n_cols, 1, nanpol, false, true, offsets, n_groups, "grouped lin_reg", F, doff, bag, s)) return 1;
  if (kw->weighted) { set_error("grouped lin_reg: weighted fits are not batched"); return 1; }
  return 0;
}

// The batched fit shared by pl_lr_by and pl_lr_pred_by: checks, upload of [y | X] in group order, offsets, K5.
// want_pred picks the solver settings of pl_lr_pred over pl_lr's (lr_solve_opts: only the f32 NNLS sweep count differs).
// On return F holds the frame, and doff / dbeta / dst (n_groups + 1, n_groups x q, n_groups) the device offsets,
// coefficients and statuses.
template <typename T>
struct GroupedFit {
  Frame<T> F;
  int q = 0, add_bias = 0;
  int64_t* doff = nullptr; double* dbeta = nullptr; int* dst = nullptr;
  GroupWork wl;     // with want_pred: the fit's work list, for the predict pass
};

template <typename T>
int grouped_fit(const pdsb_column* cols, int n_cols, const int64_t* offsets, int64_t n_groups, const pdsb_lr_kwargs* kw,
                const NullPolicy& pol, int want_pred, GroupedFit<T>& G, DevBag& bag, cudaStream_t s) {
  Frame<T>& F = G.F;
  if (lr_by_frame<T>(cols, n_cols, offsets, n_groups, kw, pol, F, G.doff, bag, s)) return 1;
  const pdsb_solve_opts o = lr_solve_opts(kw, F.p, 1, sizeof(T) == 4, want_pred);     // pl_lr(_pred) per group, batched
  G.q = F.p + o.add_bias; G.add_bias = o.add_bias;
  G.dbeta = bag.alloc<double>((size_t)n_groups * G.q);
  G.dst = bag.alloc<int>((size_t)n_groups);
  if (!G.dbeta || !G.dst) return 1;
  return grouped_lin_reg<T>(F.X(), F.ld, F.Y(), G.doff, n_groups, F.n, F.p, o, G.dbeta, G.dst, s, &bag,
                            want_pred ? &G.wl : nullptr);
}

// The per-group result from the device beta [n_groups x t x q] and status: coefficients rounded to T, valid = status 0.
// With dsv, the singular values [n_groups][q] as well, rounded to T.
template <typename T>
int grouped_coeffs_result(const double* dbeta, const int* dst, int64_t n_groups, int q, pdsb_host_result* out,
                          cudaStream_t s, int t = 1, const double* dsv = nullptr) {
  std::vector<double> hb((size_t)n_groups * t * q), hsv(dsv ? hb.size() : 0);
  std::vector<int> hs;
  PDSB_CUDA_OK(cudaMemcpyAsync(hb.data(), dbeta, hb.size() * sizeof(double), cudaMemcpyDeviceToHost, s));
  if (dsv) PDSB_CUDA_OK(cudaMemcpyAsync(hsv.data(), dsv, hsv.size() * sizeof(double), cudaMemcpyDeviceToHost, s));
  if (download_status(dst, (size_t)n_groups, hs, s)) return 1;
  out->is_f32 = sizeof(T) == 4; out->n_coef = q; out->n_targets = t; out->n_rows = n_groups;
  T* c = reinterpret_cast<T*>(result_buf(out, hb.size() * sizeof(T)));
  T* sv = dsv ? reinterpret_cast<T*>(result_buf(out, hsv.size() * sizeof(T))) : nullptr;
  if (!c || (dsv && !sv) || !(out->valid = valid_from_status(out, hs))) return 1;
  for (size_t i = 0; i < hb.size(); ++i) c[i] = (T)hb[i];
  for (size_t i = 0; i < hsv.size(); ++i) sv[i] = (T)hsv[i];
  out->coeffs = c; out->singular_values = sv;
  return 0;
}

template <typename T>
int host_grouped_t(const pdsb_column* cols, int n_cols, const int64_t* offsets, int64_t n_groups,
                   const pdsb_lr_kwargs* kw, pdsb_host_result* out) {
  cudaStream_t s;
  if (thread_stream(&s)) return 1;
  NullPolicy pol;
  if (parse_null_policy(kw->null_policy, &pol)) return 1;
  DevBag bag(s);
  GroupedFit<T> G;
  if (grouped_fit<T>(cols, n_cols, offsets, n_groups, kw, pol, 0, G, bag, s)) return 1;
  return grouped_coeffs_result<T>(G.dbeta, G.dst, n_groups, G.q, out, s);
}

// pl_ar_coeffs_by: per group, pl_lr_by on the group's lagged columns (x.slice(lag) against x.shift(i).slice(lag)), from
// one upload of x in key order (K5's AR pass, kernels/k5_grouped.cu).  Null policy, as pl_lr does it per column:
// "raise" fails on any null; "skip" uploads nulls as NaN, so every row a null reaches as target or lag drops out; a fill
// uploads x filled for its use as a lag, and the row mask from x's validity drops the rows whose target is null.
template <typename T>
int host_grouped_ar_t(const pdsb_column& x, const int64_t* offsets, int64_t n_groups, int lag, const pdsb_lr_kwargs* kw,
                      pdsb_host_result* out) {
  NvtxRange nv("pdsb:host_grouped_ar");
  cudaStream_t s;
  if (thread_stream(&s)) return 1;
  NullPolicy pol;
  if (parse_null_policy(kw->null_policy, &pol)) return 1;
  const int64_t n = col_len(x);
  if (check_group_offsets(offsets, n_groups, n, "grouped query_ar_coeffs")) return 1;
  if (lag < 1 || lag > 64) {
    set_error("grouped query_ar_coeffs: lag=%d; the batched fit takes 1 to 64 lags (use the per-group loop)", lag);
    return 1;
  }
  if (kw->weighted) { set_error("grouped query_ar_coeffs: weighted fits are not batched"); return 1; }
  const bool nulls = col_nulls(x) > 0;
  int mode = 0;                      // upload_column: 0 null -> NaN, 1 null -> fill
  if (nulls) {
    switch (pol.kind) {
      case NullKind::RAISE: set_error("Nulls found in data"); return 1;
      case NullKind::SKIP: break;
      case NullKind::FILL: mode = 1; break;
      default: set_error("grouped query_ar_coeffs: null_policy '%s' is not batched", kw->null_policy); return 1;
    }
  }
  DevBag bag(s);
  const int64_t ld = pad_ld(n);
  T* dx = bag.alloc<T>((size_t)ld);
  if (!dx) return 1;
  UploadPlan plan;
  if (upload_column<T>(x, dx, mode, pol.fill_as<T>(), bag, plan, s)) return 1;
  T* mask = nullptr;
  if (mode == 1 && !(mask = row_mask<T>(&x, 1, n, ld, bag, plan, s))) return 1;
  if (plan.run(s)) return 1;
  const int q = lag + (kw->bias ? 1 : 0);
  double* dbeta = bag.alloc<double>((size_t)n_groups * q);
  int* dst = bag.alloc<int>((size_t)n_groups);
  int64_t* doff = nullptr;
  if (!dbeta || !dst || upload_offsets(offsets, n_groups, doff, bag, s)) return 1;
  const pdsb_solve_opts o = lr_solve_opts(kw, lag, 1, sizeof(T) == 4, 0);     // pl_lr per group, batched
  if (grouped_ar_lin_reg<T>(dx, mask, doff, n_groups, n, lag, o, dbeta, dst, s)) return 1;
  return grouped_coeffs_result<T>(dbeta, dst, n_groups, q, out, s);
}

// pl_lr_multi_by: per group, pl_lr_by's fit of every target on the features (K5 with t right-hand sides,
// grouped_lin_reg_multi).  The frame is pl_lr_multi's, built once in key order: build_frame's multi-target null rules give
// the per-group loop's messages, and every one of them is decided row by row, so the batched call fails exactly when the
// loop does.  The offsets are checked as pl_lr_by checks them; the solve options are pl_lr_multi's (LSTSQ, no l1).
template <typename T>
int host_grouped_multi_t(const pdsb_column* cols, int n_cols, const int64_t* offsets, int64_t n_groups,
                         const pdsb_lr_kwargs* kw, int t, pdsb_host_result* out) {
  NvtxRange nv("pdsb:host_grouped_multi");
  cudaStream_t s;
  if (thread_stream(&s)) return 1;
  NullPolicy pol;
  if (parse_null_policy(kw->null_policy, &pol)) return 1;
  DevBag bag(s);
  Frame<T> F;
  int64_t* doff = nullptr;
  if (grouped_frame<T>(cols, n_cols, t, pol, true, false, offsets, n_groups, "grouped lin_reg", F, doff, bag, s)) return 1;
  pdsb_solve_opts o = lr_solve_opts(kw, F.p, t, sizeof(T) == 4, 0);
  o.method = PDSB_METHOD_LSTSQ; o.l1_reg = 0.0;
  const int q = F.p + o.add_bias;
  double* dbeta = bag.alloc<double>((size_t)n_groups * t * q);
  int* dst = bag.alloc<int>((size_t)n_groups);
  if (!dbeta || !dst) return 1;
  if (grouped_lin_reg_multi<T>(F.Z, F.ld, t, F.p, doff, n_groups, F.n, o, dbeta, dst, s)) return 1;
  return grouped_coeffs_result<T>(dbeta, dst, n_groups, q, out, s, t);
}

// The predict pass of a grouped fit G (K5 pass 3 on the fit's work list) and its per-row result: pred / resid in one
// copy each; the validity bytes only when some row is masked or some group's fit is not OK.
template <typename T>
int grouped_pred_result(const GroupedFit<T>& G, int64_t n_groups, const T* mask, pdsb_host_result* out, DevBag& bag,
                        cudaStream_t s) {
  const Frame<T>& F = G.F;
  const int64_t n = F.n;
  T* dpred = bag.alloc<T>((size_t)n);
  T* dresid = bag.alloc<T>((size_t)n);
  uint8_t* dvalid = bag.alloc<uint8_t>((size_t)n);
  if (!dpred || !dresid || !dvalid) return 1;
  if (grouped_predict<T>(F.X(), F.ld, F.Y(), G.doff, n_groups, n, F.p, G.add_bias, G.dbeta, G.dst, mask, dpred, dresid,
                         dvalid, s, PDSB_GLM_GAUSSIAN, &G.wl)) return 1;
  std::vector<int> hs;
  if (result_copy(out, out->pred, dpred, (size_t)n * sizeof(T), s) ||
      result_copy(out, out->resid, dresid, (size_t)n * sizeof(T), s) ||
      download_status(G.dst, (size_t)n_groups, hs, s)) return 1;
  bool all_ok = !mask;
  for (int64_t g = 0; g < n_groups && all_ok; ++g) all_ok = hs[g] == PDSB_OK;
  if (!all_ok) {
    if (result_copy(out, out->valid, dvalid, (size_t)n, s)) return 1;
    PDSB_CUDA_OK(cudaStreamSynchronize(s));
  }
  out->is_f32 = sizeof(T) == 4; out->n_coef = G.q; out->n_targets = 1; out->n_rows = n;
  return 0;
}

// pl_lr_pred_by: the fit of pl_lr_by with pl_lr_pred's solver settings, then K5's predict pass on the same stream and
// the fit's work list.  The fit sees null rows as NaN, as pl_lr_by's does; the predict pass tells them apart from
// genuine NaN values by a row mask built from the Arrow validity, as build_frame does for pl_lr_pred.  pred / resid
// come back in one copy each; the validity bytes are copied only when some row is null or some group's fit is.
template <typename T>
int host_grouped_pred_t(const pdsb_column* cols, int n_cols, const int64_t* offsets, int64_t n_groups,
                        const pdsb_lr_kwargs* kw, pdsb_host_result* out) {
  NvtxRange nv("pdsb:host_grouped_pred");
  cudaStream_t s;
  if (thread_stream(&s)) return 1;
  NullPolicy pol;
  if (parse_null_policy(kw->null_policy, &pol)) return 1;
  DevBag bag(s);
  GroupedFit<T> G;
  if (grouped_fit<T>(cols, n_cols, offsets, n_groups, kw, pol, 1, G, bag, s)) return 1;
  const Frame<T>& F = G.F;
  const int64_t n = F.n;
  T* mask = nullptr;
  if (F.any_null) {
    UploadPlan plan;
    if (!(mask = row_mask<T>(cols, n_cols, n, F.ld, bag, plan, s)) || plan.run(s)) return 1;
  }
  return grouped_pred_result<T>(G, n_groups, mask, out, bag, s);
}

// pl_lin_reg_report_by: per group, pl_lin_reg_report on that group's rows (K17, kernels/k17_grouped_report.cu).  The frame
// and its checks are pl_lr_by's; var(y) is computed on the device over each group's non-null y, so it needs the y
// column's validity: a null y and a NaN y are both NaN in the frame.  report [n_groups][8][q] f64; valid [n_groups]: 0
// for a group with fewer kept rows than coefficients (a null list).
template <typename T>
int host_grouped_report_t(const pdsb_column* cols, int n_cols, const int64_t* offsets, int64_t n_groups,
                          const pdsb_lr_kwargs* kw, pdsb_host_result* out) {
  NvtxRange nv("pdsb:host_grouped_report");
  cudaStream_t s;
  if (thread_stream(&s)) return 1;
  NullPolicy pol;
  if (parse_null_policy(kw->null_policy, &pol)) return 1;
  if (n_cols - 1 > 64) { set_error("grouped lin_reg_report: %d features; at most 64 are supported", n_cols - 1); return 1; }
  DevBag bag(s);
  Frame<T> F;
  int64_t* doff = nullptr;
  if (lr_by_frame<T>(cols, n_cols, offsets, n_groups, kw, pol, F, doff, bag, s)) return 1;
  T* ymask = nullptr;
  if (col_nulls(cols[0]) > 0) {
    UploadPlan plan;
    if (!(ymask = row_mask<T>(cols, 1, F.n, F.ld, bag, plan, s)) || plan.run(s)) return 1;
  }
  const int add_bias = kw->bias ? 1 : 0, q = F.p + add_bias;
  double* dout = bag.alloc<double>((size_t)n_groups * 8 * q);
  int* dst = bag.alloc<int>((size_t)n_groups);
  if (!dout || !dst) return 1;
  if (grouped_report<T>(F.X(), F.ld, F.Y(), ymask, doff, n_groups, F.n, F.p, add_bias, se_type_from_string(kw->std_err),
                        dout, dst, s)) return 1;
  std::vector<int> hs;
  if (result_copy(out, out->report, dout, (size_t)n_groups * 8 * q * sizeof(double), s) ||
      download_status(dst, (size_t)n_groups, hs, s) || !(out->valid = valid_from_status(out, hs))) return 1;
  out->is_f32 = sizeof(T) == 4; out->n_coef = q; out->n_targets = 1; out->n_rows = n_groups;
  return 0;
}

// pl_lr_w_rcond_by: per group, pl_lr_w_rcond on that group's rows (K19, kernels/k19_grouped_rcond.cu).  The frame and its
// checks are pl_lr_by's; the kernel takes |rcond| from kw->tol and floors it per group, as host_lin_reg_t does for one
// call.  coeffs and singular_values [n_groups][q] rounded to T; valid [n_groups]: 0 for a group with fewer kept rows than
// coefficients (null lists).
template <typename T>
int host_grouped_rcond_t(const pdsb_column* cols, int n_cols, const int64_t* offsets, int64_t n_groups,
                         const pdsb_lr_kwargs* kw, pdsb_host_result* out) {
  NvtxRange nv("pdsb:host_grouped_rcond");
  cudaStream_t s;
  if (thread_stream(&s)) return 1;
  NullPolicy pol;
  if (parse_null_policy(kw->null_policy, &pol)) return 1;
  if (n_cols - 1 > 64) { set_error("grouped lin_reg_w_rcond: %d features; at most 64 are supported", n_cols - 1); return 1; }
  DevBag bag(s);
  Frame<T> F;
  int64_t* doff = nullptr;
  if (lr_by_frame<T>(cols, n_cols, offsets, n_groups, kw, pol, F, doff, bag, s)) return 1;
  pdsb_solve_opts o{};
  o.p = F.p; o.t = 1; o.add_bias = kw->bias ? 1 : 0; o.method = PDSB_METHOD_RCOND; o.l2_reg = kw->l2_reg; o.tol = kw->tol;
  const int q = F.p + o.add_bias;
  double* dbeta = bag.alloc<double>((size_t)n_groups * q);
  double* dsv = bag.alloc<double>((size_t)n_groups * q);
  int* dst = bag.alloc<int>((size_t)n_groups);
  if (!dbeta || !dsv || !dst) return 1;
  if (grouped_lin_reg_rcond<T>(F.X(), F.ld, F.Y(), doff, n_groups, F.n, F.p, o, dbeta, dsv, dst, s)) return 1;
  return grouped_coeffs_result<T>(dbeta, dst, n_groups, q, out, s, 1, dsv);
}

// pl_logistic_by / pl_logistic_pred_by: per group, host_logistic on that group's rows alone, for all groups in one K16
// call (kernels/k16_grouped_logistic.cu).  The frame is built as host_logistic builds it, with the kwarg's null policy
// (so every policy works, and "skip" drops rows through the mask); a group left without a kept row is host_logistic's
// "Empty data".  Coefficients, or the probabilities of K5's predict pass with the binomial link (K10's
// predict_strided rule), come back in one copy; the validity bytes only with a mask.
int host_grouped_logistic(const pdsb_column* cols, int n_cols, const int64_t* offsets, int64_t n_groups,
                          const pdsb_lr_kwargs* kw, int want_pred, pdsb_host_result* out) {
  NvtxRange nv("pdsb:host_grouped_logistic");
  typedef double T;
  cudaStream_t s;
  if (thread_stream(&s)) return 1;
  NullPolicy pol;
  if (parse_null_policy(kw->null_policy, &pol)) return 1;
  DevBag bag(s);
  Frame<T> F;
  int64_t* doff = nullptr;
  if (grouped_frame<T>(cols, n_cols, 1, pol, false, false, offsets, n_groups, "grouped lin_reg", F, doff, bag, s)) return 1;
  const int p = F.p, add_bias = kw->bias ? 1 : 0, q = p + add_bias;
  const int64_t n = F.n;
  if (p > 64) { set_error("logistic_reg: more than 64 features are not supported"); return 1; }
  double* dbeta = bag.alloc<double>((size_t)n_groups * q);
  int* dst = bag.alloc<int>((size_t)n_groups);
  if (!dbeta || !dst) return 1;
  if (grouped_logistic(F.X(), F.ld, F.Y(), F.mask, doff, n_groups, n, p, add_bias, kw->l1_reg, kw->l2_reg, kw->tol,
                       kw->max_iter, dbeta, dst, nullptr, s)) return 1;
  out->is_f32 = 0; out->n_coef = q; out->n_targets = 1;
  if (want_pred) {
    T* dpred = bag.alloc<T>((size_t)n);
    uint8_t* dvalid = bag.alloc<uint8_t>((size_t)n);
    if (!dpred || !dvalid) return 1;
    if (grouped_predict<T>(F.X(), F.ld, nullptr, doff, n_groups, n, p, add_bias, dbeta, nullptr, F.mask, dpred, nullptr,
                           dvalid, s, PDSB_GLM_BINOMIAL)) return 1;
    if (result_copy(out, out->pred, dpred, (size_t)n * sizeof(T), s)) return 1;
    if (F.mask && result_copy(out, out->valid, dvalid, (size_t)n, s)) return 1;
    out->n_rows = n;
  } else {
    if (result_copy(out, out->coeffs, dbeta, (size_t)n_groups * q * sizeof(double), s)) return 1;
    out->n_rows = n_groups;
  }
  std::vector<int> hs;
  if (download_status(dst, (size_t)n_groups, hs, s)) return 1;
  for (int64_t g = 0; g < n_groups; ++g)
    if (hs[g] == PDSB_LOGISTIC_EMPTY) { set_error("Empty data"); return 1; }
  return 0;
}

// pl_singular_values_by / pl_pca_by / pl_principal_components_by: per group, host_pca_t on that group's rows (K18,
// kernels/k18_grouped_pca.cu).  Nulls are uploaded as NaN and the row mask marks the rows that have one, so the device
// takes each column's mean over its own non-null values and drops the masked rows from the Gram.  The whole-call errors
// are the loop's: the first group in order that would fail its single call decides the message.
template <typename T>
int host_pca_by_t(const pdsb_column* cols, int n_cols, const int64_t* offsets, int64_t n_groups, int mode, int k,
                  int center, pdsb_host_result* out) {
  NvtxRange nv("pdsb:host_pca_by");
  cudaStream_t s;
  if (thread_stream(&s)) return 1;
  const int p = n_cols;
  const int64_t n = col_len(cols[0]);
  for (int c = 1; c < n_cols; ++c)
    if (col_len(cols[c]) != n) { set_error("Seires don't have the same length."); return 1; }
  if (check_group_offsets(offsets, n_groups, n)) return 1;
  bool any_null = false;
  for (int c = 0; c < n_cols; ++c) any_null |= col_nulls(cols[c]) > 0;
  if (mode == 2 && any_null) { set_error("Nulls are found in data and this method doesn't allow nulls."); return 1; }
  out->is_f32 = 0; out->n_coef = p;
  std::vector<int> hst((size_t)n_groups * 2, 0);       // every group empty when n == 0: dim 0, nothing to run
  DevBag bag(s);
  T* X = nullptr;
  int64_t* doff = nullptr;
  double *dmean = nullptr, *dsig = nullptr, *dV = nullptr, *dout = nullptr;
  int* dst = nullptr;
  const int64_t ld = pad_ld(n);
  if (n > 0) {
    UploadPlan plan;
    X = bag.alloc<T>((size_t)ld * p);
    dmean = center ? bag.alloc<double>((size_t)n_groups * p) : nullptr;
    dsig = bag.alloc<double>((size_t)n_groups * p);
    dV = bag.alloc<double>((size_t)n_groups * p * p);
    dst = bag.alloc<int>((size_t)n_groups * 2);
    if (!X || (center && !dmean) || !dsig || !dV || !dst) return 1;
    for (int c = 0; c < n_cols; ++c)
      if (upload_column<T>(cols[c], X + (size_t)c * ld, 0, T(0), bag, plan, s)) return 1;
    T* mask = nullptr;
    if (any_null && !(mask = row_mask<T>(cols, n_cols, n, ld, bag, plan, s))) return 1;
    if (plan.run(s) || upload_offsets(offsets, n_groups, doff, bag, s)) return 1;
    if (grouped_pca<T>(X, ld, mask, doff, n_groups, n, p, center, dmean, dsig, dV, dst, s)) return 1;
    if (mode == 2) {
      if (!(dout = bag.alloc<double>((size_t)k * n))) return 1;
      if (grouped_project<T>(X, ld, doff, n_groups, n, p, dmean, dV, k, dout, n, s)) return 1;
    }
    if (download_status(dst, hst.size(), hst, s)) return 1;
  }
  for (int64_t g = 0; g < n_groups; ++g) {
    const int64_t len = offsets[g + 1] - offsets[g];
    if (mode == 2) {
      if (len < k) continue;                                       // pca.rs:90-93: NaN rows, no error
      if (len < p) {
        set_error("principal_components: %lld rows < %d features is not supported (k <= rows < features)", (long long)len, p);
        return 1;
      }
    }
    if (len > 0 && hst[2 * g] != PDSB_PCA_OK) { set_error("SVD algorithm did not converge."); return 1; }
    if (mode == 1 && hst[2 * g + 1] < p) { set_error("pca: %d rows < %d features is not supported", hst[2 * g + 1], p); return 1; }
  }
  if (mode == 2) {
    out->n_targets = k; out->n_rows = n;
    if (n == 0) return (out->pred = result_buf(out, 0)) ? 0 : 1;
    if (result_copy(out, out->pred, dout, (size_t)k * n * sizeof(double), s)) return 1;
    PDSB_CUDA_OK(cudaStreamSynchronize(s));
    return 0;
  }
  out->n_rows = n_groups;
  if (mode == 1) {
    if (result_copy(out, out->singular_values, dsig, (size_t)n_groups * p * sizeof(double), s) ||
        result_copy(out, out->coeffs, dV, (size_t)n_groups * p * p * sizeof(double), s)) return 1;
    PDSB_CUDA_OK(cudaStreamSynchronize(s));
    return 0;
  }
  // mode 0: each group's first dim_g values, one after the other, and the list offsets
  std::vector<double> hs((size_t)n_groups * p);
  if (n > 0) {
    PDSB_CUDA_OK(cudaMemcpyAsync(hs.data(), dsig, hs.size() * sizeof(double), cudaMemcpyDeviceToHost, s));
    PDSB_CUDA_OK(cudaStreamSynchronize(s));
  }
  int64_t* lo = static_cast<int64_t*>(result_buf(out, (size_t)(n_groups + 1) * sizeof(int64_t)));
  if (!lo) return 1;
  lo[0] = 0;
  for (int64_t g = 0; g < n_groups; ++g) lo[g + 1] = lo[g] + hst[2 * g + 1];
  double* sv = static_cast<double*>(result_buf(out, (size_t)lo[n_groups] * sizeof(double)));
  if (!sv) return 1;
  for (int64_t g = 0; g < n_groups; ++g)
    for (int i = 0; i < hst[2 * g + 1]; ++i) sv[lo[g] + i] = hs[(size_t)g * p + i];
  out->singular_values = sv; out->coeffs = lo;
  return 0;
}

// f(row) for every null row of c, in row order
template <typename F>
void for_each_null(const pdsb_column& c, F f) {
  int64_t r0 = 0;
  for (int i = 0; i < c.n_chunks; ++i) {
    const pdsb_chunk& ch = c.chunks[i];
    if (ch.validity)
      for (int64_t j = 0; j < ch.length; ++j) {
        const int64_t b = ch.offset + j;
        if (!((ch.validity[b >> 3] >> (b & 7)) & 1)) f(r0 + j);
      }
    r0 += ch.length;
  }
}

// pl_isotonic_regression_by: per group, host_isotonic_regression on the group's rows, in one device call (K15).  The
// reference's checks run over all groups of >= 2 rows in its order (y nulls, w nulls, w <= 0), so when groups fail for
// different reasons the message can differ from the one Polars' loop stops at (DESIGN §5).  One-row groups pass y
// through, validity included, without looking at their weight.
int host_grouped_isotonic(const pdsb_column* cols, int n_cols, const int64_t* offsets, int64_t n_groups, int has_weights,
                          int increasing, pdsb_host_result* out) {
  NvtxRange nv("pdsb:host_grouped_isotonic");
  if (n_cols < (has_weights ? 2 : 1)) {
    set_error("isotonic_regression: expected %d inputs, got %d", has_weights ? 2 : 1, n_cols); return 1;
  }
  if (cols[0].dtype != PDSB_F64) { set_error("invalid series dtype: expected `Float64` for input 0"); return 1; }
  const int64_t n = col_len(cols[0]);
  if (check_group_offsets(offsets, n_groups, n, "grouped isotonic_regression")) return 1;
  out->is_f32 = 0; out->n_rows = n; out->n_targets = 1;
  // the group of each null row, walked in row order; true if it has >= 2 rows
  auto null_in_fitted_group = [&](const pdsb_column& c) {
    bool hit = false;
    int64_t g = 0;
    for_each_null(c, [&](int64_t r) {
      while (offsets[g + 1] <= r) ++g;
      hit |= offsets[g + 1] - offsets[g] >= 2;
    });
    return hit;
  };
  bool fitted = false;                            // some group of >= 2 rows
  for (int64_t g = 0; g < n_groups && !fitted; ++g) fitted = offsets[g + 1] - offsets[g] >= 2;
  if (fitted && col_nulls(cols[0]) > 0 && null_in_fitted_group(cols[0])) { set_error("Input should not contain nulls."); return 1; }
  // With no group of >= 2 rows the weights are never read, so their dtype and length go unchecked: the single call
  // answers n <= 1 the same way, before it looks at w.
  if (fitted && has_weights) {
    if (cols[1].dtype != PDSB_F64) { set_error("invalid series dtype: expected `Float64` for input 1"); return 1; }
    if (col_len(cols[1]) != n) { set_error("Weights should not contain nulls and must be the same length as y."); return 1; }
    if (col_nulls(cols[1]) > 0 && null_in_fitted_group(cols[1])) { set_error("Weight should not contain nulls."); return 1; }
  }
  double* pred = nullptr;
  if (fitted) {
    cudaStream_t s;
    if (thread_stream(&s)) return 1;
    DevBag bag(s);
    double* dyw[2] = {nullptr, nullptr};     // y, w
    double* dout = bag.alloc<double>((size_t)n);
    int* dst = bag.alloc<int>((size_t)n_groups);
    int64_t* doff = nullptr;
    if (!dout || !dst || upload_f64(cols, has_weights ? 2 : 1, n, dyw, bag, s) || upload_offsets(offsets, n_groups, doff, bag, s))
      return 1;
    if (pdsb_dev_grouped_isotonic_f64(dyw[0], dyw[1], doff, n_groups, n, increasing, dout, dst, s)) return 1;
    std::vector<int> st;
    if (result_copy(out, pred, dout, (size_t)n * sizeof(double), s) || download_status(dst, (size_t)n_groups, st, s))
      return 1;
    for (int64_t g = 0; g < n_groups; ++g)
      if (offsets[g + 1] - offsets[g] >= 2 && (st[g] & PDSB_ISO_NONPOSITIVE_WEIGHT)) {
        set_error("Weight should not contain negative values."); return 1;
      }
  } else if (!(pred = static_cast<double*>(result_buf(out, (size_t)n * sizeof(double))))) {
    return 1;
  }
  out->pred = pred;
  // one-row groups: y as it is, a null included
  RowReader y{cols[0]};
  for (int64_t g = 0; g < n_groups; ++g) {
    if (offsets[g + 1] - offsets[g] != 1) continue;
    const int64_t r = offsets[g];
    pred[r] = 0.0;
    const bool valid = y.at(r, &pred[r]);
    if (!valid && !out->valid) {
      if (!(out->valid = static_cast<uint8_t*>(result_buf(out, (size_t)n)))) return 1;
      memset(out->valid, 1, (size_t)n);
    }
    if (!valid) out->valid[r] = 0;
  }
  return 0;
}

// pl_recursive_lr_by (rolling = 0) and the rolling twin: per group, host_online_t on the group's rows, in one device
// call (K6 over groups).  The single call's checks run group by group in group order, so the call fails with the message
// Polars' loop stops at; skip is per group, as each single call sets it from its own rows' nulls (after the rolling
// rename of the policy).  The frame is built once for all rows: a null becomes NaN or the fill value in every group
// alike.  The checks (grouped_online_checks) read host data only; host_grouped_online_t is the device part.
const char* online_name(int rolling) { return rolling ? "grouped rolling_lin_reg" : "grouped recursive_lin_reg"; }

struct GroupedOnline {
  NullPolicy pol;
  int64_t n = 0;
  int q = 0, add_bias = 0;
  std::vector<uint8_t> skip;   // [n_groups] 0 / 1
  bool any_skip = false;
};

int grouped_online_checks(const pdsb_column* cols, int n_cols, const int64_t* offsets, int64_t n_groups,
                          const pdsb_lr_kwargs* kw, int rolling, GroupedOnline& a) {
  NullPolicy& pol = a.pol;
  if (parse_null_policy(kw->null_policy, &pol)) return 1;
  if (rolling) {   // as host_online_t
    if (pol.kind == NullKind::SKIP) pol.kind = NullKind::SKIP_WINDOW;
    else if (pol.kind == NullKind::FILL) pol.kind = NullKind::FILL_WINDOW;
  }
  const int64_t n = checked_rows(cols, n_cols, 1);
  if (n < 0) return 1;
  if (check_group_offsets(offsets, n_groups, n, online_name(rolling))) return 1;
  std::vector<uint8_t> any_null((size_t)n_groups, 0), y_null((size_t)n_groups, 0);   // per group: a null row, a null y
  for (int c = 0; c < n_cols; ++c) {
    if (col_nulls(cols[c]) == 0) continue;
    int64_t g = 0;
    for_each_null(cols[c], [&](int64_t r) {
      while (offsets[g + 1] <= r) ++g;
      any_null[g] = 1;
      if (c == 0) y_null[g] = 1;
    });
  }
  a.n = n;
  a.add_bias = kw->bias ? 1 : 0;
  const int q = a.q = n_cols - 1 + a.add_bias;
  std::vector<uint8_t>& skip = a.skip;
  skip.assign((size_t)n_groups, 0);
  for (int64_t g = 0; g < n_groups; ++g) {
    const int64_t len = offsets[g + 1] - offsets[g];
    if (len == 0) { set_error("Empty data"); return 1; }
    if (pol.kind == NullKind::RAISE && any_null[g]) { set_error("Nulls found in data"); return 1; }
    if (len < q) { set_error("#Data < #features. No conclusive result."); return 1; }
    if (kw->n < 1) { set_error("window / start_with must be >= 1"); return 1; }
    if (kw->n > len) { set_error("#Data < window size. No conclusive result."); return 1; }
    if (rolling) skip[g] = (pol.kind == NullKind::SKIP_WINDOW && any_null[g]) || (pol.kind == NullKind::FILL_WINDOW && y_null[g]);
    else skip[g] = (pol.kind == NullKind::SKIP && any_null[g]) || (pol.kind == NullKind::FILL && y_null[g]);
    a.any_skip |= skip[g] != 0;
  }
  return 0;
}

template <typename T>
int host_grouped_online_t(const pdsb_column* cols, int n_cols, const int64_t* offsets, int64_t n_groups,
                          const pdsb_lr_kwargs* kw, int rolling, const GroupedOnline& a, pdsb_host_result* out) {
  NvtxRange nv(rolling ? "pdsb:host_grouped_rolling" : "pdsb:host_grouped_recursive");
  const int64_t n = a.n;
  const int q = a.q, add_bias = a.add_bias;
  const bool any_skip = a.any_skip;
  cudaStream_t s;
  if (thread_stream(&s)) return 1;
  DevBag bag(s);
  Frame<T> F;
  int64_t* doff = nullptr;
  if (grouped_frame<T>(cols, n_cols, 1, a.pol, false, true, offsets, n_groups, online_name(rolling), F, doff, bag, s))
    return 1;
  uint8_t* dskip = any_skip ? bag.alloc<uint8_t>((size_t)n_groups) : nullptr;
  T* dco = bag.alloc<T>((size_t)n * q);
  T* dpr = bag.alloc<T>((size_t)n);
  uint8_t* dva = bag.alloc<uint8_t>((size_t)n);
  if ((any_skip && !dskip) || !dco || !dpr || !dva) return 1;
  if (any_skip) PDSB_CUDA_OK(cudaMemcpyAsync(dskip, a.skip.data(), (size_t)n_groups, cudaMemcpyHostToDevice, s));
  if (rolling ? grouped_rolling_lin_reg<T>(F.X(), F.ld, F.Y(), doff, dskip, n_groups, n, F.p, add_bias, kw->n,
                                           kw->min_size, kw->lambda, dco, dpr, dva, s)
              : grouped_recursive_lin_reg<T>(F.X(), F.ld, F.Y(), doff, dskip, n_groups, n, F.p, add_bias, kw->n, kw->lambda,
                                             dco, dpr, dva, s)) return 1;
  out->is_f32 = sizeof(T) == 4; out->n_coef = q; out->n_targets = 1; out->n_rows = n;
  if (result_copy(out, out->coeffs, dco, (size_t)n * q * sizeof(T), s) ||
      result_copy(out, out->pred, dpr, (size_t)n * sizeof(T), s) ||
      result_copy(out, out->valid, dva, (size_t)n, s)) return 1;
  PDSB_CUDA_OK(cudaStreamSynchronize(s));
  return 0;
}

// pl_wls_by / pl_wls_pred_by: per group, the single weighted pl_lr / pl_lr_pred on that group's rows (inputs [w, y,
// features...]), from one upload in key order and one K5 launch sequence with the weighted moments pass
// (grouped_wls_lin_reg).  Every decision the single call takes from host data is settled here, group by group in key
// order, before any device work (wls_group_checks); the rest follows pl_lr_by (DESIGN §5 item 33).
//
// The single call masks a row when the policy is "skip" and one of y, x is null, or a fill and y is null.  With a mask
// it counts the rows as llround(sum of w over the unmasked rows), and a NaN / inf / null weight on any row of the call
// makes that sum NaN: fewer rows than coefficients is "#Data < #features. No conclusive result.", any other count but the
// group's length is "Shape of weights is not the same as the data.".
int wls_group_checks(const pdsb_column* data, int n_data, const pdsb_column& w, const int64_t* offsets, int64_t n_groups,
                     const NullPolicy& pol, int q) {
  std::vector<uint8_t> any_null((size_t)n_groups, 0), y_null((size_t)n_groups, 0);
  for (int c = 0; c < n_data; ++c) {
    if (col_nulls(data[c]) == 0) continue;
    int64_t g = 0;
    for_each_null(data[c], [&](int64_t r) {
      while (offsets[g + 1] <= r) ++g;
      any_null[g] = 1;
      if (c == 0) y_null[g] = 1;
    });
  }
  RowReader wr{w};
  std::vector<RowReader> dr;
  for (int c = 0; c < n_data; ++c) dr.push_back(RowReader{data[c]});
  for (int64_t g = 0; g < n_groups; ++g) {
    const int64_t len = offsets[g + 1] - offsets[g];
    if (len == 0) continue;
    if (pol.kind == NullKind::RAISE && any_null[g]) { set_error("Nulls found in data"); return 1; }
    const bool masked = (pol.kind == NullKind::SKIP && any_null[g]) || (pol.kind == NullKind::FILL && y_null[g]);
    if (masked) {
      const int mask_cols = pol.kind == NullKind::SKIP ? n_data : 1;
      double sw = 0.0;
      bool finite = true;
      for (int64_t r = offsets[g]; r < offsets[g + 1]; ++r) {
        double v = NAN, d;
        finite = wr.at(r, &v) && std::isfinite(v) && finite;
        bool kept = true;
        for (int c = 0; c < mask_cols; ++c) kept = dr[c].at(r, &d) && kept;
        if (kept) sw += v;
      }
      const int64_t n_valid = finite ? (int64_t)llround(sw) : INT64_MIN;
      if (n_valid < q) { set_error("#Data < #features. No conclusive result."); return 1; }
      if (n_valid != len) { set_error("Shape of weights is not the same as the data."); return 1; }
    }
  }
  return 0;
}

// The host-only part of pl_wls_by: the single call's shape checks, the offsets, the feature limit and the group
// decisions, in that order
struct GroupedWls {
  NullPolicy pol;
  int64_t n = 0;
  int p = 0, q = 0, add_bias = 0;
};

int grouped_wls_checks(const pdsb_column* cols, int n_cols, const int64_t* offsets, int64_t n_groups,
                       const pdsb_lr_kwargs* kw, GroupedWls& a) {
  if (parse_null_policy(kw->null_policy, &a.pol)) return 1;
  const pdsb_column* data = cols + 1;
  const int n_data = n_cols - 1;
  a.n = checked_rows(data, n_data, 1);
  if (a.n < 0 || check_weights(cols[0], a.n)) return 1;
  if (check_group_offsets(offsets, n_groups, a.n, "grouped weighted lin_reg")) return 1;
  a.p = n_data - 1; a.add_bias = kw->bias ? 1 : 0; a.q = a.p + a.add_bias;
  if (a.p > 64) { set_error("grouped weighted lin_reg: %d features; at most 64 are supported", a.p); return 1; }
  return wls_group_checks(data, n_data, cols[0], offsets, n_groups, a.pol, a.q);
}

template <typename T>
int host_grouped_wls_t(const pdsb_column* cols, int n_cols, const int64_t* offsets, int64_t n_groups,
                       const pdsb_lr_kwargs* kw, int want_pred, const GroupedWls& a, pdsb_host_result* out) {
  NvtxRange nv("pdsb:host_grouped_wls");
  cudaStream_t s;
  if (thread_stream(&s)) return 1;
  const NullPolicy& pol = a.pol;
  const pdsb_column* data = cols + 1;
  const int n_data = n_cols - 1;
  const int64_t n = a.n;
  const int p = a.p, q = a.q;
  DevBag bag(s);
  GroupedFit<T> G;
  Frame<T>& F = G.F;
  // online: a null becomes NaN (a fill for the features under a fill policy), a null weight NaN, and the moments pass
  // drops every row with a NaN
  if (build_frame<T>(data, n_data, 1, &cols[0], pol, false, true, F, bag, s) || upload_offsets(offsets, n_groups, G.doff, bag, s))
    return 1;
  pdsb_solve_opts o = lr_solve_opts(kw, p, 1, sizeof(T) == 4, want_pred);
  o.method = PDSB_METHOD_LSTSQ; o.l2_reg = 0.0; o.singular_x_tol = 0.0;   // faer_weighted_lr: no ridge, no gate
  G.q = q; G.add_bias = a.add_bias;
  G.dbeta = bag.alloc<double>((size_t)n_groups * q);
  G.dst = bag.alloc<int>((size_t)n_groups);
  if (!G.dbeta || !G.dst) return 1;
  if (grouped_wls_lin_reg<T>(F.X(), F.ld, F.Y(), F.w, G.doff, n_groups, n, p, o, G.dbeta, G.dst, s, &bag,
                             want_pred ? &G.wl : nullptr)) return 1;
  if (!want_pred) return grouped_coeffs_result<T>(G.dbeta, G.dst, n_groups, q, out, s);
  // the rows the single call masks (and returns as null): a null y or x under "skip", a null y under a fill
  const int mask_cols = pol.kind == NullKind::SKIP ? n_data : (pol.kind == NullKind::FILL ? 1 : 0);
  bool any_masked = false;
  for (int c = 0; c < mask_cols; ++c) any_masked |= col_nulls(data[c]) > 0;
  T* mask = nullptr;
  if (any_masked) {
    UploadPlan plan;
    if (!(mask = row_mask<T>(data, mask_cols, n, F.ld, bag, plan, s)) || plan.run(s)) return 1;
  }
  return grouped_pred_result<T>(G, n_groups, mask, out, bag, s);
}

int null_group_args(const int64_t* offsets, const void* kw, const void* cols, const void* out) {
  if (!offsets) { set_error("null group offsets"); return 1; }
  return null_args(kw, cols, out);
}

// pdsb_host_grouped_recursive and pdsb_host_grouped_rolling: null arguments, then the group checks, then the device part
template <bool ARGS_FIRST>
int host_grouped_online(const pdsb_column* cols, int n_cols, const int64_t* offsets, int64_t n_groups,
                        const pdsb_lr_kwargs* kw, int f32, int rolling, pdsb_host_result* out) {
  GroupedOnline a;
  return guarded<ARGS_FIRST>(out, [&] {
    return null_group_args(offsets, kw, cols, out) || grouped_online_checks(cols, n_cols, offsets, n_groups, kw, rolling, a);
  }, [&] {
    return f32 ? host_grouped_online_t<float>(cols, n_cols, offsets, n_groups, kw, rolling, a, out)
               : host_grouped_online_t<double>(cols, n_cols, offsets, n_groups, kw, rolling, a, out);
  });
}

}  // namespace
}  // namespace pdsb

using namespace pdsb;

extern "C" {

int pdsb_host_grouped_recursive(const pdsb_column* cols, int n_cols, const int64_t* group_offsets, int64_t n_groups,
                                const pdsb_lr_kwargs* kw, int f32, pdsb_host_result* out) {
  return host_grouped_online<false>(cols, n_cols, group_offsets, n_groups, kw, f32, 0, out);
}
int pdsb_host_grouped_rolling(const pdsb_column* cols, int n_cols, const int64_t* group_offsets, int64_t n_groups,
                              const pdsb_lr_kwargs* kw, int f32, pdsb_host_result* out) {
  return host_grouped_online<true>(cols, n_cols, group_offsets, n_groups, kw, f32, 1, out);
}
int pdsb_host_grouped_lin_reg(const pdsb_column* cols, int n_cols, const int64_t* group_offsets, int64_t n_groups,
                              const pdsb_lr_kwargs* kw, int f32, pdsb_host_result* out) {
  return guarded(out, [&] { return null_group_args(group_offsets, kw, cols, out); }, [&] {
    return f32 ? host_grouped_t<float>(cols, n_cols, group_offsets, n_groups, kw, out)
               : host_grouped_t<double>(cols, n_cols, group_offsets, n_groups, kw, out);
  });
}
int pdsb_host_grouped_ar(const pdsb_column* cols /* x */, const int64_t* group_offsets, int64_t n_groups, int lag,
                         const pdsb_lr_kwargs* kw, int f32, pdsb_host_result* out) {
  return guarded(out, [&] { return null_group_args(group_offsets, kw, cols, out); }, [&] {
    return f32 ? host_grouped_ar_t<float>(*cols, group_offsets, n_groups, lag, kw, out)
               : host_grouped_ar_t<double>(*cols, group_offsets, n_groups, lag, kw, out);
  });
}
int pdsb_host_grouped_lin_reg_pred(const pdsb_column* cols, int n_cols, const int64_t* group_offsets, int64_t n_groups,
                                   const pdsb_lr_kwargs* kw, int f32, pdsb_host_result* out) {
  return guarded(out, [&] { return null_group_args(group_offsets, kw, cols, out); }, [&] {
    return f32 ? host_grouped_pred_t<float>(cols, n_cols, group_offsets, n_groups, kw, out)
               : host_grouped_pred_t<double>(cols, n_cols, group_offsets, n_groups, kw, out);
  });
}
int pdsb_host_grouped_wls(const pdsb_column* cols, int n_cols, const int64_t* group_offsets, int64_t n_groups,
                          const pdsb_lr_kwargs* kw, int f32, int want_pred, pdsb_host_result* out) {
  GroupedWls a;
  return guarded<true>(out, [&] {
    return null_group_args(group_offsets, kw, cols, out) || grouped_wls_checks(cols, n_cols, group_offsets, n_groups, kw, a);
  }, [&] {
    return f32 ? host_grouped_wls_t<float>(cols, n_cols, group_offsets, n_groups, kw, want_pred, a, out)
               : host_grouped_wls_t<double>(cols, n_cols, group_offsets, n_groups, kw, want_pred, a, out);
  });
}
int pdsb_host_grouped_report(const pdsb_column* cols, int n_cols, const int64_t* group_offsets, int64_t n_groups,
                             const pdsb_lr_kwargs* kw, int f32, pdsb_host_result* out) {
  return guarded(out, [&] { return null_group_args(group_offsets, kw, cols, out); }, [&] {
    return f32 ? host_grouped_report_t<float>(cols, n_cols, group_offsets, n_groups, kw, out)
               : host_grouped_report_t<double>(cols, n_cols, group_offsets, n_groups, kw, out);
  });
}
int pdsb_host_grouped_lin_reg_rcond(const pdsb_column* cols, int n_cols, const int64_t* group_offsets,
                                    int64_t n_groups, const pdsb_lr_kwargs* kw, int f32, pdsb_host_result* out) {
  return guarded(out, [&] { return null_group_args(group_offsets, kw, cols, out); }, [&] {
    return f32 ? host_grouped_rcond_t<float>(cols, n_cols, group_offsets, n_groups, kw, out)
               : host_grouped_rcond_t<double>(cols, n_cols, group_offsets, n_groups, kw, out);
  });
}
int pdsb_host_grouped_lin_reg_multi(const pdsb_column* cols, int n_cols, const int64_t* group_offsets,
                                    int64_t n_groups, const pdsb_lr_kwargs* kw, int n_targets, int f32,
                                    pdsb_host_result* out) {
  return guarded(out, [&] {
    if (null_group_args(group_offsets, kw, cols, out)) return 1;
    if (n_targets < 1 || n_targets >= n_cols) { set_error("last_target_idx out of range"); return 1; }
    return 0;
  }, [&] {
    return f32 ? host_grouped_multi_t<float>(cols, n_cols, group_offsets, n_groups, kw, n_targets, out)
               : host_grouped_multi_t<double>(cols, n_cols, group_offsets, n_groups, kw, n_targets, out);
  });
}
int pdsb_host_grouped_logistic(const pdsb_column* cols, int n_cols, const int64_t* group_offsets, int64_t n_groups,
                               const pdsb_lr_kwargs* kw, int want_pred, pdsb_host_result* out) {
  return guarded(out, [&] { return null_group_args(group_offsets, kw, cols, out); },
                 [&] { return host_grouped_logistic(cols, n_cols, group_offsets, n_groups, kw, want_pred, out); });
}

int pdsb_host_pca_by(const pdsb_column* cols, int n_cols, const int64_t* group_offsets, int64_t n_groups, int mode,
                     int k, int center, pdsb_host_result* out) {
  return guarded(out, [&] {
    if (!cols || !out || !group_offsets || n_cols < 1 || mode < 0 || mode > 2) { set_error("pca: invalid arguments"); return 1; }
    if (n_cols > 64) { set_error("grouped pca: %d features; at most 64 are supported", n_cols); return 1; }
    if (mode == 2 && (k < 1 || k > n_cols)) { set_error("Input `k` should be between 1 and the number of features inclusive."); return 1; }
    return 0;
  }, [&] {
    return all_f32(cols, n_cols) ? host_pca_by_t<float>(cols, n_cols, group_offsets, n_groups, mode, k, center, out)
                                 : host_pca_by_t<double>(cols, n_cols, group_offsets, n_groups, mode, k, center, out);
  });
}

int pdsb_host_grouped_isotonic(const pdsb_column* cols, int n_cols, const int64_t* group_offsets, int64_t n_groups,
                               int has_weights, int increasing, pdsb_host_result* out) {
  return guarded(out, [&] {
    if (!cols || !out || !group_offsets) { set_error("isotonic_regression: invalid arguments"); return 1; }
    return 0;
  }, [&] { return host_grouped_isotonic(cols, n_cols, group_offsets, n_groups, has_weights, increasing, out); });
}

}  // extern "C"
