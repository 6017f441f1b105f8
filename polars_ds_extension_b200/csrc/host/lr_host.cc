// Host layer of the C ABI (pdsb_host_*): the orchestration the reference does in Rust inside each
// `#[polars_expr] fn pl_lr*` (/root/reference/src/num_ext/linear_regression.rs:419-1283) — kwargs dispatch, null
// policy, packing — rewritten around a device-resident, column-major design matrix:
//   Arrow chunks --H2D (straight DMA when dtype matches and no nulls, else raw upload + K1 cast/validity)-->
//   Z = [targets | features] in HBM  -->  K2 moments  -->  K3 solve  -->  K4 predict / K6 online / K9 report
//   --> D2H into pooled pinned buffers handed to the caller.
// Dropped rows (null policy skip / fill-with-null-target) are zeroed + masked instead of filtered, so no compaction
// pass exists; the physical ones column of the reference (:180-182) is never built.
#include "../common.h"
#include "../kernels/kernels.h"
#include "host.h"
#include <cstring>
#include <cmath>
#include <cfloat>
#include <strings.h>
#include <algorithm>
#include <functional>

namespace pdsb {

int parse_null_policy(const char* s, NullPolicy* out) {
  if (!s) s = "";
  if (!strcasecmp(s, "raise")) { *out = {NullKind::RAISE, 0.0}; return 0; }
  if (!strcasecmp(s, "skip")) { *out = {NullKind::SKIP, 0.0}; return 0; }
  if (!strcasecmp(s, "zero")) { *out = {NullKind::FILL, 0.0}; return 0; }
  if (!strcasecmp(s, "one")) { *out = {NullKind::FILL, 1.0}; return 0; }
  if (!strcasecmp(s, "ignore")) { *out = {NullKind::IGNORE, 0.0}; return 0; }
  if (!strcasecmp(s, "skip_window")) { *out = {NullKind::SKIP_WINDOW, 0.0}; return 0; }
  char* end = nullptr;
  double v = strtod(s, &end);
  if (end != s && end && *end == '\0') { *out = {NullKind::FILL, v}; return 0; }
  set_error("Invalid NullPolicy.");
  return 1;
}

int solver_from_string(const char* s) {
  if (s && !strcmp(s, "svd")) return PDSB_SOLVER_SVD;
  if (s && !strcmp(s, "choleskey")) return PDSB_SOLVER_CHOLESKEY;
  return PDSB_SOLVER_QR;
}

int se_type_from_string(const char* s) {
  if (!s) return 0;
  if (!strcmp(s, "hc0")) return 1;
  if (!strcmp(s, "hc1")) return 2;
  if (!strcmp(s, "hc2")) return 3;
  if (!strcmp(s, "hc3")) return 4;
  return 0;
}

namespace {

template <typename T> struct DT;
template <> struct DT<float> { static constexpr int code = PDSB_F32; };
template <> struct DT<double> { static constexpr int code = PDSB_F64; };

size_t dtype_size(int dt) {
  switch (dt) {
    case PDSB_F32: case PDSB_I32: case PDSB_U32: return 4;
    case PDSB_F64: case PDSB_I64: case PDSB_U64: return 8;
    case PDSB_I16: case PDSB_U16: return 2;
    case PDSB_I8: case PDSB_U8: return 1;
    default: return 0;  // BOOL is bit-packed
  }
}

int64_t col_len(const pdsb_column& c) {
  int64_t n = 0;
  for (int i = 0; i < c.n_chunks; ++i) n += c.chunks[i].length;
  return n;
}

int64_t chunk_nulls(const pdsb_chunk& ch) {
  if (!ch.validity || ch.length == 0) return 0;
  int64_t valid = 0;
  int64_t b = ch.offset;
  const int64_t end = ch.offset + ch.length;
  for (; b < end && (b & 7); ++b) valid += (ch.validity[b >> 3] >> (b & 7)) & 1;       // head bits
  const int64_t full_end = b + ((end - b) & ~int64_t(7));
  const uint8_t* v = ch.validity + (b >> 3);
  int64_t nbytes = (full_end - b) >> 3;
  while (nbytes >= 8) { uint64_t w; memcpy(&w, v, 8); valid += __builtin_popcountll(w); v += 8; nbytes -= 8; }
  while (nbytes-- > 0) valid += __builtin_popcount(*v++);
  for (b = full_end; b < end; ++b) valid += (ch.validity[b >> 3] >> (b & 7)) & 1;      // tail bits
  return ch.length - valid;
}

int64_t col_nulls(const pdsb_column& c) {
  if (c.null_count >= 0) return c.null_count;
  int64_t k = 0;
  for (int i = 0; i < c.n_chunks; ++i) k += chunk_nulls(c.chunks[i]);
  return k;
}

// All host->device copies of one frame are collected first and executed together (h2d.cc: pinned sources DMA directly,
// pageable sources are staged by several host threads); kernels that consume uploaded raw bytes run afterwards.
struct UploadPlan {
  std::vector<H2DSeg> segs;
  std::vector<std::function<int()>> after;      // K1 launches that read the uploaded raw / validity bytes
  int run(cudaStream_t s) {
    if (h2d_execute(segs, s)) return 1;
    for (auto& f : after) if (f()) return 1;
    segs.clear(); after.clear();
    return 0;
  }
};

// Upload one column into dst[0..n) as T.  mode: 0 null->NaN, 1 null->fill, 2 null->0
template <typename T>
int upload_column(const pdsb_column& c, T* dst, int mode, double fill, DevBag& bag, UploadPlan& plan, cudaStream_t s) {
  int64_t off = 0;
  for (int i = 0; i < c.n_chunks; ++i) {
    const pdsb_chunk& ch = c.chunks[i];
    if (ch.length == 0) continue;
    const bool has_null = ch.validity && (c.null_count != 0) && chunk_nulls(ch) > 0;
    if (c.dtype == DT<T>::code && !has_null) {
      const T* src = reinterpret_cast<const T*>(ch.data) + ch.offset;
      plan.segs.push_back({dst + off, src, (size_t)ch.length * sizeof(T)});
    } else {
      size_t esz = dtype_size(c.dtype);
      const uint8_t* raw;
      size_t raw_bytes;
      int64_t bit_off = ch.offset & 7;
      if (c.dtype == PDSB_BOOL) {
        raw = reinterpret_cast<const uint8_t*>(ch.data) + (ch.offset >> 3);
        raw_bytes = (size_t)((bit_off + ch.length + 7) >> 3);
      } else {
        raw = reinterpret_cast<const uint8_t*>(ch.data) + (size_t)ch.offset * esz;
        raw_bytes = (size_t)ch.length * esz;
      }
      uint8_t* d_raw = bag.alloc<uint8_t>(raw_bytes + 16);
      if (!d_raw) return 1;
      plan.segs.push_back({d_raw, raw, raw_bytes});
      uint8_t* d_val = nullptr;
      if (has_null) {
        size_t vb = (size_t)((bit_off + ch.length + 7) >> 3);
        d_val = bag.alloc<uint8_t>(vb + 16);
        if (!d_val) return 1;
        plan.segs.push_back({d_val, ch.validity + (ch.offset >> 3), vb});
      }
      const int dt = c.dtype; const int64_t len = ch.length; T* out = dst + off;
      plan.after.push_back([=] { return pack_chunk<T>(d_raw, dt, d_val, bit_off, len, out, mode, fill, s); });
    }
    off += ch.length;
  }
  return 0;
}

// The per-row null mask of cols[0 .. n_cols): a new [ld] array, 1 where every one of the columns is valid and 0 where one
// is null.  The fill to 1 is launched now; the validity uploads and the launches that clear the null rows go into plan.
template <typename T>
T* row_mask(const pdsb_column* cols, int n_cols, int64_t n, int64_t ld, DevBag& bag, UploadPlan& plan, cudaStream_t s) {
  T* rowmask = bag.alloc<T>((size_t)ld);
  if (!rowmask || fill_value<T>(rowmask, n, T(1), s)) return nullptr;
  for (int c = 0; c < n_cols; ++c) {
    int64_t off = 0;
    for (int i = 0; i < cols[c].n_chunks; ++i) {
      const pdsb_chunk& ch = cols[c].chunks[i];
      if (ch.length && ch.validity && chunk_nulls(ch) > 0) {
        int64_t bit_off = ch.offset & 7;
        size_t vb = (size_t)((bit_off + ch.length + 7) >> 3);
        uint8_t* d_val = bag.alloc<uint8_t>(vb + 16);
        if (!d_val) return nullptr;
        plan.segs.push_back({d_val, ch.validity + (ch.offset >> 3), vb});
        const int64_t len = ch.length; T* rm = rowmask + off;
        plan.after.push_back([=] { return and_validity<T>(d_val, bit_off, len, rm, s); });
      }
      off += ch.length;
    }
  }
  return rowmask;
}

struct ResultOwner { std::vector<void*> pinned; };

void* result_buf(pdsb_host_result* r, size_t bytes) {
  if (!r->_owner) r->_owner = new ResultOwner();
  void* p = pinned_alloc(bytes ? bytes : 8);
  if (p) reinterpret_cast<ResultOwner*>(r->_owner)->pinned.push_back(p);
  return p;
}

// *dst = a result buffer of `bytes`, filled from the device array `src` on `s` (complete at the next synchronize)
template <typename U>
int result_copy(pdsb_host_result* r, U*& dst, const void* src, size_t bytes, cudaStream_t s) {
  void* p = result_buf(r, bytes);
  if (!p) return 1;
  dst = static_cast<U*>(p);
  PDSB_CUDA_OK(cudaMemcpyAsync(p, src, bytes, cudaMemcpyDeviceToHost, s));
  return 0;
}

// The reference's shape checks on [targets | features], in its order; returns the row count, or -1 with the error set.
int64_t checked_rows(const pdsb_column* cols, int n_cols, int n_targets) {
  if (n_cols < n_targets + 1) { set_error("Data is empty"); return -1; }
  const int64_t n = col_len(cols[0]);
  for (int c = 1; c < n_cols; ++c)
    if (col_len(cols[c]) != n) { set_error("Seires don't have the same length."); return -1; }
  if (n == 0) { set_error("Empty data"); return -1; }
  return n;
}

// apart from checked_rows: lin_reg checks the weights' length before the null policy, the reports after it
int check_weights(const pdsb_column& w, int64_t n) {
  if (col_len(w) != n) { set_error("Shape of weights is not the same as the data."); return 1; }
  return 0;
}

// pl_lr's dispatch (linear_regression.rs:436-498): OLS / ridge (gated), NNLS, and coordinate descent for lasso / elastic
// net / positive ridge; the f32 twin hard-codes the iteration counts (_f32.rs:343,351,362).
pdsb_solve_opts lr_solve_opts(const pdsb_lr_kwargs* kw, int p, int t, bool is_f32, int want_pred) {
  pdsb_solve_opts o{};
  o.p = p; o.t = t; o.add_bias = kw->bias ? 1 : 0; o.solver = solver_from_string(kw->solver);
  o.l1_reg = kw->l1_reg; o.l2_reg = kw->l2_reg; o.tol = kw->tol; o.singular_x_tol = kw->singular_x_tol;
  o.positive = kw->positive; o.max_iter = (int)kw->max_iter;
  const bool l1 = kw->l1_reg > 0.0, l2 = kw->l2_reg > 0.0;
  if (!l1 && !kw->positive) o.method = PDSB_METHOD_LSTSQ;
  else if (!l1 && !l2 && kw->positive) { o.method = PDSB_METHOD_NNLS; if (is_f32) o.max_iter = want_pred ? 2000 : 200; }
  else {
    o.method = PDSB_METHOD_CD;
    if (!l1) { o.l1_reg = 0.0; o.positive = 1; }
    if (is_f32) o.max_iter = 2000;
  }
  return o;
}

// ---------------------------------------------------------------------------------------------------
// Shared front end: null policy + upload of [targets | features] (+ weights) into the device frame.
// ---------------------------------------------------------------------------------------------------
template <typename T>
struct Frame {
  T* Z = nullptr;       // [ld x (t + p)] column-major: targets first, then features
  int64_t ld = 0, n = 0;
  int p = 0, t = 0;
  T* mask = nullptr;    // per-row validity (nullptr: every row valid)
  T* w = nullptr;
  bool any_null = false;
  const T* Y() const { return Z; }
  const T* X() const { return Z + (size_t)t * ld; }
};

// online = rolling/recursive: rows are never dropped, nulls become NaN (or the fill value) and the kernel masks them
template <typename T>
int build_frame(const pdsb_column* cols, int n_cols, int n_targets, const pdsb_column* wcol, const NullPolicy& pol,
                bool multi, bool online, Frame<T>& F, DevBag& bag, cudaStream_t s) {
  const int64_t n = checked_rows(cols, n_cols, n_targets);
  if (n < 0) return 1;
  F.n = n; F.t = n_targets; F.p = n_cols - n_targets; F.ld = pad_ld(n);
  bool y_null = false, x_null = false;
  for (int c = 0; c < n_targets; ++c) y_null |= col_nulls(cols[c]) > 0;
  for (int c = n_targets; c < n_cols; ++c) x_null |= col_nulls(cols[c]) > 0;
  F.any_null = y_null || x_null;
  std::vector<int> mode(n_cols, 0);
  int mask_cols = 0;                      // nulls of columns [0, mask_cols) drop the row
  double fill = pol.fill;
  if (F.any_null) {
    if (multi) {   // series_to_mat_for_multi_lr, linear_regression.rs:301-332
      if (pol.kind == NullKind::RAISE) { set_error("Nulls found in data"); return 1; }
      if (pol.kind != NullKind::FILL) { set_error("The null policy is not supported by multi-target linear regression."); return 1; }
      if (y_null) { set_error("Filling null doesn't work for multi-target lstsq when there are nulls in any of the targets."); return 1; }
      for (int c = n_targets; c < n_cols; ++c) mode[c] = 1;
    } else {
      switch (pol.kind) {
        case NullKind::RAISE: set_error("Nulls found in data"); return 1;
        case NullKind::IGNORE: case NullKind::SKIP_WINDOW: break;   // null -> NaN
        case NullKind::SKIP:
          if (online) break;                                        // rows kept as NaN, kernel skips them
          mask_cols = n_cols;
          for (int c = 0; c < n_cols; ++c) mode[c] = 2;
          break;
        case NullKind::FILL: case NullKind::FILL_WINDOW:
          for (int c = n_targets; c < n_cols; ++c) mode[c] = 1;
          if (y_null && !online && pol.kind == NullKind::FILL) { mask_cols = 1; mode[0] = 2; }
          break;
      }
    }
  }
  NvtxRange nv("pdsb:build_frame");
  UploadPlan plan;
  F.Z = bag.alloc<T>((size_t)F.ld * n_cols);
  if (!F.Z) return 1;
  for (int c = 0; c < n_cols; ++c)
    if (upload_column<T>(cols[c], F.Z + (size_t)c * F.ld, mode[c], fill, bag, plan, s)) return 1;
  if (mask_cols && !(F.mask = row_mask<T>(cols, mask_cols, n, F.ld, bag, plan, s))) return 1;
  if (wcol) {
    if (check_weights(*wcol, n)) return 1;
    F.w = bag.alloc<T>((size_t)F.ld);
    if (!F.w) return 1;
    if (upload_column<T>(*wcol, F.w, 0, 0.0, bag, plan, s)) return 1;
  }
  if (plan.run(s)) return 1;
  if (mask_cols)
    for (int c = 0; c < n_cols; ++c)
      if (zero_masked<T>(F.Z + (size_t)c * F.ld, F.mask, n, s)) return 1;
  return 0;
}

// ---- row slices of Arrow-style columns (zero-copy: chunk views with adjusted offset / length) ----
struct ColSlice {
  std::vector<pdsb_column> cols;
  std::vector<std::vector<pdsb_chunk>> chunks;
};
void slice_columns(const pdsb_column* cols, int n_cols, int64_t r0, int64_t r1, ColSlice& out) {
  out.cols.assign(cols, cols + n_cols);
  out.chunks.assign(n_cols, {});
  for (int c = 0; c < n_cols; ++c) {
    int64_t pos = 0;
    for (int k = 0; k < cols[c].n_chunks; ++k) {
      const pdsb_chunk& ch = cols[c].chunks[k];
      const int64_t lo = std::max(r0, pos), hi = std::min(r1, pos + ch.length);
      if (hi > lo) { pdsb_chunk v = ch; v.offset = ch.offset + (lo - pos); v.length = hi - lo; out.chunks[c].push_back(v); }
      pos += ch.length;
    }
    out.cols[c].n_chunks = (int)out.chunks[c].size();
    out.cols[c].chunks = out.chunks[c].data();
    if (out.cols[c].null_count != 0) out.cols[c].null_count = -1;      // recount inside the slice
  }
}

// One row shard of a lin_reg call: everything that lives on ONE device.
template <typename T>
struct LrShard {
  int64_t r0 = 0, r1 = 0;
  ColSlice data, w;
  cudaStream_t s = nullptr;
  std::unique_ptr<DevBag> bag;
  Frame<T> F;
  double* dM = nullptr; double* dbeta = nullptr; double* daux = nullptr; int* dstatus = nullptr;
  T* dpred = nullptr; T* dresid = nullptr; uint8_t* dvalid = nullptr;
  std::vector<double> hbeta, haux;
  int hstatus = 0;
  double hcount = 0.0;
  std::string err;
};

struct LrPlan {       // what every shard needs to know about the call
  NullPolicy pol; bool multi, weighted; int n_targets, want_pred, w_rcond;
  pdsb_solve_opts o; int p, t, q, q1;
};

// phase 1 (on the shard's device): null policy + upload + partial moments
template <typename T>
int shard_moments(LrShard<T>& S, const LrPlan& P) {
  NvtxRange nv("pdsb:shard_moments");
  if (thread_stream(&S.s)) return 1;
  S.bag.reset(new DevBag(S.s));
  const pdsb_column* wcol = P.weighted ? &S.w.cols[0] : nullptr;
  if (build_frame<T>(S.data.cols.data(), (int)S.data.cols.size(), P.n_targets, wcol, P.pol, P.multi, false, S.F, *S.bag, S.s)) return 1;
  S.dM = S.bag->template alloc<double>((size_t)P.q1 * P.q1);
  S.dbeta = S.bag->template alloc<double>((size_t)P.q * P.t);
  S.daux = S.bag->template alloc<double>((size_t)P.q * P.q + P.q);
  S.dstatus = S.bag->template alloc<int>(4);
  if (!S.dM || !S.dbeta || !S.daux || !S.dstatus) return 1;
  if (moments<T>(MomentsPrecision::TF32_ALLOWED, S.F.X(), S.F.ld, S.F.Y(), S.F.ld, S.F.w, S.F.mask, S.F.n, P.p, P.t, S.dM, S.s)) return 1;
  return 0;
}

// phase 2: [all-reduce of the moments] -> solve -> predict the shard -> D2H into the caller's buffers
template <typename T>
int shard_finish(LrShard<T>& S, const LrPlan& P, DeviceGroup* grp, int idx, bool world, T* hp, T* hr, uint8_t* hv,
                 int64_t n_total) {
  NvtxRange nv("pdsb:shard_finish");
  cudaStream_t s = S.s;
  const size_t mcount = (size_t)P.q1 * P.q1;
  if (grp && group_allreduce_f64(grp, idx, S.dM, mcount, s)) return 1;      // NVLink: k x (p+t+1)^2 f64
  if (world && world_allreduce_f64(S.dM, mcount, s)) return 1;
  if (solve_from_moments(S.dM, P.o, S.dbeta, S.dstatus, P.w_rcond ? S.daux : nullptr, s)) return 1;
  S.hbeta.resize((size_t)P.q * P.t); S.haux.resize(P.q);
  PDSB_CUDA_OK(cudaMemcpyAsync(S.hbeta.data(), S.dbeta, S.hbeta.size() * sizeof(double), cudaMemcpyDeviceToHost, s));
  PDSB_CUDA_OK(cudaMemcpyAsync(&S.hstatus, S.dstatus, sizeof(int), cudaMemcpyDeviceToHost, s));
  PDSB_CUDA_OK(cudaMemcpyAsync(&S.hcount, S.dM + mcount - 1, sizeof(double), cudaMemcpyDeviceToHost, s));
  if (P.w_rcond) PDSB_CUDA_OK(cudaMemcpyAsync(S.haux.data(), S.daux, P.q * sizeof(double), cudaMemcpyDeviceToHost, s));
  if (P.want_pred) {
    const Frame<T>& F = S.F;
    S.dpred = S.bag->template alloc<T>((size_t)F.ld * P.t);
    S.dresid = S.bag->template alloc<T>((size_t)F.ld * P.t);
    S.dvalid = S.bag->template alloc<uint8_t>((size_t)F.ld);
    if (!S.dpred || !S.dresid || !S.dvalid) return 1;
    if (predict_resid<T>(F.X(), F.ld, F.Y(), F.ld, nullptr, F.mask, F.n, P.p, P.t, P.o.add_bias, S.dbeta, S.dstatus, S.dpred,
                         S.dresid, F.ld, S.dvalid, nullptr, s)) return 1;
    for (int k = 0; k < P.t; ++k) {
      PDSB_CUDA_OK(cudaMemcpyAsync(hp + (size_t)k * n_total + S.r0, S.dpred + (size_t)k * F.ld, (size_t)F.n * sizeof(T), cudaMemcpyDeviceToHost, s));
      PDSB_CUDA_OK(cudaMemcpyAsync(hr + (size_t)k * n_total + S.r0, S.dresid + (size_t)k * F.ld, (size_t)F.n * sizeof(T), cudaMemcpyDeviceToHost, s));
    }
    if (hv) PDSB_CUDA_OK(cudaMemcpyAsync(hv + S.r0, S.dvalid, (size_t)F.n, cudaMemcpyDeviceToHost, s));
  }
  PDSB_CUDA_OK(cudaStreamSynchronize(s));
  return 0;
}

int64_t shard_min_rows() {
  static int64_t v = [] { const char* e = getenv("PDS_B200_SHARD_MIN_ROWS"); return e && atoll(e) > 0 ? atoll(e) : (int64_t)1 << 21; }();
  return v;
}

template <typename T>
int host_lin_reg_t(const pdsb_column* cols, int n_cols, const pdsb_lr_kwargs* kw, int n_targets, int want_pred,
                   int w_rcond, pdsb_host_result* out) {
  NvtxRange nv("pdsb:host_lin_reg");
  LrPlan P{};
  if (parse_null_policy(kw->null_policy, &P.pol)) return 1;
  P.multi = n_targets > 1;
  P.weighted = kw->weighted && !P.multi && !w_rcond;
  P.n_targets = n_targets; P.want_pred = want_pred; P.w_rcond = w_rcond;
  const pdsb_column* wcol = P.weighted ? &cols[0] : nullptr;
  const pdsb_column* data = P.weighted ? cols + 1 : cols;
  const int n_data = P.weighted ? n_cols - 1 : n_cols;
  const int64_t n = checked_rows(data, n_data, n_targets);
  if (n < 0 || (wcol && check_weights(*wcol, n))) return 1;
  const int p = n_data - n_targets, t = n_targets;
  const int q = p + (kw->bias ? 1 : 0);
  P.p = p; P.t = t; P.q = q; P.q1 = p + t + 1;

  const bool is_f32 = sizeof(T) == 4;
  const int world = world_enabled() ? world_size() : 1;
  // the rcond, weighted and multi-target fits replace the dispatch's method; LSTSQ and RCOND read none of the
  // iterative solvers' fields (l1_reg, positive, max_iter) it may have set
  pdsb_solve_opts& o = P.o;
  o = lr_solve_opts(kw, p, t, is_f32, want_pred);
  if (w_rcond) {
    o.method = PDSB_METHOD_RCOND;
    const double eps = is_f32 ? (double)FLT_EPSILON : DBL_EPSILON;
    double rc = is_f32 ? (double)(float)kw->tol : kw->tol;
    // with a world communicator n is this rank's share; the threshold only needs max(n_total, q) to the scale of eps
    o.tol = std::max(rc, eps * (double)std::max<int64_t>(n * world, q));
    o.singular_x_tol = 0.0;
  } else if (P.weighted) {
    o.method = PDSB_METHOD_LSTSQ; o.l2_reg = 0.0; o.singular_x_tol = 0.0;   // faer_weighted_lr: no ridge, no gate
  } else if (P.multi) {
    o.method = PDSB_METHOD_LSTSQ; o.l1_reg = 0.0;
  }

  // ---- shards: one per device of the active group when the call is big enough to pay for it ----
  DeviceGroup* grp = (n >= shard_min_rows()) ? active_group() : nullptr;
  if (grp && world > 1) { set_error("a device group (PDS_B200_DEVICES) and a world communicator cannot be combined"); return 1; }
  const int k = grp ? (int)grp->devices.size() : 1;
  std::vector<LrShard<T>> sh(k);
  for (int i = 0; i < k; ++i) {
    // contiguous row ranges, boundaries on multiples of 1024 rows (whole stages of the Gram kernel)
    auto cut = [&](int j) { return j >= k ? n : std::min<int64_t>(n, ((n * j / k) + 1023) / 1024 * 1024); };
    sh[i].r0 = cut(i); sh[i].r1 = cut(i + 1);
    if (k == 1) {
      sh[i].data.cols.assign(data, data + n_data);
      if (wcol) sh[i].w.cols.assign(wcol, wcol + 1);
    } else {
      slice_columns(data, n_data, sh[i].r0, sh[i].r1, sh[i].data);
      if (wcol) slice_columns(wcol, 1, sh[i].r0, sh[i].r1, sh[i].w);
    }
  }
  auto run_all = [&](const std::function<int(int)>& fn) -> int {
    if (k == 1) { int rc = fn(0); if (rc) sh[0].err = get_error(); return rc; }
    std::vector<std::future<int>> fu;
    for (int i = 0; i < k; ++i)
      fu.push_back(grp->workers[i]->submit([&, i] { int rc = fn(i); if (rc) sh[i].err = get_error(); return rc; }));
    int rc = 0;
    for (auto& f : fu) rc |= f.get();
    return rc;
  };
  auto first_error = [&] { for (auto& S : sh) if (!S.err.empty()) { set_error("%s", S.err.c_str()); return; } };
  // device scratch is released on the thread (device) that made it
  struct Cleanup { std::function<void()> f; ~Cleanup() { f(); } } cleanup{[&] { run_all([&](int i) { sh[i].bag.reset(); return 0; }); }};

  if (run_all([&](int i) { return sh[i].r1 > sh[i].r0 || k == 1 ? shard_moments<T>(sh[i], P) : (set_error("empty shard"), 1); })) { first_error(); return 1; }
  bool any_mask = false;
  for (auto& S : sh) any_mask |= S.F.mask != nullptr;
  if (!P.multi && !any_mask && world == 1 && n < q) { set_error("#Data < #features. No conclusive result."); return 1; }

  T* hp = nullptr; T* hr = nullptr; uint8_t* hv = nullptr;
  if (want_pred) {
    hp = reinterpret_cast<T*>(result_buf(out, (size_t)n * t * sizeof(T)));
    hr = reinterpret_cast<T*>(result_buf(out, (size_t)n * t * sizeof(T)));
    if (any_mask) hv = reinterpret_cast<uint8_t*>(result_buf(out, (size_t)n));
    if (!hp || !hr || (any_mask && !hv)) return 1;
  }
  if (run_all([&](int i) { return shard_finish<T>(sh[i], P, grp, i, world > 1, hp, hr, hv, n); })) { first_error(); return 1; }

  const LrShard<T>& S0 = sh[0];
  if (any_mask || world > 1) {
    const int64_t n_valid = (int64_t)llround(S0.hcount);        // the reduced moments hold the global row count
    if (!P.multi && n_valid < q) { set_error("#Data < #features. No conclusive result."); return 1; }
    if (P.weighted && world == 1 && n_valid != n) { set_error("Shape of weights is not the same as the data."); return 1; }
  }
  out->is_f32 = is_f32; out->n_coef = q; out->n_targets = t; out->gated = S0.hstatus != 0; out->n_rows = want_pred ? n : 0;
  if (!want_pred) {
    T* c = reinterpret_cast<T*>(result_buf(out, (size_t)q * t * sizeof(T)));
    if (!c) return 1;
    for (size_t i = 0; i < (size_t)q * t; ++i) c[i] = (T)S0.hbeta[i];
    out->coeffs = c;
    if (w_rcond) {
      T* sv = reinterpret_cast<T*>(result_buf(out, (size_t)q * sizeof(T)));
      if (!sv) return 1;
      for (int i = 0; i < q; ++i) sv[i] = (T)S0.haux[i];
      out->singular_values = sv;
    }
    return 0;
  }
  out->pred = hp; out->resid = hr; out->valid = hv;
  return 0;
}

template <typename T>
int host_report_t(const pdsb_column* cols, int n_cols, const pdsb_lr_kwargs* kw, int weighted, pdsb_host_result* out) {
  cudaStream_t s;
  if (thread_stream(&s)) return 1;
  NullPolicy pol;
  if (parse_null_policy(kw->null_policy, &pol)) return 1;
  const int skip = weighted ? 2 : 1;       // [w] var y x...
  if (n_cols < skip + 2) { set_error("Data is empty"); return 1; }
  const pdsb_column& vc = cols[skip - 1];
  double y_var = NAN;
  if (col_len(vc) > 0 && vc.n_chunks > 0) {
    const pdsb_chunk& ch = vc.chunks[0];
    bool valid = !ch.validity || ((ch.validity[ch.offset >> 3] >> (ch.offset & 7)) & 1);
    if (valid && ch.length > 0) {
      if (vc.dtype == PDSB_F64) y_var = reinterpret_cast<const double*>(ch.data)[ch.offset];
      else if (vc.dtype == PDSB_F32) y_var = reinterpret_cast<const float*>(ch.data)[ch.offset];
    }
  }
  DevBag bag(s);
  Frame<T> F;
  if (build_frame<T>(cols + skip, n_cols - skip, 1, weighted ? &cols[0] : nullptr, pol, false, false, F, bag, s)) return 1;
  const int add_bias = kw->bias ? 1 : 0;
  const int q = F.p + add_bias;
  if (!F.mask && F.n < q) { set_error("#Data < #features. No conclusive result."); return 1; }
  double* dout = bag.alloc<double>((size_t)8 * q);
  if (!dout) return 1;
  const int se = weighted ? 0 : se_type_from_string(kw->std_err);
  if (report_stats<T>(F.X(), F.ld, F.Y(), F.w, F.mask, F.n, F.p, add_bias, se, y_var, dout, s)) return 1;
  out->is_f32 = sizeof(T) == 4; out->n_coef = q; out->n_targets = 1;
  if (result_copy(out, out->report, dout, (size_t)8 * q * sizeof(double), s)) return 1;
  PDSB_CUDA_OK(cudaStreamSynchronize(s));
  return 0;
}

template <typename T>
int host_online_t(const pdsb_column* cols, int n_cols, const pdsb_lr_kwargs* kw, int rolling, pdsb_host_result* out) {
  cudaStream_t s;
  if (thread_stream(&s)) return 1;
  NullPolicy pol;
  if (parse_null_policy(kw->null_policy, &pol)) return 1;
  if (rolling) {   // linear_regression.rs:1214-1219
    if (pol.kind == NullKind::SKIP) pol.kind = NullKind::SKIP_WINDOW;
    else if (pol.kind == NullKind::FILL) pol.kind = NullKind::FILL_WINDOW;
  }
  DevBag bag(s);
  Frame<T> F;
  if (build_frame<T>(cols, n_cols, 1, nullptr, pol, false, true, F, bag, s)) return 1;
  const int add_bias = kw->bias ? 1 : 0;
  const int q = F.p + add_bias;
  if (F.n < q) { set_error("#Data < #features. No conclusive result."); return 1; }
  if (kw->n < 1) { set_error("window / start_with must be >= 1"); return 1; }
  if (kw->n > F.n) { set_error("#Data < window size. No conclusive result."); return 1; }
  bool y_null = col_nulls(cols[0]) > 0;
  int skip = 0;
  if (F.any_null) {
    if (rolling) skip = (pol.kind == NullKind::SKIP_WINDOW) || (pol.kind == NullKind::FILL_WINDOW && y_null);
    else skip = (pol.kind == NullKind::SKIP) || (pol.kind == NullKind::FILL && y_null);
  }
  T* dco = bag.alloc<T>((size_t)F.n * q);
  T* dpr = bag.alloc<T>((size_t)F.n);
  uint8_t* dva = bag.alloc<uint8_t>((size_t)F.n);
  if (!dco || !dpr || !dva) return 1;
  const int64_t window = rolling ? kw->n : 0;
  const int64_t min_rows = rolling ? kw->min_size : kw->n;
  if (online_lin_reg<T>(F.X(), F.ld, F.Y(), F.n, F.p, add_bias, window, min_rows, skip, kw->lambda, nullptr, 0, dco, dpr, dva, s)) return 1;
  out->is_f32 = sizeof(T) == 4; out->n_coef = q; out->n_targets = 1; out->n_rows = F.n;
  if (result_copy(out, out->coeffs, dco, (size_t)F.n * q * sizeof(T), s) ||
      result_copy(out, out->pred, dpr, (size_t)F.n * sizeof(T), s) ||
      result_copy(out, out->valid, dva, (size_t)F.n, s)) return 1;
  PDSB_CUDA_OK(cudaStreamSynchronize(s));
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
};

// The offsets are user data (an Int64 column): every group must be a row range inside the frame of n rows, or the
// kernels would read outside X / y.  pl_lr_by, pl_lr_pred_by and the grouped logistic_reg share these checks.
int check_group_offsets(const int64_t* offsets, int64_t n_groups, int64_t n) {
  if (n_groups < 1 || offsets[0] != 0 || offsets[n_groups] != n) { set_error("grouped lin_reg: bad group offsets"); return 1; }
  for (int64_t g = 0; g < n_groups; ++g)
    if (offsets[g] < 0 || offsets[g] > offsets[g + 1] || offsets[g + 1] > n) {
      set_error("grouped lin_reg: group offsets must be non-decreasing and within [0, n] (group %lld)", (long long)g);
      return 1;
    }
  return 0;
}

template <typename T>
int grouped_fit(const pdsb_column* cols, int n_cols, const int64_t* offsets, int64_t n_groups, const pdsb_lr_kwargs* kw,
                const NullPolicy& pol, int want_pred, GroupedFit<T>& G, DevBag& bag, cudaStream_t s) {
  Frame<T>& F = G.F;
  // nulls: only "skip" maps onto the batched kernel (row -> NaN -> dropped inside its group)
  for (int c = 0; c < n_cols; ++c)
    if (col_nulls(cols[c]) > 0 && pol.kind != NullKind::SKIP) {
      if (pol.kind == NullKind::RAISE) set_error("Nulls found in data");
      else set_error("grouped lin_reg: only null_policy='skip' is supported with nulls");
      return 1;
    }
  NullPolicy nanpol{NullKind::IGNORE, 0.0};
  if (build_frame<T>(cols, n_cols, 1, nullptr, nanpol, false, true, F, bag, s)) return 1;
  if (check_group_offsets(offsets, n_groups, F.n)) return 1;
  if (kw->weighted) { set_error("grouped lin_reg: weighted fits are not batched"); return 1; }
  const pdsb_solve_opts o = lr_solve_opts(kw, F.p, 1, sizeof(T) == 4, want_pred);     // pl_lr(_pred) per group, batched
  G.q = F.p + o.add_bias; G.add_bias = o.add_bias;
  G.doff = bag.alloc<int64_t>((size_t)n_groups + 1);
  G.dbeta = bag.alloc<double>((size_t)n_groups * G.q);
  G.dst = bag.alloc<int>((size_t)n_groups);
  if (!G.doff || !G.dbeta || !G.dst) return 1;
  PDSB_CUDA_OK(cudaMemcpyAsync(G.doff, offsets, (size_t)(n_groups + 1) * sizeof(int64_t), cudaMemcpyHostToDevice, s));
  return grouped_lin_reg<T>(F.X(), F.ld, F.Y(), G.doff, n_groups, F.n, F.p, o, G.dbeta, G.dst, s);
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
  const int q = G.q;
  std::vector<double> hb((size_t)n_groups * q);
  std::vector<int> hs((size_t)n_groups);
  PDSB_CUDA_OK(cudaMemcpyAsync(hb.data(), G.dbeta, hb.size() * sizeof(double), cudaMemcpyDeviceToHost, s));
  PDSB_CUDA_OK(cudaMemcpyAsync(hs.data(), G.dst, hs.size() * sizeof(int), cudaMemcpyDeviceToHost, s));
  PDSB_CUDA_OK(cudaStreamSynchronize(s));
  out->is_f32 = sizeof(T) == 4; out->n_coef = q; out->n_targets = 1; out->n_rows = n_groups;
  T* c = reinterpret_cast<T*>(result_buf(out, (size_t)n_groups * q * sizeof(T)));
  uint8_t* v = reinterpret_cast<uint8_t*>(result_buf(out, (size_t)n_groups));
  if (!c || !v) return 1;
  for (size_t i = 0; i < hb.size(); ++i) c[i] = (T)hb[i];
  for (int64_t g = 0; g < n_groups; ++g) v[g] = hs[g] == 0;
  out->coeffs = c; out->valid = v;
  return 0;
}

// pl_lr_pred_by: the fit of pl_lr_by with pl_lr_pred's solver settings, then K5's predict pass on the same stream.  The
// fit sees null rows as NaN, as pl_lr_by's does; the predict pass tells them apart from genuine NaN values by a row mask built from the
// Arrow validity, as build_frame does for pl_lr_pred.  pred / resid come back in one copy each; the validity bytes are
// copied only when some row is null or some group's fit is.
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
  T* dpred = bag.alloc<T>((size_t)n);
  T* dresid = bag.alloc<T>((size_t)n);
  uint8_t* dvalid = bag.alloc<uint8_t>((size_t)n);
  if (!dpred || !dresid || !dvalid) return 1;
  if (grouped_predict<T>(F.X(), F.ld, F.Y(), G.doff, n_groups, n, F.p, G.add_bias, G.dbeta, G.dst, mask, dpred, dresid,
                         dvalid, s)) return 1;
  std::vector<int> hs((size_t)n_groups);
  if (result_copy(out, out->pred, dpred, (size_t)n * sizeof(T), s) ||
      result_copy(out, out->resid, dresid, (size_t)n * sizeof(T), s)) return 1;
  PDSB_CUDA_OK(cudaMemcpyAsync(hs.data(), G.dst, hs.size() * sizeof(int), cudaMemcpyDeviceToHost, s));
  PDSB_CUDA_OK(cudaStreamSynchronize(s));
  bool all_ok = !mask;
  for (int64_t g = 0; g < n_groups && all_ok; ++g) all_ok = hs[g] == PDSB_OK;
  if (!all_ok) {
    if (result_copy(out, out->valid, dvalid, (size_t)n, s)) return 1;
    PDSB_CUDA_OK(cudaStreamSynchronize(s));
  }
  out->is_f32 = sizeof(T) == 4; out->n_coef = G.q; out->n_targets = 1; out->n_rows = n;
  return 0;
}


// ---------------------------------------------------------------------------------------------------
// pl_logistic_coeffs / pl_logistic_pred (/root/reference/src/num_ext/logistic_regression.rs:10-99): f64 only.
// The reference minimises mean log-loss (+ l2/2 |w|^2, + l1 |w|_1 via OWL-QN) with L-BFGS from a seeded random start
// (logistic_solver.rs:107-146); the cost is convex, so Newton / IRLS on the device reaches the same minimiser:
// per iteration one row pass (K11: weights + working response + loss), the weighted moments (K2a) and the ridge solve
// (K3; coordinate descent on the weighted Gram when l1 > 0 = proximal Newton).  Stops like the reference when the
// gradient norm falls below max(sqrt(eps), tol); step halving whenever the cost does not decrease.
int host_logistic(const pdsb_column* cols, int n_cols, const pdsb_lr_kwargs* kw, int want_pred, pdsb_host_result* out) {
  NvtxRange nv("pdsb:host_logistic");
  typedef double T;
  cudaStream_t s;
  if (thread_stream(&s)) return 1;
  NullPolicy pol;
  if (parse_null_policy(kw->null_policy, &pol)) return 1;
  DevBag bag(s);
  Frame<T> F;
  if (build_frame<T>(cols, n_cols, 1, nullptr, pol, false, false, F, bag, s)) return 1;
  const int p = F.p, add_bias = kw->bias ? 1 : 0, q = p + add_bias, q1 = p + 2;
  const int64_t n = F.n;
  if (p > 64) { set_error("logistic_reg: more than 64 features are not supported"); return 1; }
  double m = (double)n;                       // rows that take part
  double* dM = bag.alloc<double>((size_t)q1 * q1);
  double* dbeta = bag.alloc<double>((size_t)q);
  int* dstatus = bag.alloc<int>(4);
  T* dw = bag.alloc<T>((size_t)F.ld);
  T* dz = bag.alloc<T>((size_t)F.ld);
  double* dparts = bag.alloc<double>((size_t)irls_max_parts() + 1);
  if (!dM || !dbeta || !dstatus || !dw || !dz || !dparts) return 1;
  if (F.mask) {
    if (count_mask<T>(F.mask, n, dparts, s)) return 1;
    PDSB_CUDA_OK(cudaMemcpyAsync(&m, dparts, sizeof(double), cudaMemcpyDeviceToHost, s));
    PDSB_CUDA_OK(cudaStreamSynchronize(s));
  }
  if (m < 1.0) { set_error("Empty data"); return 1; }
  const double l1 = kw->l1_reg > 0.0 ? std::max(kw->l1_reg, DBL_EPSILON) : 0.0;      // logistic_solver.rs:131-133
  const double l2 = kw->l2_reg > 0.0 ? kw->l2_reg : 0.0;
  const double gtol = std::max(std::sqrt(DBL_EPSILON), kw->tol);                      // :127
  const int64_t max_iter = kw->max_iter > 0 ? kw->max_iter : 200;
  std::vector<double> hb(q, 0.0), hb_prev(q, 0.0), hM((size_t)q1 * q1), hparts((size_t)irls_max_parts());
  PDSB_CUDA_OK(cudaMemsetAsync(dbeta, 0, sizeof(double) * q, s));
  pdsb_solve_opts o{};
  o.p = p; o.t = 1; o.add_bias = add_bias; o.solver = PDSB_SOLVER_QR; o.singular_x_tol = 0.0; o.max_iter = 2000; o.tol = 1e-12;
  double cost_prev = INFINITY;
  int halvings = 0;
  bool failed = false;
  for (int64_t it = 0; it < max_iter; ++it) {
    int nparts = 0;
    if (irls_rows(PDSB_IRLS_LOGISTIC, F.X(), F.ld, F.Y(), F.mask, n, p, add_bias, dbeta, nullptr, dw, dz, dparts,
                  &nparts, s)) return 1;
    if (moments<T>(MomentsPrecision::F64_ACCUM, F.X(), F.ld, dz, F.ld, dw, F.mask, n, p, 1, dM, s)) return 1;
    PDSB_CUDA_OK(cudaMemcpyAsync(hM.data(), dM, hM.size() * sizeof(double), cudaMemcpyDeviceToHost, s));
    PDSB_CUDA_OK(cudaMemcpyAsync(hparts.data(), dparts, (size_t)nparts * sizeof(double), cudaMemcpyDeviceToHost, s));
    PDSB_CUDA_OK(cudaStreamSynchronize(s));
    double loss = 0.0;
    for (int i = 0; i < nparts; ++i) loss += hparts[i];
    double pen = 0.0, l1n = 0.0;
    for (int j = 0; j < p; ++j) { pen += hb[j] * hb[j]; l1n += std::fabs(hb[j]); }
    const double cost = loss / m + 0.5 * l2 * pen + l1 * l1n;
    if (!std::isfinite(cost)) { failed = true; break; }
    if (it > 0 && cost > cost_prev + 1e-14 * std::fabs(cost_prev) && halvings < 40) {
      // the full Newton step overshot: halve it and evaluate again (the reference's line search plays this role)
      for (int j = 0; j < q; ++j) hb[j] = 0.5 * (hb[j] + hb_prev[j]);
      PDSB_CUDA_OK(cudaMemcpyAsync(dbeta, hb.data(), sizeof(double) * q, cudaMemcpyHostToDevice, s));
      PDSB_CUDA_OK(cudaStreamSynchronize(s));
      ++halvings;
      continue;
    }
    halvings = 0;
    // gradient of the smooth part from the weighted moments [X | z | 1]: X'(mu - y) = (X'WX) w - X'Wz
    auto col = [&](int j) { return j < p ? j : p + 1; };          // coefficient j -> moments index (bias = the ones column)
    double g2 = 0.0;
    const double sum_w = hM[(size_t)(p + 1) * q1 + (p + 1)];
    for (int j = 0; j < q; ++j) {
      double gj = -hM[(size_t)col(j) * q1 + p];
      for (int k = 0; k < q; ++k) gj += hM[(size_t)col(j) * q1 + col(k)] * hb[k];
      gj = gj / m + (j < p ? l2 * hb[j] : 0.0);
      if (l1 > 0.0 && j < p) {       // minimum-norm subgradient of the l1 term
        if (hb[j] > 0.0) gj += l1; else if (hb[j] < 0.0) gj -= l1;
        else gj = std::fabs(gj) <= l1 ? 0.0 : (gj > 0.0 ? gj - l1 : gj + l1);
      }
      g2 += gj * gj;
    }
    cost_prev = cost; hb_prev = hb;
    if (std::sqrt(g2) < gtol) break;
    if (!(sum_w > 0.0)) { failed = true; break; }
    if (l1 > 0.0) { o.method = PDSB_METHOD_CD; o.l1_reg = l1 * m / sum_w; o.l2_reg = l2 * m / sum_w; }   // K3 scales by the count entry = sum w
    else { o.method = PDSB_METHOD_LSTSQ; o.l1_reg = 0.0; o.l2_reg = l2 * m; }
    if (solve_from_moments(dM, o, dbeta, dstatus, nullptr, s)) return 1;
    PDSB_CUDA_OK(cudaMemcpyAsync(hb.data(), dbeta, sizeof(double) * q, cudaMemcpyDeviceToHost, s));
    PDSB_CUDA_OK(cudaStreamSynchronize(s));
    bool fin = true;
    for (int j = 0; j < q; ++j) fin &= std::isfinite(hb[j]);
    if (!fin) { failed = true; break; }
  }
  if (failed) for (int j = 0; j < q; ++j) hb_prev[j] = NAN;        // Mat::full(nrows, 1, NaN), logistic_solver.rs:141-144
  const std::vector<double>& best = hb_prev;                      // the last accepted iterate (argmin's best_param)
  out->is_f32 = 0; out->n_coef = q; out->n_targets = 1;
  if (!want_pred) {
    double* c = reinterpret_cast<double*>(result_buf(out, (size_t)q * sizeof(double)));
    if (!c) return 1;
    for (int j = 0; j < q; ++j) c[j] = best[j];
    out->coeffs = c;
    return 0;
  }
  PDSB_CUDA_OK(cudaMemcpyAsync(dbeta, best.data(), sizeof(double) * q, cudaMemcpyHostToDevice, s));
  if (predict_strided(F.X(), 1, F.ld, n, p, dbeta, add_bias, dz, s, PDSB_GLM_BINOMIAL)) return 1;
  if (result_copy(out, out->pred, dz, (size_t)n * sizeof(double), s)) return 1;
  uint8_t* hv = nullptr;
  std::vector<double> hmask;
  if (F.mask) {
    hv = reinterpret_cast<uint8_t*>(result_buf(out, (size_t)n));
    if (!hv) return 1;
    hmask.resize((size_t)n);
    PDSB_CUDA_OK(cudaMemcpyAsync(hmask.data(), F.mask, (size_t)n * sizeof(double), cudaMemcpyDeviceToHost, s));
  }
  PDSB_CUDA_OK(cudaStreamSynchronize(s));
  if (hv) for (int64_t i = 0; i < n; ++i) hv[i] = hmask[(size_t)i] != 0.0 ? 1 : 0;
  out->n_rows = n; out->valid = hv;
  return 0;
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
  if (build_frame<T>(cols, n_cols, 1, nullptr, pol, false, false, F, bag, s)) return 1;
  if (check_group_offsets(offsets, n_groups, F.n)) return 1;
  const int p = F.p, add_bias = kw->bias ? 1 : 0, q = p + add_bias;
  const int64_t n = F.n;
  if (p > 64) { set_error("logistic_reg: more than 64 features are not supported"); return 1; }
  int64_t* doff = bag.alloc<int64_t>((size_t)n_groups + 1);
  double* dbeta = bag.alloc<double>((size_t)n_groups * q);
  int* dst = bag.alloc<int>((size_t)n_groups);
  if (!doff || !dbeta || !dst) return 1;
  PDSB_CUDA_OK(cudaMemcpyAsync(doff, offsets, (size_t)(n_groups + 1) * sizeof(int64_t), cudaMemcpyHostToDevice, s));
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
  std::vector<int> hs((size_t)n_groups);
  PDSB_CUDA_OK(cudaMemcpyAsync(hs.data(), dst, hs.size() * sizeof(int), cudaMemcpyDeviceToHost, s));
  PDSB_CUDA_OK(cudaStreamSynchronize(s));
  for (int64_t g = 0; g < n_groups; ++g)
    if (hs[g] == PDSB_LOGISTIC_EMPTY) { set_error("Empty data"); return 1; }
  return 0;
}

// pl_singular_values / pl_pca / pl_principal_components (src/num_ext/pca.rs:39-182).  f32 columns stay f32 on the device
// (pdsb_dev_pca_f32 forms the products in f64); any other dtype is cast to f64 by K1, as the reference's to_f64_vec_* do.
template <typename T>
int host_pca_t(const pdsb_column* cols, int n_cols, int mode, int k, pdsb_host_result* out) {
  NvtxRange nv("pdsb:host_pca");
  cudaStream_t s;
  if (thread_stream(&s)) return 1;
  const int p = n_cols;
  const int64_t n = col_len(cols[0]);
  for (int c = 1; c < n_cols; ++c)
    if (col_len(cols[c]) != n) { set_error("Seires don't have the same length."); return 1; }
  if (p > 259) { set_error("pca: %d features; at most 259 are supported", p); return 1; }
  out->is_f32 = 0; out->n_coef = p;
  if (mode == 2) {
    for (int c = 0; c < n_cols; ++c)
      if (col_nulls(cols[c]) > 0) { set_error("Nulls are found in data and this method doesn't allow nulls."); return 1; }
    out->n_targets = k; out->n_rows = n;
    if (n < k) {                                                   // pca.rs:90-93
      double* pr = reinterpret_cast<double*>(result_buf(out, (size_t)k * n * sizeof(double)));
      if (!pr) return 1;
      for (int64_t i = 0; i < (int64_t)k * n; ++i) pr[i] = NAN;
      out->pred = pr;
      return 0;
    }
    if (n < p) { set_error("principal_components: %lld rows < %d features is not supported (k <= rows < features)", (long long)n, p); return 1; }
  } else if (n == 0) {                                            // no rows: dim = 0
    if (mode == 1 && p > 0) { set_error("pca: 0 rows < %d features is not supported", p); return 1; }
    out->n_rows = 0;
    out->singular_values = result_buf(out, 0);
    return out->singular_values ? 0 : 1;
  }
  DevBag bag(s);
  Frame<T> F;
  NullPolicy pol{mode == 2 ? NullKind::RAISE : NullKind::SKIP, 0.0};
  if (build_frame<T>(cols, n_cols, 0, nullptr, pol, false, false, F, bag, s)) return 1;
  double* dsig = bag.alloc<double>((size_t)p);
  double* dV = bag.alloc<double>((size_t)p * p);
  int* dst = bag.alloc<int>(2);
  if (!dsig || !dV || !dst) return 1;
  int rc;
  if constexpr (sizeof(T) == 4) rc = pdsb_dev_pca_f32(F.X(), F.ld, F.mask, n, p, dsig, dV, dst, s);
  else rc = pdsb_dev_pca_f64(F.X(), F.ld, F.mask, n, p, dsig, dV, dst, s);
  if (rc) return 1;
  int hst[2];
  PDSB_CUDA_OK(cudaMemcpyAsync(hst, dst, sizeof(hst), cudaMemcpyDeviceToHost, s));
  PDSB_CUDA_OK(cudaStreamSynchronize(s));
  if (hst[0] != PDSB_PCA_OK) { set_error("SVD algorithm did not converge."); return 1; }
  const int dim = hst[1];
  if (mode == 1 && dim < p) { set_error("pca: %d rows < %d features is not supported", dim, p); return 1; }
  if (mode != 2) {
    out->n_rows = dim;
    if (result_copy(out, out->singular_values, dsig, (size_t)dim * sizeof(double), s)) return 1;
    if (mode == 1 && result_copy(out, out->coeffs, dV, (size_t)dim * p * sizeof(double), s)) return 1;
    PDSB_CUDA_OK(cudaStreamSynchronize(s));
    return 0;
  }
  double* dout = bag.alloc<double>((size_t)k * n);
  if (!dout) return 1;
  if constexpr (sizeof(T) == 4) rc = pdsb_dev_project_f32(F.X(), F.ld, n, p, dV, k, dout, n, s);
  else rc = pdsb_dev_project_f64(F.X(), F.ld, n, p, dV, k, dout, n, s);
  if (rc) return 1;
  if (result_copy(out, out->pred, dout, (size_t)k * n * sizeof(double), s)) return 1;
  PDSB_CUDA_OK(cudaStreamSynchronize(s));
  return 0;
}

// pl_smooth_spline (src/num_ext/splines.rs:99-119): x and y as the wrapper casts them (Float64); chunked and sliced
// columns are uploaded chunk by chunk, so nothing relies on the wrapper's rechunk.
int host_smooth_spline(const pdsb_column* cols, int n_cols, double lambda, pdsb_host_result* out) {
  NvtxRange nv("pdsb:host_smooth_spline");
  if (n_cols != 2) { set_error("smooth_spline: expected 2 inputs (x, y), got %d", n_cols); return 1; }
  for (int c = 0; c < 2; ++c)
    if (cols[c].dtype != PDSB_F64) { set_error("invalid series dtype: expected `Float64` for input %d", c); return 1; }
  if (col_nulls(cols[0]) > 0 || col_nulls(cols[1]) > 0) { set_error("Input x or y has nulls."); return 1; }
  const int64_t n = col_len(cols[0]);
  if (col_len(cols[1]) != n) { set_error("Input lengths are not the same."); return 1; }
  if (n < 3) { set_error("Must have >= 3 points."); return 1; }
  if (!(lambda >= 0.0)) { set_error("Input `lambda_` must be nonnegative."); return 1; }
  cudaStream_t s;
  if (thread_stream(&s)) return 1;
  DevBag bag(s);
  double* dx = bag.alloc<double>((size_t)n);
  double* dy = bag.alloc<double>((size_t)n);
  double* dg = bag.alloc<double>((size_t)n);
  int* dst = bag.alloc<int>(1);
  if (!dx || !dy || !dg || !dst) return 1;
  UploadPlan plan;
  if (upload_column<double>(cols[0], dx, 0, 0.0, bag, plan, s) || upload_column<double>(cols[1], dy, 0, 0.0, bag, plan, s) ||
      plan.run(s))
    return 1;
  if (pdsb_dev_smooth_spline_f64(dx, dy, n, lambda, dg, dst, s)) return 1;
  out->is_f32 = 0; out->n_rows = n; out->n_targets = 1;
  if (result_copy(out, out->pred, dg, (size_t)n * sizeof(double), s)) return 1;
  int st = 0;
  PDSB_CUDA_OK(cudaMemcpyAsync(&st, dst, sizeof(int), cudaMemcpyDeviceToHost, s));
  PDSB_CUDA_OK(cudaStreamSynchronize(s));
  if (st & PDSB_SPLINE_NOT_INCREASING) { set_error("Input is not increasing."); return 1; }
  return 0;
}

// pl_isotonic_regression (src/num_ext/isotonic_regression.rs): y (and w) as the wrapper casts them (Float64); chunked and
// sliced columns are uploaded chunk by chunk.  n <= 1 is answered here, validity included.
int host_isotonic_regression(const pdsb_column* cols, int n_cols, int has_weights, int increasing,
                             pdsb_host_result* out) {
  NvtxRange nv("pdsb:host_isotonic_regression");
  if (n_cols < (has_weights ? 2 : 1)) {
    set_error("isotonic_regression: expected %d inputs, got %d", has_weights ? 2 : 1, n_cols); return 1;
  }
  if (cols[0].dtype != PDSB_F64) { set_error("invalid series dtype: expected `Float64` for input 0"); return 1; }
  const int64_t n = col_len(cols[0]);
  out->is_f32 = 0; out->n_rows = n; out->n_targets = 1;
  if (n <= 1) {                                   // y as it is, a lone null included
    double* v = static_cast<double*>(result_buf(out, sizeof(double)));
    if (!v) return 1;
    *v = 0.0;
    if (n == 1) {
      const pdsb_chunk* ch = nullptr;
      for (int i = 0; i < cols[0].n_chunks && !ch; ++i) if (cols[0].chunks[i].length) ch = &cols[0].chunks[i];
      const bool valid = !ch->validity || ((ch->validity[ch->offset >> 3] >> (ch->offset & 7)) & 1);
      if (valid) *v = static_cast<const double*>(ch->data)[ch->offset];
      uint8_t* vb = static_cast<uint8_t*>(result_buf(out, 1));
      if (!vb) return 1;
      *vb = valid ? 1 : 0;
      out->valid = vb;
    }
    out->pred = v;
    return 0;
  }
  if (col_nulls(cols[0]) > 0) { set_error("Input should not contain nulls."); return 1; }
  if (has_weights) {
    if (cols[1].dtype != PDSB_F64) { set_error("invalid series dtype: expected `Float64` for input 1"); return 1; }
    if (col_len(cols[1]) != n) { set_error("Weights should not contain nulls and must be the same length as y."); return 1; }
    if (col_nulls(cols[1]) > 0) { set_error("Weight should not contain nulls."); return 1; }
  }
  cudaStream_t s;
  if (thread_stream(&s)) return 1;
  DevBag bag(s);
  double* dy = bag.alloc<double>((size_t)n);
  double* dw = has_weights ? bag.alloc<double>((size_t)n) : nullptr;
  double* dout = bag.alloc<double>((size_t)n);
  int* dst = bag.alloc<int>(1);
  if (!dy || (has_weights && !dw) || !dout || !dst) return 1;
  UploadPlan plan;
  if (upload_column<double>(cols[0], dy, 0, 0.0, bag, plan, s) ||
      (has_weights && upload_column<double>(cols[1], dw, 0, 0.0, bag, plan, s)) || plan.run(s))
    return 1;
  if (pdsb_dev_isotonic_f64(dy, dw, n, increasing, dout, dst, s)) return 1;
  if (result_copy(out, out->pred, dout, (size_t)n * sizeof(double), s)) return 1;
  int st = 0;
  PDSB_CUDA_OK(cudaMemcpyAsync(&st, dst, sizeof(int), cudaMemcpyDeviceToHost, s));
  PDSB_CUDA_OK(cudaStreamSynchronize(s));
  if (st & PDSB_ISO_NONPOSITIVE_WEIGHT) { set_error("Weight should not contain negative values."); return 1; }
  return 0;
}

}  // namespace
}  // namespace pdsb

using namespace pdsb;

extern "C" {

void pdsb_host_result_free(pdsb_host_result* r) {
  if (!r || !r->_owner) return;
  ResultOwner* o = reinterpret_cast<ResultOwner*>(r->_owner);
  for (void* p : o->pinned) pinned_free(p);
  delete o;
  memset(r, 0, sizeof(*r));
}

#define PDSB_GUARD(call)                                    \
  do {                                                      \
    if (require_device()) return 1;                         \
    if (!kw || !cols || !out) { set_error("null argument"); return 1; } \
    memset(out, 0, sizeof(*out));                           \
    int rc = (call);                                        \
    if (rc) pdsb_host_result_free(out);                     \
    return rc;                                              \
  } while (0)

int pdsb_host_lin_reg(const pdsb_column* cols, int n_cols, const pdsb_lr_kwargs* kw, int f32, int n_targets,
                      int want_pred, int w_rcond, pdsb_host_result* out) {
  PDSB_GUARD(f32 ? host_lin_reg_t<float>(cols, n_cols, kw, n_targets, want_pred, w_rcond, out)
                 : host_lin_reg_t<double>(cols, n_cols, kw, n_targets, want_pred, w_rcond, out));
}
int pdsb_host_report(const pdsb_column* cols, int n_cols, const pdsb_lr_kwargs* kw, int f32, int weighted,
                     pdsb_host_result* out) {
  PDSB_GUARD(f32 ? host_report_t<float>(cols, n_cols, kw, weighted, out)
                 : host_report_t<double>(cols, n_cols, kw, weighted, out));
}
int pdsb_host_online(const pdsb_column* cols, int n_cols, const pdsb_lr_kwargs* kw, int f32, int rolling,
                     pdsb_host_result* out) {
  PDSB_GUARD(f32 ? host_online_t<float>(cols, n_cols, kw, rolling, out)
                 : host_online_t<double>(cols, n_cols, kw, rolling, out));
}
int pdsb_host_logistic(const pdsb_column* cols, int n_cols, const pdsb_lr_kwargs* kw, int want_pred, pdsb_host_result* out) {
  PDSB_GUARD(host_logistic(cols, n_cols, kw, want_pred, out));
}
int pdsb_host_grouped_lin_reg(const pdsb_column* cols, int n_cols, const int64_t* group_offsets, int64_t n_groups,
                              const pdsb_lr_kwargs* kw, int f32, pdsb_host_result* out) {
  if (!group_offsets) { set_error("null group offsets"); return 1; }
  PDSB_GUARD(f32 ? host_grouped_t<float>(cols, n_cols, group_offsets, n_groups, kw, out)
                 : host_grouped_t<double>(cols, n_cols, group_offsets, n_groups, kw, out));
}
int pdsb_host_grouped_lin_reg_pred(const pdsb_column* cols, int n_cols, const int64_t* group_offsets, int64_t n_groups,
                                   const pdsb_lr_kwargs* kw, int f32, pdsb_host_result* out) {
  if (!group_offsets) { set_error("null group offsets"); return 1; }
  PDSB_GUARD(f32 ? host_grouped_pred_t<float>(cols, n_cols, group_offsets, n_groups, kw, out)
                 : host_grouped_pred_t<double>(cols, n_cols, group_offsets, n_groups, kw, out));
}
int pdsb_host_grouped_logistic(const pdsb_column* cols, int n_cols, const int64_t* group_offsets, int64_t n_groups,
                               const pdsb_lr_kwargs* kw, int want_pred, pdsb_host_result* out) {
  if (!group_offsets) { set_error("null group offsets"); return 1; }
  PDSB_GUARD(host_grouped_logistic(cols, n_cols, group_offsets, n_groups, kw, want_pred, out));
}

int pdsb_host_pca(const pdsb_column* cols, int n_cols, int mode, int k, pdsb_host_result* out) {
  if (require_device()) return 1;
  if (!cols || !out || n_cols < 1 || mode < 0 || mode > 2) { set_error("pca: invalid arguments"); return 1; }
  if (mode == 2 && (k < 1 || k > n_cols)) { set_error("Input `k` should be between 1 and the number of features inclusive."); return 1; }
  memset(out, 0, sizeof(*out));
  bool all_f32 = true;
  for (int c = 0; c < n_cols; ++c) all_f32 &= cols[c].dtype == PDSB_F32;
  const int rc = all_f32 ? host_pca_t<float>(cols, n_cols, mode, k, out) : host_pca_t<double>(cols, n_cols, mode, k, out);
  if (rc) pdsb_host_result_free(out);
  return rc;
}

int pdsb_host_smooth_spline(const pdsb_column* cols, int n_cols, double lambda, pdsb_host_result* out) {
  if (require_device()) return 1;
  if (!cols || !out) { set_error("smooth_spline: invalid arguments"); return 1; }
  memset(out, 0, sizeof(*out));
  const int rc = host_smooth_spline(cols, n_cols, lambda, out);
  if (rc) pdsb_host_result_free(out);
  return rc;
}

int pdsb_host_isotonic_regression(const pdsb_column* cols, int n_cols, int has_weights, int increasing,
                                  pdsb_host_result* out) {
  if (require_device()) return 1;
  if (!cols || !out) { set_error("isotonic_regression: invalid arguments"); return 1; }
  memset(out, 0, sizeof(*out));
  const int rc = host_isotonic_regression(cols, n_cols, has_weights, increasing, out);
  if (rc) pdsb_host_result_free(out);
  return rc;
}

}  // extern "C"
