// K17 — group_by(key).agg(pds.lin_reg_report(...)): every group's OLS report in one launch sequence.
//
// Polars' loop makes one pl_lin_reg_report call per group (K9: moments, K3's INV solve, K4's residual pass, the HC
// weights and a weighted moments pass, a one-CTA finalize).  Here the frame stays in HBM in key order, as for pl_lr_by:
//   pass 0 + 1  K5's work list and grouped moments (group_moments, k5_grouped.cu): the kept-row count n_g and X'X, X'y;
//   pass 2      one thread per group: group_solve (k5_solve.h) with PDSB_METHOD_INV, K3's report solve (pivoted QR, no
//               ridge, no rank gate, G^-1 as q more right-hand sides): beta [n_groups x q] and G^-1 [n_groups x q x q];
//   pass 3      one warp per item of the pass-0 queue: the group's beta (and G^-1 for hc2 / hc3) staged once, then the
//               item's rows streamed once: e = y - [x | 1] beta by predict_row.h's rule, SSR = sum e^2 in f64, the
//               omega-weighted meat sum omega z z^T (hc0..hc3, omega by report_rows.h's hc_weight), and count / mean / M2
//               of the non-null y values (Chan's merge); nothing is written per row;
//               at its start the warps also take the groups, 32 at a time, for n_g and t_{0.975, n_g - q};
//   pass 4      one warp per group: the item partials summed in item order, var(y) rounded to T, then the 8 x q block by
//               report_rows.h's report_column (K9's finalize rule).
// Item partials are combined in a fixed order, so a group's report is bit for bit the same whichever warp ran its items
// and whatever the other groups hold.  HBM bytes per row: (p + 1) s in pass 1 and again in pass 3 (plus s for the y
// validity when y has nulls); nothing per row is written.
#include "../common.h"
#include "kernels.h"
#include "../host/host.h"
#include "k5_solve.h"
#include "predict_row.h"
#include "report_rows.h"

namespace pdsb {

namespace {

constexpr int RS_WARPS = 8;      // warps per CTA of the se pass
constexpr int RH_WARPS = 4;      // warps per CTA of the HC pass
constexpr int RP_MAXP = 64;      // group_moments' feature limit
// pass-3 partial k of item it lives at part[k * n_items + it]: k = 0 SSR, 1..3 count / mean / M2 of the non-null y,
// 4 + m (hc0..hc3) meat entry m, packed upper triangle over the coefficients [x | 1]
constexpr int RP_HEAD = 4;

// count / mean / M2 of a set of values, merged by Chan et al.'s rule (never sum y^2 - (sum y)^2 / n)
struct YVar { double n, mean, m2; };
__device__ __forceinline__ void yvar_add(YVar& a, double y) {
  a.n += 1.0;
  const double d = y - a.mean;
  a.mean += d / a.n;
  a.m2 += d * (y - a.mean);
}
__device__ __forceinline__ YVar yvar_merge(const YVar& a, const YVar& b) {
  const double n = a.n + b.n;
  if (n == 0.0) return a;
  const double d = b.mean - a.mean, f = b.n / n;
  return {n, a.mean + d * f, a.m2 + b.m2 + d * d * (a.n * f)};
}
// lane 0 ends with the warp's SSR and y terms, reduced in a fixed pattern
__device__ __forceinline__ void warp_item_partials(double ssr, YVar v, double* __restrict__ part, int64_t n_items,
                                                   int64_t item) {
  for (int off = 16; off; off >>= 1) {
    ssr += __shfl_xor_sync(0xffffffffu, ssr, off);
    const YVar o{__shfl_xor_sync(0xffffffffu, v.n, off), __shfl_xor_sync(0xffffffffu, v.mean, off),
                 __shfl_xor_sync(0xffffffffu, v.m2, off)};
    v = yvar_merge(v, o);
  }
  if ((threadIdx.x & 31) == 0) {
    part[0 * n_items + item] = ssr;
    part[1 * n_items + item] = v.n;
    part[2 * n_items + item] = v.mean;
    part[3 * n_items + item] = v.m2;
  }
}

struct GroupScalars {
  const double* part1; int nm; const int64_t* item_start; int64_t n_groups;
  double* gstat; unsigned long long* tqueue;
};

// t_{0.975, nu}.  For nu >= 500 the Cornish-Fisher expansion of the Student-t quantile in 1 / nu to the fifth term
// (Abramowitz & Stegun 26.7.5 and its next term) about z = Phi^-1(0.975): its truncation error is below 1e-16 relative
// there (5e-15 at nu = 200, against a 40-digit root of the incomplete beta), i.e. the correctly rounded quantile, which
// the root search of special.h (some hundred microseconds of serial f64 work per group at nu ~ 1e4) returns too.
// Below 500, student_t_ppf itself (K9's).
__device__ __forceinline__ double t_quantile_975(double nu) {
  if (!(nu >= 500.0)) return student_t_ppf(0.975, nu);
  const double z = 1.9599639845400543, z2 = z * z;
  const double g1 = z * (z2 + 1.0) / 4.0;
  const double g2 = z * ((5.0 * z2 + 16.0) * z2 + 3.0) / 96.0;
  const double g3 = z * (((3.0 * z2 + 19.0) * z2 + 17.0) * z2 - 15.0) / 384.0;
  const double g4 = z * ((((79.0 * z2 + 776.0) * z2 + 1482.0) * z2 - 1920.0) * z2 - 945.0) / 92160.0;
  const double g5 = z * (((((27.0 * z2 + 339.0) * z2 + 930.0) * z2 - 1782.0) * z2 - 765.0) * z2 + 17955.0) / 368640.0;
  const double u = 1.0 / nu;
  return z + u * (g1 + u * (g2 + u * (g3 + u * (g4 + u * g5))));
}

// The per-group scalars pass 4 needs before its rows: gstat[g] = n_g (pass 1's count moment summed in item order) and
// gstat[n_groups + g] = t_{0.975, n_g - q} (t_quantile_975).  A warp takes 32 groups (a lane each) from its own counter
// at the start of pass 3, so the quantiles of small groups (a serial root search each) are computed next to the warps
// that stream rows instead of after them.
__device__ __forceinline__ void group_scalars(const double* __restrict__ part1, int nm, const int64_t* __restrict__ item_start,
                                              int64_t n_groups, int64_t n_items, int q, const int* __restrict__ status,
                                              double* __restrict__ gstat, unsigned long long* __restrict__ tqueue) {
  const int64_t n_chunks = (n_groups + 31) / 32;
  for (int64_t c = pop_item(tqueue); c < n_chunks; c = pop_item(tqueue)) {
    const int64_t g = c * 32 + (threadIdx.x & 31);
    if (g < n_groups && status[g] == PDSB_OK) {
      double n = 0.0;
      for (int64_t it = item_start[g]; it < item_start[g + 1]; ++it) n += part1[(size_t)(nm - 1) * n_items + it];
      gstat[g] = n;
      gstat[n_groups + g] = t_quantile_975(n - (double)q);
    }
  }
}

// ---------------- pass 3, std_err = "se": SSR and the y terms ----------------
// rows [row, row + VEC): e by predict_row.h's rule; a row is kept (enters SSR) when none of x, y is NaN / inf, pass 1's
// rule; y enters the variance when its validity (ymask, nullable) is not 0
template <typename T, int VEC>
__device__ __forceinline__ void se_rows(const T* __restrict__ X, int64_t ldx, const T* __restrict__ y,
                                        const T* __restrict__ ymask, int64_t row, int p, const T* sb, double& ssr,
                                        YVar& yv) {
  T probe[VEC], acc[VEC];
#pragma unroll
  for (int v = 0; v < VEC; ++v) probe[v] = T(0);
  predict_acc<T, VEC>(sb, p, [&](int c, T (&xv)[VEC]) {
    load_rows<T, VEC>(X + (int64_t)c * ldx + row, xv);
#pragma unroll
    for (int v = 0; v < VEC; ++v) probe[v] = fma(xv[v], T(0), probe[v]);
  }, acc);
  T yvv[VEC], mv[VEC];
  load_rows<T, VEC>(y + row, yvv);
  if (ymask) load_rows<T, VEC>(ymask + row, mv);
#pragma unroll
  for (int v = 0; v < VEC; ++v) {
    const T e = resid_of(yvv[v], acc[v]);
    if (fma(yvv[v], T(0), probe[v]) == T(0)) ssr += (double)e * (double)e;
    if (!ymask || mv[v] != T(0)) yvar_add(yv, (double)yvv[v]);
  }
}

template <typename T, bool VECTOR>
__global__ void __launch_bounds__(RS_WARPS * 32)
report_se_kernel(const T* __restrict__ X, int64_t ldx, const T* __restrict__ y, const T* __restrict__ ymask,
                 const int64_t* __restrict__ rows, const int64_t* __restrict__ group, int64_t n_items, int p,
                 int add_bias, const double* __restrict__ beta, const int* __restrict__ status,
                 double* __restrict__ part, unsigned long long* __restrict__ queue, GroupScalars gs) {
  constexpr int VEC = VECTOR ? 16 / sizeof(T) : 1;
  __shared__ T sbeta[RS_WARPS][RP_MAXP + 1];
  const int lane = threadIdx.x & 31;
  T* sb = sbeta[threadIdx.x >> 5];
  const int q = p + (add_bias ? 1 : 0);
  group_scalars(gs.part1, gs.nm, gs.item_start, gs.n_groups, n_items, q, status, gs.gstat, gs.tqueue);
  for (int64_t item = pop_item(queue); item < n_items; item = pop_item(queue)) {
    const int64_t g = group[item];
    if (status[g] != PDSB_OK) continue;            // a null report: pass 4 reads nothing of it
    const int64_t r0 = rows[2 * item], r1 = rows[2 * item + 1];
    __syncwarp();                                  // the previous item's reads of sb are done
    for (int i = lane; i <= p; i += 32) sb[i] = staged_beta<T>(beta, (size_t)g * q, i, p, add_bias, true);
    __syncwarp();
    double ssr = 0.0;
    YVar yv{0.0, 0.0, 0.0};
    walk_item_rows<VEC>(r0, r1, [&](int64_t row, auto v) {
      se_rows<T, decltype(v)::value>(X, ldx, y, ymask, row, p, sb, ssr, yv);
    });
    warp_item_partials(ssr, yv, part, n_items, item);
  }
}

// ---------------- pass 3, hc0..hc3: SSR, the y terms and the meat ----------------
// Per warp of dynamic shared memory: a [32][q + 2] f64 tile (a row's z = [x | 1] and omega), G^-1 as T (hc2 / hc3) and
// the staged beta.  Each lane takes one row of a 32-row batch: e, omega = hc_weight (its row of the tile, G^-1 from
// shared memory), then every lane adds its share of the q (q + 1) / 2 meat entries over the batch's 32 rows in f64.
__host__ __device__ inline size_t hc_warp_bytes(int p, int q, int se_type, int tsize) {
  const size_t b = (size_t)32 * (q + 2) * 8 + (se_type >= 3 ? (size_t)q * q * tsize : 0) + (size_t)(p + 1) * tsize;
  return (b + 15) & ~size_t(15);
}

template <typename T>
__global__ void __launch_bounds__(RH_WARPS * 32)
report_hc_kernel(const T* __restrict__ X, int64_t ldx, const T* __restrict__ y, const T* __restrict__ ymask,
                 const int64_t* __restrict__ rows, const int64_t* __restrict__ group, int64_t n_items, int p,
                 int add_bias, int se_type, const double* __restrict__ beta, const double* __restrict__ ginv,
                 const int* __restrict__ status, double* __restrict__ part, unsigned long long* __restrict__ queue,
                 GroupScalars gs) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int lane = threadIdx.x & 31;
  const int q = p + (add_bias ? 1 : 0), ld = q + 2, nmq = q * (q + 1) / 2;
  group_scalars(gs.part1, gs.nm, gs.item_start, gs.n_groups, n_items, q, status, gs.gstat, gs.tqueue);
  const bool lev = se_type >= 3;
  unsigned char* mine = smem_raw + (size_t)(threadIdx.x >> 5) * hc_warp_bytes(p, q, se_type, sizeof(T));
  double* tile = reinterpret_cast<double*>(mine);
  T* gi = reinterpret_cast<T*>(tile + (size_t)32 * ld);
  T* sb = gi + (lev ? (size_t)q * q : 0);
  double* my = tile + (size_t)lane * ld;
  const int per_lane = (nmq + 31) / 32;
  for (int64_t item = pop_item(queue); item < n_items; item = pop_item(queue)) {
    const int64_t g = group[item];
    if (status[g] != PDSB_OK) continue;
    const int64_t r0 = rows[2 * item], r1 = rows[2 * item + 1];
    __syncwarp();
    for (int i = lane; i <= p; i += 32) sb[i] = staged_beta<T>(beta, (size_t)g * q, i, p, add_bias, true);
    if (lev) for (int i = lane; i < q * q; i += 32) gi[i] = (T)ginv[(size_t)g * q * q + i];
    __syncwarp();
    double ssr = 0.0;
    YVar yv{0.0, 0.0, 0.0};
    double acc[PACKED_ACC];
    for (int m = 0; m < per_lane; ++m) acc[m] = 0.0;
    for (int64_t rb = r0; rb < r1; rb += 32) {
      const int64_t r = rb + lane;
      const bool in = r < r1;
      T probe = T(0), pr[1];
      predict_acc<T, 1>(sb, p, [&](int c, T (&xv)[1]) {
        xv[0] = in ? X[(int64_t)c * ldx + r] : T(0);
        probe = fma(xv[0], T(0), probe);
        my[c] = (double)xv[0];
      }, pr);
      const T yr = in ? y[r] : T(0);
      const bool keep = in && fma(yr, T(0), probe) == T(0);
      const T e = resid_of(yr, pr[0]);
      if (in && (!ymask || ymask[r] != T(0))) yvar_add(yv, (double)yr);
      if (keep) {
        ssr += (double)e * (double)e;
        if (add_bias) my[p] = 1.0;
        my[q] = (double)hc_weight<T>(e, q, se_type, [&](int a) { return (T)my[a]; }, [&](int a, int b) { return gi[a * q + b]; });
      } else {
        for (int a = 0; a <= q; ++a) my[a] = 0.0;
      }
      __syncwarp();
      tile_triangle_sum(tile, ld, q, tile + q, ld, acc);     // omega z_i z_j: omega in column q
      __syncwarp();
    }
    warp_item_partials(ssr, yv, part, n_items, item);
    for (int m = 0; m < per_lane; ++m) {
      const int k = lane + 32 * m;
      if (k < nmq) part[(size_t)(RP_HEAD + k) * n_items + item] = acc[m];
    }
  }
}

// ---------------- pass 4: per-group finalize ----------------
// One warp per group, FIN_WARPS groups per CTA (one resident warp per group at 1e4 groups: each lane's Student-t
// survival function is a serial evaluation, and waves of one-warp CTAs would queue behind it): SSR, var(y) (rounded to
// T: the loop's t.var() input has the data's type) and the meat, each summed over the group's items in item order, n_g
// and t_alpha from pass 3; then report_column for every coefficient.  A group whose solve is not OK (fewer kept rows than
// coefficients) gets a NaN block.
constexpr int FIN_WARPS = 4;
__global__ void __launch_bounds__(FIN_WARPS * 32)
report_finalize_grouped_kernel(const double* __restrict__ part3, const int64_t* __restrict__ item_start,
                               int64_t n_groups, int64_t n_items, int p, int add_bias, int se_type, int is_f32,
                               const double* __restrict__ beta, const double* __restrict__ ginv,
                               const int* __restrict__ status, const double* __restrict__ gstat,
                               double* __restrict__ out) {
  extern __shared__ double smeat_all[];      // q (q + 1) / 2 per warp with hc0..hc3
  const int lane = threadIdx.x & 31;
  const int64_t g = (int64_t)blockIdx.x * FIN_WARPS + (threadIdx.x >> 5);
  if (g >= n_groups) return;
  const int q = p + (add_bias ? 1 : 0), nmq = q * (q + 1) / 2;
  double* smeat = smeat_all + (size_t)(threadIdx.x >> 5) * (se_type > 0 ? nmq : 0);
  double* o = out + (size_t)g * 8 * q;
  if (status[g] != PDSB_OK) {
    for (int i = lane; i < 8 * q; i += 32) o[i] = nan("");
    return;
  }
  const int64_t it0 = item_start[g], it1 = item_start[g + 1];
  double ssr = 0.0, var = 0.0;
  if (lane == 0) {
    YVar v{0.0, 0.0, 0.0};
    for (int64_t it = it0; it < it1; ++it) {
      ssr += part3[it];
      v = yvar_merge(v, YVar{part3[(size_t)1 * n_items + it], part3[(size_t)2 * n_items + it], part3[(size_t)3 * n_items + it]});
    }
    var = v.n > 1.0 ? v.m2 / (v.n - 1.0) : nan("");
    if (is_f32) var = (double)(float)var;
  }
  ssr = __shfl_sync(0xffffffffu, ssr, 0);
  var = __shfl_sync(0xffffffffu, var, 0);
  if (se_type > 0)
    for (int k = lane; k < nmq; k += 32) {
      double s = 0.0;
      for (int64_t it = it0; it < it1; ++it) s += part3[(size_t)(RP_HEAD + k) * n_items + it];
      smeat[k] = s;
    }
  __syncwarp();
  const double n = gstat[g], t_alpha = gstat[n_groups + g];
  for (int i = lane; i < q; i += 32)
    report_column(i, q, se_type, n, ssr, ssr, var, t_alpha, beta + (size_t)g * q, ginv + (size_t)g * q * q,
                  [&](int r, int c) { return smeat[packed_index(r, c, q)]; }, o);
}

}  // namespace

template <typename T>
int grouped_report(const T* X, int64_t ldx, const T* y, const T* ymask, const int64_t* offsets, int64_t n_groups,
                   int64_t n, int p, int add_bias, int se_type, double* out, int* status, cudaStream_t s) {
  if (n_groups <= 0) return 0;
  if (p < 1 || p > RP_MAXP) { set_error("grouped lin_reg_report: p=%d not supported (1..%d)", p, RP_MAXP); return 1; }
  if (se_type < 0 || se_type > 4) { set_error("grouped lin_reg_report: std_err %d not supported", se_type); return 1; }
  if (!X || !y || !offsets || !out || !status) { set_error("grouped lin_reg_report: null argument"); return 1; }
  const int q = p + (add_bias ? 1 : 0), nmq = q * (q + 1) / 2;
  const bool hc = se_type > 0;
  DevBag bag(s);
  // pass 0 + 1; pass 3 takes its items from the same list
  GroupWork wl;
  double* part1 = nullptr;
  if (build_work_list(offsets, n_groups, n, ItemCount::EXACT, ItemMaps::ROWS_AND_GROUP, bag, wl, s) ||
      group_moments<T>(X, ldx, y, offsets, n_groups, p, wl, bag, &part1, s))
    return 1;
  const int64_t n_items = wl.n_items;
  // pass 2
  double* beta = bag.alloc<double>((size_t)n_groups * q);
  double* ginv = bag.alloc<double>((size_t)n_groups * q * q);
  if (!beta || !ginv) return 1;
  const int nrhs = group_solve_nrhs(PDSB_METHOD_INV, q);
  double* ws = nullptr;
  if (!group_solve_launch(p, q, nrhs).shared && !(ws = bag.alloc<double>(((size_t)q * q + (size_t)q * nrhs + q) * n_groups)))
    return 1;
  GroupSolveArgs a;
  a.part = part1; a.item_start = wl.item_start; a.offsets = offsets; a.n_groups = n_groups; a.n_items = n_items;
  a.p = p; a.add_bias = add_bias; a.solver = PDSB_SOLVER_QR; a.l2 = 0.0; a.tol = 0.0;
  a.method = PDSB_METHOD_INV; a.positive = 0; a.max_iter = 0; a.l1 = 0.0; a.cd_tol = 0.0;
  a.ws = ws; a.beta = beta; a.status = status; a.ginv = ginv;
  if (launch_group_solve(a, s)) return 1;
  // pass 3
  double* part3 = bag.alloc<double>((size_t)(RP_HEAD + (hc ? nmq : 0)) * n_items);
  double* gstat = bag.alloc<double>((size_t)2 * n_groups);
  if (!part3 || !gstat) return 1;
  PDSB_CUDA_OK(cudaMemsetAsync(wl.queue, 0, 2 * sizeof(unsigned long long), s));
  const int q1 = p + 2;
  const GroupScalars gs{part1, q1 * (q1 + 1) / 2, wl.item_start, n_groups, gstat, wl.queue + 1};
  if (!hc) {
    const bool vec_ok = rows_vec_ok<T>(ldx, {X, y, ymask});
    auto kern = vec_ok ? report_se_kernel<T, true> : report_se_kernel<T, false>;
    const int grid = persistent_grid(kern, RS_WARPS * 32, 0, n_items, 4);
    if (!grid) return 1;
    kern<<<grid, RS_WARPS * 32, 0, s>>>(X, ldx, y, ymask, wl.rows, wl.group, n_items, p, add_bias, beta, status, part3,
                                        wl.queue, gs);
  } else {
    const size_t smem = RH_WARPS * hc_warp_bytes(p, q, se_type, sizeof(T));
    auto kern = report_hc_kernel<T>;
    const int grid = persistent_grid(kern, RH_WARPS * 32, smem, n_items, 1);
    if (!grid) return 1;
    kern<<<grid, RH_WARPS * 32, smem, s>>>(X, ldx, y, ymask, wl.rows, wl.group, n_items, p, add_bias, se_type, beta, ginv,
                                           status, part3, wl.queue, gs);
  }
  PDSB_LAUNCH_OK();
  count_launch();
  // pass 4
  const size_t fsmem = hc ? (size_t)FIN_WARPS * nmq * sizeof(double) : 0;
  if (smem_opt_in(report_finalize_grouped_kernel, fsmem)) return 1;
  report_finalize_grouped_kernel<<<(unsigned)ceil_div(n_groups, (int64_t)FIN_WARPS), FIN_WARPS * 32, fsmem, s>>>(
      part3, wl.item_start, n_groups, n_items, p, add_bias, se_type, sizeof(T) == 4, beta, ginv, status, gstat, out);
  PDSB_LAUNCH_OK();
  count_launch();
  return 0;
}

template int grouped_report<float>(const float*, int64_t, const float*, const float*, const int64_t*, int64_t, int64_t,
                                   int, int, int, double*, int*, cudaStream_t);
template int grouped_report<double>(const double*, int64_t, const double*, const double*, const int64_t*, int64_t,
                                    int64_t, int, int, int, double*, int*, cudaStream_t);

}  // namespace pdsb
