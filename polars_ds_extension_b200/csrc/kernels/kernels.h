// Internal launch wrappers of the device kernels (C++), used by the C-ABI layer in host/api.cc.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include "../../../include/pdsb.h"

namespace pdsb {

constexpr int FRAME_ROWS = 128;   // rows per block of the row-blocked frame layout: [block][column][FRAME_ROWS]

// K2 moments M = [X | Y | 1]' diag(w) [X | Y | 1] (q1 x q1 f64, row-major, q1 = p + t + 1 <= 260; the "1" column is
// `mask` when given).  X = p columns, Y = t columns: column-major with leading dimensions ldx / ldy (bstride == 0), or
// columns of one row-blocked frame of bstride / FRAME_ROWS columns (ldx, ldy unused).  moments() picks the kernel; the
// contract says what the caller lets f32 data be multiplied and summed in (f64 data always gets f64 products and sums):
enum class MomentsPrecision {
  TF32_ALLOWED,   // register kernel (f32 products), wgmma (3xTF32 products), DMMA, tile.  Honours pdsb_set_moments_path
                  // and records pdsb_last_moments_path (thread-local)
  F64_ACCUM,      // DMMA (f64 products), else the tile kernel (f32 products, f64 sums)
  F64_PRODUCTS,   // column-major only: DMMA; f32 operands the DMMA kernels do not take are widened to f64 first
};
template <typename T>
int moments(MomentsPrecision prec, const T* X, int64_t ldx, const T* Y, int64_t ldy, const T* w, const T* mask, int64_t n,
            int p, int t, double* M, cudaStream_t s, int64_t bstride = 0);
int last_moments_path();         // pdsb_last_moments_path
void force_moments_path(int);    // pdsb_set_moments_path

// The moments kernels, each with the test of the calls it takes; moments() is the only caller of the launchers.
// K2s register moments (K5's kernel), f32, one target
bool moments_small_supported(int64_t n, int p, int t, int64_t bstride);
template <typename T>
int moments_small(const T* X, int64_t ldx, const T* y, int64_t n, int p, double* M, cudaStream_t s);
// K2b wgmma + TMA, f32, 3xTF32 split (hi/lo), f64 flush; p <= 64 features, t <= 4 targets.  Returns 0 ok, 1 error,
// -1 when the tensor maps cannot be encoded at run time.
bool moments_wgmma_supported(const float* X, int64_t ldx, const float* Y, int64_t ldy, int64_t n, int p, int t,
                             int64_t bstride);
int moments_wgmma_f32(const float* X, int64_t ldx, const float* Y, int64_t ldy, const float* mask, int64_t n, int p, int t,
                      double* M, cudaStream_t s, int64_t bstride);
void set_tc_mode(int m);   // 1 raw hi operand (default), 0 the hi rows clear the low 13 bits themselves (cross-check)
// K2a FP64 tensor cores (f64 products; f32 columns widened on the fly), column-major, up to 64 columns
template <typename T>
bool moments_dmma_supported(const T* X, int64_t ldx, const T* Y, int64_t ldy, const T* w, const T* mask, int64_t n, int p,
                            int t, int64_t bstride);
template <typename T>
int moments_dmma(const T* X, int64_t ldx, const T* Y, int64_t ldy, const T* w, const T* mask, int64_t n, int p, int t,
                 double* M, cudaStream_t s);
// K2a register tiles (DFMA / FFMA: products in T, f64 sums), any call
template <typename T>
int moments_tile(const T* X, int64_t ldx, const T* Y, int64_t ldy, const T* w, const T* mask, int64_t n, int p, int t,
                 double* M, cudaStream_t s, int64_t bstride);

// K3 single-CTA solve on the moments
int solve_from_moments(const double* M, const pdsb_solve_opts& o, double* beta, int* status, double* aux,
                       cudaStream_t s);

// K4 predict / residual / SSR
template <typename T>
int predict_resid(const T* X, int64_t ldx, const T* Y, int64_t ldy, const T* w, const T* mask, int64_t n,
                  int p, int t, int add_bias, const double* beta, const int* status, T* pred, T* resid,
                  int64_t ldo, uint8_t* valid, double* ssr, cudaStream_t s);
// K4 on a row-blocked frame (16-byte aligned): X = columns [xcol, xcol+p), Y = columns [ycol, ycol+t); pred / resid /
// valid column-major with leading dimension ldo
int predict_frame_f32(const float* frame, int64_t n, int ncols, int xcol, int p, int ycol, int t, int add_bias,
                      const float* mask, const double* beta, const int* status, float* pred, float* resid, int64_t ldo,
                      uint8_t* valid, double* ssr, cudaStream_t s);

// K1 pack: src column chunk (any numeric dtype, optional validity bitmap) -> T column
// mode: 0 null->NaN, 1 null->fill, 2 null->0 (row masked elsewhere)
template <typename T>
int pack_chunk(const void* src, int src_dtype, const uint8_t* validity, int64_t bit_offset, int64_t len,
               T* dst, int mode, T fill, cudaStream_t s, int64_t bstride = 0, int64_t row0 = 0);
// column-major [n x ncols] (ld) -> row-blocked frame
template <typename T>
int to_frame(const T* src, int64_t ld, int64_t n, int ncols, T* frame, cudaStream_t s);
// rowmask[i] &= validity bit (rowmask pre-set to 1)
template <typename T>
int and_validity(const uint8_t* validity, int64_t bit_offset, int64_t len, T* rowmask, cudaStream_t s);
template <typename T>
int fill_value(T* dst, int64_t len, T v, cudaStream_t s);
// zero rows of a column where rowmask == 0
template <typename T>
int zero_masked(T* col, const T* rowmask, int64_t len, cudaStream_t s);
template <typename T>
int count_mask(const T* rowmask, int64_t len, double* out, cudaStream_t s);
// *out = sum of v[0..len) / len, summed in a fixed order (single block, the reduction shape of count_mask): reproducible
template <typename T>
int mean_values(const T* v, int64_t len, double* out, cudaStream_t s);

// K5 pass 0, the work list of one call: a group of len rows has ceil(len / 8192) items of equal size, an empty group one
// empty item.  item_start [n_groups + 1]: the first item of each group; rows [n_items][2] (when asked for): each item's
// row range; group [n_items] (when asked for): each item's group; queue [2]: the item counter of a persistent grid and
// a second counter for the caller, both zeroed by whoever launches on them.
struct GroupWork {
  int64_t* item_start = nullptr;
  int64_t* rows = nullptr;
  int64_t* group = nullptr;
  int64_t n_items = 0;
  unsigned long long* queue = nullptr;
};
struct DevBag;
// EXACT reads the item count back (one synchronisation); BOUND sizes for group_items_bound and reads nothing back: the
// items past the real count lie after the last group's rows, so they are empty.
enum class ItemCount { EXACT, BOUND };
enum class ItemMaps { NONE, ROWS, ROWS_AND_GROUP };
// n_groups >= 1; the buffers come from bag
int build_work_list(const int64_t* offsets, int64_t n_groups, int64_t n, ItemCount count, ItemMaps maps, DevBag& bag,
                    GroupWork& wl, cudaStream_t s);
int64_t group_items_bound(int64_t n, int64_t n_groups);

// Launch helpers of the grouped kernels.  smem_opt_in: a kernel that needs more than 48 KB of dynamic shared memory
// has to opt in.  persistent_grid: the opt-in, then as many CTAs of `threads` threads as are resident at once
// (fallback_occ per SM when the occupancy query fails), but no more than n_items items at one per warp need; 0 on error.
int smem_opt_in(const void* kernel, size_t smem);
int persistent_grid(const void* kernel, int threads, size_t smem, int64_t n_items, int fallback_occ);
template <typename K> int smem_opt_in(K* kernel, size_t smem) { return smem_opt_in((const void*)kernel, smem); }
template <typename K> int persistent_grid(K* kernel, int threads, size_t smem, int64_t n_items, int fallback_occ) {
  return persistent_grid((const void*)kernel, threads, smem, n_items, fallback_occ);
}

// K5 grouped (segmented) OLS / ridge, one warp per problem.  With bag and wl the call's work list (exact, rows and
// item -> group) comes back in wl for grouped_predict, its buffers in bag.
template <typename T>
int grouped_lin_reg(const T* X, int64_t ldx, const T* y, const int64_t* offsets, int64_t n_groups,
                    int64_t n, int p, const pdsb_solve_opts& o, double* beta, int* status, cudaStream_t s,
                    DevBag* bag = nullptr, GroupWork* wl = nullptr);
// K5 weighted (group_by().agg(lin_reg(weights=w))): grouped_lin_reg with row weights w (same layout as y): every product
// of the moments pass is w z_i z_j, a row with a NaN / inf in x, y or w drops out, and the "fewer rows than
// coefficients" gate counts the kept rows (not sum w).  With w = 1 the result is bit for bit grouped_lin_reg's.
// o.method PDSB_METHOD_LSTSQ only; 1 <= p <= 64.  bag / wl as for grouped_lin_reg.
template <typename T>
int grouped_wls_lin_reg(const T* X, int64_t ldx, const T* y, const T* w, const int64_t* offsets, int64_t n_groups,
                        int64_t n, int p, const pdsb_solve_opts& o, double* beta, int* status, cudaStream_t s,
                        DevBag* bag = nullptr, GroupWork* wl = nullptr);
// K5 on t targets (group_by().agg(lin_reg(target=[...]))): Z = [y_0 .. y_{t-1} | x_0 .. x_{p-1}] column-major with
// leading dimension ld, null rows as NaN.  beta [n_groups][t][p + bias], status [n_groups]; target c of group g is bit for
// bit grouped_lin_reg's on [x | y_c] when both run the same moments kernel (p + t <= 11, or p >= 11) and no value is
// NaN / inf; a row with a NaN / inf in any column drops out for every target.  o.method PDSB_METHOD_LSTSQ only;
// t, p >= 1, p + t <= 65.
template <typename T>
int grouped_lin_reg_multi(const T* Z, int64_t ld, int t, int p, const int64_t* offsets, int64_t n_groups, int64_t n,
                          const pdsb_solve_opts& o, double* beta, int* status, cudaStream_t s);
// K5 on an autoregression (group_by().agg(query_ar_coeffs(x, lag))): group g = rows [offsets[g], offsets[g+1]) of the one
// column x (device offsets); its design is target rows t = lag .. m-1 with y_t = x_t and features x_{t-1} .. x_{t-lag},
// and its beta / status are bit for bit grouped_lin_reg's on those lagged columns materialised per group.  x holds the
// feature values (nulls filled, or NaN to drop every row they reach); mask (nullable, per-row 0 / 1): 0 drops row t as a
// target only.  1 <= lag <= 64.
template <typename T>
int grouped_ar_lin_reg(const T* x, const T* mask, const int64_t* offsets, int64_t n_groups, int64_t n, int lag,
                       const pdsb_solve_opts& o, double* beta, int* status, cudaStream_t s);
// K5 pass 3: pred / resid / valid of every row of [X | y] in group order, with the beta [n_groups x (p+bias)] and status
// [n_groups] of grouped_lin_reg and K4's per-row arithmetic.  mask (nullable): per-row 0 / 1, 0 = null row.
// inv_link = PDSB_GLM_BINOMIAL (f64 only; the logistic_reg probabilities): pred = sigmoid(X beta + bias), valid = mask
// only; y, status and resid are not used.  wl (nullable): a work list of these offsets with rows and item -> group, as
// grouped_lin_reg returns it; without one the pass builds its own.
template <typename T>
int grouped_predict(const T* X, int64_t ldx, const T* y, const int64_t* offsets, int64_t n_groups, int64_t n, int p,
                    int add_bias, const double* beta, const int* status, const T* mask, T* pred, T* resid,
                    uint8_t* valid, cudaStream_t s, int inv_link = PDSB_GLM_GAUSSIAN, const GroupWork* wl = nullptr);
// K5 pass 1 of a batched fit on the work list wl (rows needed for p <= 10): the per-item moments of [X | y | 1] with
// null / NaN rows dropped, *part [(p+2)(p+3)/2][wl.n_items] from bag.  1 <= p <= 64.
template <typename T>
int group_moments(const T* X, int64_t ldx, const T* y, const int64_t* offsets, int64_t n_groups, int p,
                  const GroupWork& wl, DevBag& bag, double** part, cudaStream_t s);
// K17 grouped lin_reg_report: for every group [offsets[g], offsets[g+1]) of [X | y] (null rows NaN), the 8 x q block of
// pl_lin_reg_report on its kept rows, out [n_groups][8][q] f64, and status [n_groups] (PDSB_GATED: fewer kept rows than
// coefficients, the block is NaN).  ymask (nullable): per-row 0 / 1, the y validity, for var(y).  se_type 0..4.
template <typename T>
int grouped_report(const T* X, int64_t ldx, const T* y, const T* ymask, const int64_t* offsets, int64_t n_groups,
                   int64_t n, int p, int add_bias, int se_type, double* out, int* status, cudaStream_t s);

// K19 grouped lin_reg_w_rcond: for every group [offsets[g], offsets[g+1]) of [X | y] (null rows NaN), K3's RCOND fit on
// its kept rows with the tolerance max(rcond, eps_T max(len_g, q)), rcond = o.tol rounded to T.  beta and sv
// [n_groups][q] f64 (sv descending), status [n_groups] (PDSB_GATED: fewer kept rows than coefficients, both NaN).
// o: add_bias, l2_reg, tol.  1 <= p <= 64.
template <typename T>
int grouped_lin_reg_rcond(const T* X, int64_t ldx, const T* y, const int64_t* offsets, int64_t n_groups, int64_t n,
                          int p, const pdsb_solve_opts& o, double* beta, double* sv, int* status, cudaStream_t s);

// K16 grouped logistic_reg (f64): every group's Newton / IRLS fit of host_logistic in one launch sequence.  X, y, mask
// (nullable, per-row 0 / 1) in group order, offsets device [n_groups + 1].  beta [n_groups x (p + add_bias)] (the last
// accepted iterate, NaN for a failed or empty group), status [n_groups] (pdsb_logistic_status), *n_iter (host,
// nullable): the iterations the call ran.
int grouped_logistic(const double* X, int64_t ldx, const double* y, const double* mask, const int64_t* offsets,
                     int64_t n_groups, int64_t n, int p, int add_bias, double l1, double l2, double tol,
                     int64_t max_iter, double* beta, int* status, int64_t* n_iter, cudaStream_t s);
// every group's GLM.fit (k16_grouped_logistic.cu): offsets on the device, outputs on the device, n_iter per group
int grouped_glm(const double* X, int64_t ldx, const double* y, const double* mask, const int64_t* offsets,
                int64_t n_groups, int64_t n, int p, int add_bias, int family, double tol, int64_t max_iter, double* beta,
                int* status, int64_t* n_iter, cudaStream_t s);

// K5 pass 1 for MixedModel on the work list wl: per-item moments of [X | y | 1] with every row shifted by its group's
// first row (generic kernel, p <= 64, f64; NaN rows are kept).  part: [(p+2)(p+3)/2][wl.n_items].
int group_moments_shifted(const double* X, int64_t ldx, const double* y, const int64_t* offsets, int64_t n_groups, int p,
                          const GroupWork& wl, double* part, cudaStream_t s);

// K12 MixedModel (random-intercept REML) on [X | y] in group order, column-major with leading dimension ld.
// out: coeffs[p], std_errors[p], dfs[p], gamma, resid_variance, evaluations, status (PDSB_MIXED_*), all f64.
enum { PDSB_MIXED_OK = 0, PDSB_MIXED_NOT_PD = 1, PDSB_MIXED_RESID_VAR = 2 };
int mixed_reml(const double* Z, int64_t ld, const int64_t* offsets, int64_t n_groups, int64_t n, int p,
               const uint8_t* between /* device, p flags */, int64_t max_iter, double tol, double* out, cudaStream_t s);
// stable sort of the rows by code: sorted codes and the row map; then offsets[g] = first sorted row of group g
int mixed_order_rows(const int64_t* codes, int64_t n, int64_t n_groups, int64_t* rows, int64_t* offsets, cudaStream_t s);

// K6/K7 rolling + recursive
template <typename T>
int online_lin_reg(const T* X, int64_t ldx, const T* y, int64_t n, int p, int add_bias, int64_t window,
                   int64_t min_rows, int skip, double lambda, const double* m0 /* moments of the preceding rows or null */,
                   int64_t row0 /* global index of row 0 */, T* coeffs, T* pred, uint8_t* valid, cudaStream_t s);
// recursive_lin_reg(...).over(key): group g = rows [offsets[g], offsets[g+1]) (device offsets), skip [n_groups] device
// flags or null; per group, bit for bit online_lin_reg (window 0, no m0, row0 0) on the group's rows
template <typename T>
int grouped_recursive_lin_reg(const T* X, int64_t ldx, const T* y, const int64_t* offsets, const uint8_t* skip,
                              int64_t n_groups, int64_t n, int p, int add_bias, int64_t min_rows, double lambda,
                              T* coeffs, T* pred, uint8_t* valid, cudaStream_t s);
// rolling_lin_reg(...).over(key): per group, bit for bit online_lin_reg (window >= 1, skip[g], no m0, row0 0) on the
// group's rows; window < 1 is refused
template <typename T>
int grouped_rolling_lin_reg(const T* X, int64_t ldx, const T* y, const int64_t* offsets, const uint8_t* skip,
                            int64_t n_groups, int64_t n, int p, int add_bias, int64_t window, int64_t min_rows,
                            double lambda, T* coeffs, T* pred, uint8_t* valid, cudaStream_t s);
// pass-C kernel of the last online_lin_reg / grouped_recursive_lin_reg / grouped_rolling_lin_reg launch on this thread
// (pdsb_last_online_path)
int last_online_path();

// K10 dense-matrix callers (model classes): strided gather to column-major, strided predict, Woodbury update
// dst[c * ld + r] = src[(rows ? rows[r] : r) * rs + c * cs]: the transpose, with the rows in the order of `rows` if given
int gather_colmajor(const double* src, int64_t rs, int64_t cs, int64_t n, int p, const int64_t* rows, double* dst,
                    int64_t ld, cudaStream_t s);
// inv_link: a pdsb_glm_family; out = g^-1(X beta + bias) with that family's canonical link (GAUSSIAN = identity)
int predict_strided(const double* X, int64_t rs, int64_t cs, int64_t n, int p, const double* beta, int has_bias,
                    double* out, cudaStream_t s, int inv_link = PDSB_GLM_GAUSSIAN);
int woodbury_update(double* inv, double* w, int q, int has_bias, const double* x, double y, double c, cudaStream_t s);

// K11 IRLS row pass of logistic_reg and GLM.fit (X column-major, ld ldx): w and z for every row, 0 where mask (nullable)
// is 0.  family: PDSB_IRLS_LOGISTIC (clamped weight; per-block log-loss partials in loss_parts, their count in
// *n_parts <= irls_max_parts()) or a pdsb_glm_family (loss_parts and n_parts unused).  ymean != null (GLM only): first
// iteration, mu_0 from y and *ymean (device), beta unused; otherwise eta = X beta (+ bias).
enum { PDSB_IRLS_LOGISTIC = -1 };
int irls_max_parts();
int irls_rows(int family, const double* X, int64_t ldx, const double* y, const double* mask, int64_t n, int p,
              int add_bias, const double* beta, const double* ymean, double* w, double* z, double* loss_parts,
              int* n_parts, cudaStream_t s);

// K13 PCA.  pca_eigen: eigen-decomposition of G = M[0:p, 0:p] (M: q1 x q1 moments, count at [q1-1][q1-1]); sigma[p] and
// V (p x p column-major) sorted descending and sign-fixed; status[0] = PDSB_PCA_*, status[1] = min(count, p).
enum { PDSB_PCA_OK = 0, PDSB_PCA_NONFINITE = 1 };
int pca_eigen(const double* M, int q1, int p, double* sigma, double* V, int* status, cudaStream_t s);
// out[:, j] = X V[:, j] for j < k (f64; out column-major with leading dimension ldo)
template <typename T>
int pca_project(const T* X, int64_t ldx, int64_t n, int p, const double* V, int k, double* out, int64_t ldo,
                cudaStream_t s);
// K18 grouped PCA (k18_grouped_pca.cu).  Group g is rows [offsets[g], offsets[g+1]) of X (device offsets); mask
// (nullable): per-row 0 / 1, a masked row leaves its group's Gram and a masked NaN is a null for the means.  center: the
// Gram of x - mean_g, mean [n_groups][p] written.  sigma [n_groups][p], V [n_groups][p x p] (column r = weight vector r),
// status [n_groups][2] as pca_eigen's.  1 <= p <= 64.
template <typename T>
int grouped_pca(const T* X, int64_t ldx, const T* mask, const int64_t* offsets, int64_t n_groups, int64_t n, int p,
                int center, double* mean, double* sigma, double* V, int* status, cudaStream_t s);
// out[j * ldo + r] = (x_r - mean_g) V_g[:, j] for j < k and every row r of group g (mean nullable: no centring); NaN for
// every row of a group with fewer than k rows
template <typename T>
int grouped_project(const T* X, int64_t ldx, const int64_t* offsets, int64_t n_groups, int64_t n, int p,
                    const double* mean, const double* V, int k, double* out, int64_t ldo, cudaStream_t s);
// Y[:, c] = (double) X[:, c], c < p
int widen_f32(const float* X, int64_t ldx, int64_t n, int p, double* Y, int64_t ldy, cudaStream_t s);

// K14 smooth spline.  g = the smoothing spline of (x, y) at lambda > 0 (lambda == 0: the input checks, then g = y).
// status[0]: 0 or PDSB_SPLINE_* bits (NONFINITE only when lambda > 0; then g is all NaN).  reduced_blocks (nullable):
// 2 x 2 blocks in all reduced levels together.
enum { PDSB_SPLINE_NOT_INCREASING = 1, PDSB_SPLINE_NONFINITE = 2 };
int smooth_spline_solve(const double* x, const double* y, int64_t n, double lam, double* g, int* status,
                        int64_t* reduced_blocks, cudaStream_t s);

// K15 isotonic regression.  out = the least-squares non-decreasing (increasing != 0) or non-increasing fit of y with
// weights w (nullable: all 1).  status[0]: 0 or PDSB_ISO_* bits; when != 0, out is all NaN.  n == 0 only clears status.
enum { PDSB_ISO_NONPOSITIVE_WEIGHT = 1, PDSB_ISO_NONFINITE = 2 };
int64_t isotonic_scratch_bytes(int64_t n);
int isotonic_fit(const double* y, const double* w, int64_t n, int increasing, double* out, int* status, cudaStream_t s);
// Per group g (rows [offsets[g], offsets[g+1]), device offsets), bit for bit isotonic_fit on the group's rows alone;
// status [n_groups], one word per group.  The group's partitions and tree start at its own first row (k15_isotonic.cu).
int grouped_isotonic_fit(const double* y, const double* w, const int64_t* offsets, int64_t n_groups, int64_t n,
                         int increasing, double* out, int* status, cudaStream_t s);

// K9 report
template <typename T>
int report_stats(const T* X, int64_t ldx, const T* y, const T* w, const T* mask, int64_t n, int p,
                 int add_bias, int se_type, double y_var, double* out, cudaStream_t s);

}  // namespace pdsb
