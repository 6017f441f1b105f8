/*
 * polars_plugin_group_abi.h — expression-plugin symbols of libpds_b200 for batched group calls: every group of an
 * `.over(key)` or a `group_by(key).agg(...)` in one launch sequence, where Polars would call the single-call symbol once
 * per group.  The caller hands over the rows sorted by key and the group offsets as input 0; a per-row result is in that
 * sorted order, and the caller puts it back in the frame's row order.  Same calling convention as polars_plugin_abi.h.
 */
#ifndef POLARS_PLUGIN_GROUP_ABI_H
#define POLARS_PLUGIN_GROUP_ABI_H

#include "polars_plugin_abi.h"

#ifdef __cplusplus
extern "C" {
#endif

/* ---- lin_reg: `df.group_by(key).agg(pds.lin_reg(...))`, where Polars would call pl_lr once per group ---- */
/* additive (ours): grouped fast path, input 0 = int64 group offsets (n_groups+1), then y, features...
 * returns List<T> with n_groups rows.  See SURVEY.md §7 H1 / §8f-2. */
PDSB_DECLARE_EXPR(pl_lr_by)
PDSB_DECLARE_EXPR(pl_lr_by_f32)

/* ---- lin_reg predictions: `pds.lin_reg(*x, target=y, return_pred=True).over(key)`, where Polars would call pl_lr_pred
 * once per group ---- */
/* inputs: offsets (one non-null Int64 chunk, n_groups + 1 entries: 0, ..., n), y, features... with the rows of group g
 * at [offsets[g], offsets[g+1]); kwargs: LRKwargs, as pl_lr_pred (weighted fits are refused, nulls need "skip").
 * -> Struct {pred, resid} of Float64 (Float32 for the _f32 twin), one row per input row.  A row is null when one of its
 * inputs is null, and every row of a group is null when pl_lr_by returns that group's coefficients as null (rank gate,
 * fewer valid rows than coefficients).  A NaN value in a kept row gives NaN, not null. */
PDSB_DECLARE_EXPR(pl_lr_pred_by)
PDSB_DECLARE_EXPR(pl_lr_pred_by_f32)

/* ---- logistic regression: `df.group_by(key).agg(pds.logistic_reg(...))` and
 * `pds.logistic_reg(..., return_pred=True).over(key)`, where Polars would call pl_logistic_coeffs / pl_logistic_pred once
 * per group ---- */
/* inputs: offsets (one non-null Int64 chunk, n_groups + 1 entries: 0, ..., n), y (0/1), features... with the rows of
 * group g at [offsets[g], offsets[g+1]); kwargs: LRKwargs, as pl_logistic_coeffs.  Float64 only.  For every group, what
 * pl_logistic_coeffs / pl_logistic_pred return on that group's rows alone: every null policy, and "Empty data" when a
 * group keeps no row.
 * pl_logistic_by      -> List<Float64> "coeffs", one row per group (bias last); a list of NaN, never null, for a fit
 *                        that failed (a NaN or inf in a kept row).
 * pl_logistic_pred_by -> Float64 "pred", the probability of every input row in the sorted order; null for a row that
 *                        null_policy="skip" dropped, NaN for every other row of a failed group. */
PDSB_DECLARE_EXPR(pl_logistic_by)
PDSB_DECLARE_EXPR(pl_logistic_pred_by)

/* ---- OLS report: `df.group_by(key).agg(pds.lin_reg_report(...))`, where Polars would call pl_lin_reg_report once per
 * group ---- */
/* inputs: offsets (one non-null Int64 chunk, n_groups + 1 entries: 0, ..., n), y, features... with the rows of group g
 * at [offsets[g], offsets[g+1]); no var(y) input: each group's variance of its non-null y is computed on the device.
 * kwargs: pl_lin_reg_report's (bias, null_policy, std_err, ...).  Nulls only with null_policy="skip"; no weights; at
 * most 64 features.
 * pl_lin_reg_report_by (_f32) -> LargeList<Struct{features, beta, <std_err | hc0_se .. hc3_se>, t, p>|t|, 0.025,
 *                                0.975, r2, adj_r2}>, one list of (features + bias) structs per group: what
 *                                pl_lin_reg_report returns on that group's rows, Float64 (Float32) fields.  A null list
 *                                for a group with fewer kept rows than coefficients (an empty group included).  A NaN in
 *                                a kept row drops that row from its group's fit, as pl_lr_by does. */
PDSB_DECLARE_EXPR(pl_lin_reg_report_by)
PDSB_DECLARE_EXPR(pl_lin_reg_report_by_f32)

/* ---- PCA: `df.group_by(key).agg(pds.singular_values(...))`, `df.group_by(key).agg(pds.pca(...))` and
 * `pds.principal_components(...).over(key)`, where Polars would call pl_singular_values / pl_pca /
 * pl_principal_components once per group ---- */
/* inputs: offsets (one non-null Int64 chunk, n_groups + 1 entries: 0, ..., n), then for principal_components the k
 * literal (UInt32, one row, not permuted), then the features, un-centred, with the rows of group g at
 * [offsets[g], offsets[g+1]).  kwargs: {"center": bool}: each group's columns are centred by their own means (over each
 * column's non-null values) on the device.  At most 64 features.  Per group, what the single-call symbol returns on that
 * group's (centred) rows; an error one group's call would raise is raised for the whole call.
 * pl_singular_values_by      -> LargeList<Float64>, one list of min(kept rows, features) values per group, descending
 *                               (rows with a null are dropped; an empty group gives an empty list).
 * pl_pca_by                  -> LargeList<Struct{singular_value: Float64, weight_vector: LargeList<Float64>}>, one list
 *                               of `features` structs per group; a group with fewer kept rows than features is an error.
 * pl_principal_components_by -> Struct{pc1..pck} of Float64 per row, in the input's (key) order; NaN for every row of a
 *                               group with fewer rows than k; nulls are an error.  The schema twin declares
 *                               pc1..pc{number of feature inputs}. */
PDSB_DECLARE_EXPR(pl_singular_values_by)
PDSB_DECLARE_EXPR(pl_pca_by)
PDSB_DECLARE_EXPR(pl_principal_components_by)

/* ---- isotonic regression: `pds.isotonic_regression(...).over(key)`, where Polars would call pl_isotonic_regression
 * once per group ---- */
/* inputs: offsets (one non-null Int64 chunk, n_groups + 1 entries: 0, ..., n), then y (Float64) and, with
 * {"has_weights": true}, w (Float64), with the rows of group g at [offsets[g], offsets[g+1]).  kwargs: {"has_weights":
 * bool, "increasing": bool}, as pl_isotonic_regression.
 * pl_isotonic_regression_by -> Float64, one row per input row in the input's (key) order: per group, bit for bit what
 *                              pl_isotonic_regression returns on that group's rows (a one-row group is y as given, a null
 *                              included; a group with a non-finite y or w is all NaN).  A null y or w, or a w <= 0, in a
 *                              group of >= 2 rows fails the whole call, checked over all groups in that order.  The
 *                              schema twin declares Float64 under the name of input 1 (y). */
PDSB_DECLARE_EXPR(pl_isotonic_regression_by)

/* ---- recursive least squares: `pds.recursive_lin_reg(...).over(key)`, where Polars would call pl_recursive_lr once
 * per group ---- */
/* inputs: offsets (one non-null Int64 chunk, n_groups + 1 entries: 0, ..., n), then y and the features, with the rows of
 * group g at [offsets[g], offsets[g+1]).  kwargs: pl_recursive_lr's {"null_policy", "n" (start_with), "bias", "lambda",
 * "min_size"}.
 * pl_recursive_lr_by(_f32) -> pl_recursive_lr(_f32)'s struct {coeffs: List<T>, pred: T}, one row per input row in the
 *                             input's (key) order: per group, bit for bit what pl_recursive_lr(_f32) returns on that
 *                             group's rows, nulls included.  The single call's checks run group by group in group order,
 *                             and the first failure fails the whole call with that call's message. */
PDSB_DECLARE_EXPR(pl_recursive_lr_by)
PDSB_DECLARE_EXPR(pl_recursive_lr_by_f32)

/* ---- autoregression: `df.group_by(key).agg(pds.query_ar_coeffs(x, lag))`, where Polars would call pl_lr once per
 * group on x.shift(i).slice(lag).  Only the one column x is handed over: the lagged columns are formed on the device,
 * inside each group ---- */
/* inputs: offsets (one non-null Int64 chunk, n_groups + 1 entries: 0, ..., n), then x, with the rows of group g at
 * [offsets[g], offsets[g+1]).  kwargs: pl_lr's {"bias", "null_policy", "l1_reg", "l2_reg", "solver", "tol", "max_iter",
 * "weighted", "positive", "singular_x_tol"} plus "lag" (1 to 64).
 * pl_ar_coeffs_by(_f32) -> pl_lr(_f32)'s List<T>, one row per group: per group, what pl_lr_by(_f32) returns for the
 *                          group on its lagged columns (target x.slice(lag), features x.shift(1..lag).slice(lag), each
 *                          taken within the group), the lags in order and the bias last; null for a group with fewer
 *                          kept rows than coefficients.  Null policy: "raise" fails on any null; "skip" drops every row
 *                          a null reaches; a fill drops row t when x_t is null and fills x_t where it is a lag. */
PDSB_DECLARE_EXPR(pl_ar_coeffs_by)
PDSB_DECLARE_EXPR(pl_ar_coeffs_by_f32)

/* ---- rank-revealing least squares: `df.group_by(key).agg(pds.lin_reg_w_rcond(...))`, where Polars would call
 * pl_lr_w_rcond once per group ---- */
/* inputs: offsets (one non-null Int64 chunk, n_groups + 1 entries: 0, ..., n), y, features... with the rows of group g
 * at [offsets[g], offsets[g+1]).  kwargs: pl_lr_w_rcond's (bias, null_policy, l1_reg, l2_reg, solver, tol = |rcond|).
 * Nulls only with null_policy="skip" ("raise" fails with "Nulls found in data"); no weights; at most 64 features.
 * pl_lr_w_rcond_by (_f32) -> LargeList<Struct{coeffs: List<Float64>, singular_values: List<Float64>}> (Float32 for the
 *                            _f32 twin), one list holding one struct per group: what pl_lr_w_rcond returns on that
 *                            group's rows, with that group's own tolerance max(rcond, eps * max(group rows, features +
 *                            bias)).  A null list for a group with fewer kept rows than coefficients (an empty group
 *                            included).  A NaN or inf in a kept row drops that row from its group's fit, as pl_lr_by
 *                            does. */
PDSB_DECLARE_EXPR(pl_lr_w_rcond_by)
PDSB_DECLARE_EXPR(pl_lr_w_rcond_by_f32)

/* ---- multi-target least squares: `df.group_by(key).agg(pds.lin_reg(..., target=[y_0, ..., y_{t-1}]))`, where Polars
 * would call pl_lr_multi once per group ---- */
/* inputs: offsets (one non-null Int64 chunk, n_groups + 1 entries: 0, ..., n), target_0 .. target_{t-1}, features...
 * with the rows of group g at [offsets[g], offsets[g+1]).  kwargs: pl_lr_multi's (bias, null_policy, solver,
 * last_target_idx = t, l2_reg, singular_x_tol) and its null rules and messages: "raise" fails on any null, every other
 * policy but a fill is refused, a fill refuses null targets and fills the features.  At most 65 targets and features
 * together.
 * pl_lr_multi_by (_f32) -> Struct{<target_0>: List<Float64>, ..., <target_{t-1}>: List<Float64>} (Float32 for the _f32
 *                          twin), one row per group: per target, what pl_lr_by returns for that target alone on the
 *                          group's rows (bit for bit, for finite data and p + t <= 11 or p >= 11).  All t lists are
 *                          null for a group whose fit is null: fewer kept rows than coefficients (an empty group
 *                          included), or a gated fit.  A NaN or inf in any value of a row drops that row from its group's
 *                          fit of every target.  The schema twins declare pl_lr_multi's (knowingly wrong) type. */
PDSB_DECLARE_EXPR(pl_lr_multi_by)
PDSB_DECLARE_EXPR(pl_lr_multi_by_f32)

#ifdef __cplusplus
}
#endif
#endif
