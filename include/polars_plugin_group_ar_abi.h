/*
 * polars_plugin_group_ar_abi.h — expression-plugin symbols of libpds_b200 for grouped autoregression:
 * `df.group_by(key).agg(pds.query_ar_coeffs(x, lag))` in one launch sequence for all groups, where Polars would call pl_lr
 * once per group on x.shift(i).slice(lag).  Like pl_lr_by (polars_plugin_group_abi.h), the caller hands over the rows
 * sorted by key and the group offsets, but only the one column x: the lagged columns are formed on the device, inside
 * each group.  Same calling convention as polars_plugin_abi.h.
 */
#ifndef POLARS_PLUGIN_GROUP_AR_ABI_H
#define POLARS_PLUGIN_GROUP_AR_ABI_H

#include "polars_plugin_abi.h"

#ifdef __cplusplus
extern "C" {
#endif

#define PDSB_DECLARE_GROUP_AR_EXPR(name)                                                                   \
  void _polars_plugin_##name(SeriesExport* inputs, size_t n_inputs, const uint8_t* kwargs, size_t kwargs_len, \
                             SeriesExport* ret, void* ctx);                                              \
  void _polars_plugin_field_##name(struct ArrowSchema* in_fields, size_t n, struct ArrowSchema* out);

/* inputs: offsets (one non-null Int64 chunk, n_groups + 1 entries: 0, ..., n), then x, with the rows of group g at
 * [offsets[g], offsets[g+1]).  kwargs: pl_lr's {"bias", "null_policy", "l1_reg", "l2_reg", "solver", "tol", "max_iter",
 * "weighted", "positive", "singular_x_tol"} plus "lag" (1 to 64).
 * pl_ar_coeffs_by(_f32) -> pl_lr(_f32)'s List<T>, one row per group: per group, what pl_lr_by(_f32) returns for the
 *                          group on its lagged columns (target x.slice(lag), features x.shift(1..lag).slice(lag), each
 *                          taken within the group), the lags in order and the bias last; null for a group with fewer
 *                          kept rows than coefficients.  Null policy: "raise" fails on any null; "skip" drops every row
 *                          a null reaches; a fill drops row t when x_t is null and fills x_t where it is a lag. */
PDSB_DECLARE_GROUP_AR_EXPR(pl_ar_coeffs_by)
PDSB_DECLARE_GROUP_AR_EXPR(pl_ar_coeffs_by_f32)

#ifdef __cplusplus
}
#endif
#endif
