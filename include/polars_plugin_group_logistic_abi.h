/*
 * polars_plugin_group_logistic_abi.h — expression-plugin symbols of libpds_b200 for grouped logistic regression:
 * `df.group_by(key).agg(pds.logistic_reg(...))` and `pds.logistic_reg(..., return_pred=True).over(key)` in one launch
 * sequence for all groups, where Polars would call pl_logistic_coeffs / pl_logistic_pred once per group.  Like pl_lr_by
 * (polars_plugin_abi.h), the caller hands over the rows sorted by key and the group offsets.  Same calling convention
 * as polars_plugin_abi.h.
 */
#ifndef POLARS_PLUGIN_GROUP_LOGISTIC_ABI_H
#define POLARS_PLUGIN_GROUP_LOGISTIC_ABI_H

#include "polars_plugin_abi.h"

#ifdef __cplusplus
extern "C" {
#endif

#define PDSB_DECLARE_GROUP_LOGISTIC_EXPR(name)                                                           \
  void _polars_plugin_##name(SeriesExport* inputs, size_t n_inputs, const uint8_t* kwargs, size_t kwargs_len, \
                             SeriesExport* ret, void* ctx);                                              \
  void _polars_plugin_field_##name(struct ArrowSchema* in_fields, size_t n, struct ArrowSchema* out);

/* inputs: offsets (one non-null Int64 chunk, n_groups + 1 entries: 0, ..., n), y (0/1), features... with the rows of
 * group g at [offsets[g], offsets[g+1]); kwargs: LRKwargs, as pl_logistic_coeffs.  Float64 only.  For every group, what
 * pl_logistic_coeffs / pl_logistic_pred return on that group's rows alone: every null policy, and "Empty data" when a
 * group keeps no row.
 * pl_logistic_by      -> List<Float64> "coeffs", one row per group (bias last); a list of NaN, never null, for a fit
 *                        that failed (a NaN or inf in a kept row).
 * pl_logistic_pred_by -> Float64 "pred", the probability of every input row in the sorted order; null for a row that
 *                        null_policy="skip" dropped, NaN for every other row of a failed group. */
PDSB_DECLARE_GROUP_LOGISTIC_EXPR(pl_logistic_by)
PDSB_DECLARE_GROUP_LOGISTIC_EXPR(pl_logistic_pred_by)

#ifdef __cplusplus
}
#endif
#endif
