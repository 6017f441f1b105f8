/*
 * polars_plugin_group_isotonic_abi.h — expression-plugin symbol of libpds_b200 for grouped isotonic regression:
 * `pds.isotonic_regression(...).over(key)` in one launch sequence for all groups, where Polars would call
 * pl_isotonic_regression once per group.  Like pl_lr_pred_by (polars_plugin_group_abi.h), the caller hands over the rows
 * sorted by key and the group offsets.  Same calling convention as polars_plugin_abi.h.
 */
#ifndef POLARS_PLUGIN_GROUP_ISOTONIC_ABI_H
#define POLARS_PLUGIN_GROUP_ISOTONIC_ABI_H

#include "polars_plugin_abi.h"

#ifdef __cplusplus
extern "C" {
#endif

#define PDSB_DECLARE_GROUP_ISOTONIC_EXPR(name)                                                           \
  void _polars_plugin_##name(SeriesExport* inputs, size_t n_inputs, const uint8_t* kwargs, size_t kwargs_len, \
                             SeriesExport* ret, void* ctx);                                              \
  void _polars_plugin_field_##name(struct ArrowSchema* in_fields, size_t n, struct ArrowSchema* out);

/* inputs: offsets (one non-null Int64 chunk, n_groups + 1 entries: 0, ..., n), then y (Float64) and, with
 * {"has_weights": true}, w (Float64), with the rows of group g at [offsets[g], offsets[g+1]).  kwargs: {"has_weights":
 * bool, "increasing": bool}, as pl_isotonic_regression.
 * pl_isotonic_regression_by -> Float64, one row per input row in the input's (key) order: per group, bit for bit what
 *                              pl_isotonic_regression returns on that group's rows (a one-row group is y as given, a null
 *                              included; a group with a non-finite y or w is all NaN).  A null y or w, or a w <= 0, in a
 *                              group of >= 2 rows fails the whole call, checked over all groups in that order.  The
 *                              schema twin declares Float64 under the name of input 1 (y). */
PDSB_DECLARE_GROUP_ISOTONIC_EXPR(pl_isotonic_regression_by)

#ifdef __cplusplus
}
#endif
#endif
