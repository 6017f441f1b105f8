/*
 * polars_plugin_group_recursive_abi.h — expression-plugin symbols of libpds_b200 for grouped recursive least squares:
 * `pds.recursive_lin_reg(...).over(key)` in one launch sequence for all groups, where Polars would call pl_recursive_lr
 * once per group.  Like pl_lr_pred_by (polars_plugin_group_abi.h), the caller hands over the rows sorted by key and the
 * group offsets.  Same calling convention as polars_plugin_abi.h.
 */
#ifndef POLARS_PLUGIN_GROUP_RECURSIVE_ABI_H
#define POLARS_PLUGIN_GROUP_RECURSIVE_ABI_H

#include "polars_plugin_abi.h"

#ifdef __cplusplus
extern "C" {
#endif

#define PDSB_DECLARE_GROUP_RECURSIVE_EXPR(name)                                                          \
  void _polars_plugin_##name(SeriesExport* inputs, size_t n_inputs, const uint8_t* kwargs, size_t kwargs_len, \
                             SeriesExport* ret, void* ctx);                                              \
  void _polars_plugin_field_##name(struct ArrowSchema* in_fields, size_t n, struct ArrowSchema* out);

/* inputs: offsets (one non-null Int64 chunk, n_groups + 1 entries: 0, ..., n), then y and the features, with the rows of
 * group g at [offsets[g], offsets[g+1]).  kwargs: pl_recursive_lr's {"null_policy", "n" (start_with), "bias", "lambda",
 * "min_size"}.
 * pl_recursive_lr_by(_f32) -> pl_recursive_lr(_f32)'s struct {coeffs: List<T>, pred: T}, one row per input row in the
 *                             input's (key) order: per group, bit for bit what pl_recursive_lr(_f32) returns on that
 *                             group's rows, nulls included.  The single call's checks run group by group in group order,
 *                             and the first failure fails the whole call with that call's message. */
PDSB_DECLARE_GROUP_RECURSIVE_EXPR(pl_recursive_lr_by)
PDSB_DECLARE_GROUP_RECURSIVE_EXPR(pl_recursive_lr_by_f32)

#ifdef __cplusplus
}
#endif
#endif
