/*
 * polars_plugin_group_abi.h — expression-plugin symbols of libpds_b200 for grouped lin_reg predictions:
 * `pds.lin_reg(*x, target=y, return_pred=True).over(key)` in one launch sequence for all groups, where Polars would call
 * pl_lr_pred once per group.  Like pl_lr_by (polars_plugin_abi.h), the caller hands over the rows sorted by key and the
 * group offsets; the result is per row, in that sorted order, and the caller puts it back in the frame's row order.
 * Same calling convention as polars_plugin_abi.h.
 */
#ifndef POLARS_PLUGIN_GROUP_ABI_H
#define POLARS_PLUGIN_GROUP_ABI_H

#include "polars_plugin_abi.h"

#ifdef __cplusplus
extern "C" {
#endif

#define PDSB_DECLARE_GROUP_EXPR(name)                                                                    \
  void _polars_plugin_##name(SeriesExport* inputs, size_t n_inputs, const uint8_t* kwargs, size_t kwargs_len, \
                             SeriesExport* ret, void* ctx);                                              \
  void _polars_plugin_field_##name(struct ArrowSchema* in_fields, size_t n, struct ArrowSchema* out);

/* inputs: offsets (one non-null Int64 chunk, n_groups + 1 entries: 0, ..., n), y, features... with the rows of group g
 * at [offsets[g], offsets[g+1]); kwargs: LRKwargs, as pl_lr_pred (weighted fits are refused, nulls need "skip").
 * -> Struct {pred, resid} of Float64 (Float32 for the _f32 twin), one row per input row.  A row is null when one of its
 * inputs is null, and every row of a group is null when pl_lr_by returns that group's coefficients as null (rank gate,
 * fewer valid rows than coefficients).  A NaN value in a kept row gives NaN, not null. */
PDSB_DECLARE_GROUP_EXPR(pl_lr_pred_by)
PDSB_DECLARE_GROUP_EXPR(pl_lr_pred_by_f32)

#ifdef __cplusplus
}
#endif
#endif
