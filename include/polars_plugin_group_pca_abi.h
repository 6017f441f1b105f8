/*
 * polars_plugin_group_pca_abi.h — expression-plugin symbols of libpds_b200 for grouped PCA:
 * `df.group_by(key).agg(pds.singular_values(...))`, `df.group_by(key).agg(pds.pca(...))` and
 * `pds.principal_components(...).over(key)` in one launch sequence for all groups, where Polars would call
 * pl_singular_values / pl_pca / pl_principal_components once per group.  Like pl_lr_by (polars_plugin_abi.h), the caller
 * hands over the rows sorted by key and the group offsets.  Same calling convention as polars_plugin_abi.h.
 */
#ifndef POLARS_PLUGIN_GROUP_PCA_ABI_H
#define POLARS_PLUGIN_GROUP_PCA_ABI_H

#include "polars_plugin_abi.h"

#ifdef __cplusplus
extern "C" {
#endif

#define PDSB_DECLARE_GROUP_PCA_EXPR(name)                                                                \
  void _polars_plugin_##name(SeriesExport* inputs, size_t n_inputs, const uint8_t* kwargs, size_t kwargs_len, \
                             SeriesExport* ret, void* ctx);                                              \
  void _polars_plugin_field_##name(struct ArrowSchema* in_fields, size_t n, struct ArrowSchema* out);

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
PDSB_DECLARE_GROUP_PCA_EXPR(pl_singular_values_by)
PDSB_DECLARE_GROUP_PCA_EXPR(pl_pca_by)
PDSB_DECLARE_GROUP_PCA_EXPR(pl_principal_components_by)

#ifdef __cplusplus
}
#endif
#endif
