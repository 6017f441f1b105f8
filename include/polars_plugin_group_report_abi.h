/*
 * polars_plugin_group_report_abi.h — expression-plugin symbols of libpds_b200 for the grouped OLS report:
 * `df.group_by(key).agg(pds.lin_reg_report(...))` in one launch sequence for all groups, where Polars would call
 * pl_lin_reg_report once per group.  Like pl_lr_by (polars_plugin_abi.h), the caller hands over the rows sorted by key
 * and the group offsets.  Same calling convention as polars_plugin_abi.h.
 */
#ifndef POLARS_PLUGIN_GROUP_REPORT_ABI_H
#define POLARS_PLUGIN_GROUP_REPORT_ABI_H

#include "polars_plugin_abi.h"

#ifdef __cplusplus
extern "C" {
#endif

#define PDSB_DECLARE_GROUP_REPORT_EXPR(name)                                                             \
  void _polars_plugin_##name(SeriesExport* inputs, size_t n_inputs, const uint8_t* kwargs, size_t kwargs_len, \
                             SeriesExport* ret, void* ctx);                                              \
  void _polars_plugin_field_##name(struct ArrowSchema* in_fields, size_t n, struct ArrowSchema* out);

/* inputs: offsets (one non-null Int64 chunk, n_groups + 1 entries: 0, ..., n), y, features... with the rows of group g
 * at [offsets[g], offsets[g+1]); no var(y) input: each group's variance of its non-null y is computed on the device.
 * kwargs: pl_lin_reg_report's (bias, null_policy, std_err, ...).  Nulls only with null_policy="skip"; no weights; at
 * most 64 features.
 * pl_lin_reg_report_by (_f32) -> LargeList<Struct{features, beta, <std_err | hc0_se .. hc3_se>, t, p>|t|, 0.025,
 *                                0.975, r2, adj_r2}>, one list of (features + bias) structs per group: what
 *                                pl_lin_reg_report returns on that group's rows, Float64 (Float32) fields.  A null list
 *                                for a group with fewer kept rows than coefficients (an empty group included).  A NaN in
 *                                a kept row drops that row from its group's fit, as pl_lr_by does. */
PDSB_DECLARE_GROUP_REPORT_EXPR(pl_lin_reg_report_by)
PDSB_DECLARE_GROUP_REPORT_EXPR(pl_lin_reg_report_by_f32)

#ifdef __cplusplus
}
#endif
#endif
