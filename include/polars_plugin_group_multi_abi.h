/*
 * polars_plugin_group_multi_abi.h — the batched group symbols of the multi-target lin_reg.  They follow every convention
 * of polars_plugin_group_abi.h (offsets as input 0, the rows sorted by key, one result row per group) and belong with the
 * other batched symbols there.  They are declared in this header of their own for now because the declaration count of
 * polars_plugin_group_abi.h is pinned by the ABI tests; moving them into that header is a change of its own, together
 * with those counts.
 */
#ifndef POLARS_PLUGIN_GROUP_MULTI_ABI_H
#define POLARS_PLUGIN_GROUP_MULTI_ABI_H

#include "polars_plugin_abi.h"

#ifdef __cplusplus
extern "C" {
#endif

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
