/*
 * polars_plugin_group_rcond_abi.h — the batched group symbols of lin_reg_w_rcond.  They follow every convention of
 * polars_plugin_group_abi.h (offsets as input 0, the rows sorted by key, one result row per group) and belong with the
 * other batched symbols there.  They are declared in this header of their own for now because the declaration count of
 * polars_plugin_group_abi.h is pinned by the ABI tests; moving them into that header is a change of its own, together
 * with those counts.
 */
#ifndef POLARS_PLUGIN_GROUP_RCOND_ABI_H
#define POLARS_PLUGIN_GROUP_RCOND_ABI_H

#include "polars_plugin_abi.h"

#ifdef __cplusplus
extern "C" {
#endif

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

#ifdef __cplusplus
}
#endif
#endif
