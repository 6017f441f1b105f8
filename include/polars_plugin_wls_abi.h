/*
 * polars_plugin_wls_abi.h — expression-plugin symbols of libpds_b200 for batched weighted least squares:
 * `df.group_by(key).agg(pds.lin_reg(..., weights=w))` and `pds.lin_reg(..., weights=w, return_pred=True).over(key)` in
 * one launch sequence, where Polars would call pl_lr / pl_lr_pred once per group.  The batched calling convention of
 * polars_plugin_group_abi.h: the caller hands over the rows sorted by key and the group offsets as input 0; a per-row
 * result is in that sorted order.  Same calling convention as polars_plugin_abi.h.
 */
#ifndef POLARS_PLUGIN_WLS_ABI_H
#define POLARS_PLUGIN_WLS_ABI_H

#include "polars_plugin_abi.h"

#ifdef __cplusplus
extern "C" {
#endif

/* inputs: offsets (one non-null Int64 chunk, n_groups + 1 entries: 0, ..., n), w, y, features... with the rows of group g
 * at [offsets[g], offsets[g+1]); kwargs: LRKwargs, as pl_lr, with "weighted" set (a call without it is refused: the
 * unweighted fit is pl_lr_by's).  Per group, what pl_lr / pl_lr_pred with weights return on that group's rows: the
 * fit of the weighted normal equations (no ridge, no rank gate; l1_reg, l2_reg, positive and singular_x_tol are ignored
 * as the single weighted call ignores them; "svd" runs pivoted QR).  The call fails with the single call's message of the
 * first group, in key order, at which Polars' loop would stop (a short weight column, "raise" with a null, and the single
 * call's row count from the weights when "skip" or a fill masks a row of the group).  As pl_lr_by: a NaN / inf in a kept
 * row (x, y or w) drops the row, a null weight and, under "ignore", a null y or feature arrive as NaN and drop their row
 * too, and a group with fewer kept rows than coefficients, an empty group included, is null.
 * pl_wls_by      -> List<Float64> "coeffs" (List<Float32> for the _f32 twin), one row per group, bias last.
 * pl_wls_pred_by -> Struct {pred, resid} of Float64 (Float32), one row per input row: pred = [x | 1] beta_g and the
 *                   unweighted resid = y - pred.  A row is null when the single call masks it, and every row of a group
 *                   whose coefficients pl_wls_by returns as null. */
PDSB_DECLARE_EXPR(pl_wls_by)
PDSB_DECLARE_EXPR(pl_wls_by_f32)
PDSB_DECLARE_EXPR(pl_wls_pred_by)
PDSB_DECLARE_EXPR(pl_wls_pred_by_f32)

#ifdef __cplusplus
}
#endif

#endif /* POLARS_PLUGIN_WLS_ABI_H */
