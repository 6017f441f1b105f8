/*
 * polars_plugin_num_abi.h — expression-plugin symbols of libpds_b200 outside the lin_reg family: the PCA expressions of
 * the reference's num_ext module (src/num_ext/pca.rs:39-182; wrappers python/polars_ds/exprs/num.py:369-463) and its
 * smoothing spline (src/num_ext/splines.rs; wrapper python/polars_ds/exprs/expr_spline.py) and its isotonic regression
 * (src/num_ext/isotonic_regression.rs; wrapper python/polars_ds/exprs/num.py:1106-1136).
 * Same calling convention as polars_plugin_abi.h.  The PCA symbols take no kwargs (Polars passes an empty buffer);
 * pl_smooth_spline takes {"lambda": float}; pl_isotonic_regression takes {"has_weights": bool, "increasing": bool}.
 */
#ifndef POLARS_PLUGIN_NUM_ABI_H
#define POLARS_PLUGIN_NUM_ABI_H

#include "polars_plugin_abi.h"

#ifdef __cplusplus
extern "C" {
#endif

/* inputs: features...                -> List<f64> "singular_values", min(rows, features) values, descending  (:39)  */
PDSB_DECLARE_EXPR(pl_singular_values)
/* inputs: k (UInt32 literal), features... -> Struct "principal_components" {pc1..pck: f64}, one row per input row (:80) */
PDSB_DECLARE_EXPR(pl_principal_components)
/* inputs: features...                -> Struct "pca" {singular_value: f64, weight_vector: List<f64>}, one row per value (:126) */
PDSB_DECLARE_EXPR(pl_pca)
/* inputs: x, y (Float64); kwargs {"lambda": float} -> Float64, one value per input row (src/num_ext/splines.rs:99) */
PDSB_DECLARE_EXPR(pl_smooth_spline)
/* inputs: y (, w when has_weights) (Float64); kwargs {"has_weights": bool, "increasing": bool} -> Float64, one value per
 * input row (src/num_ext/isotonic_regression.rs) */
PDSB_DECLARE_EXPR(pl_isotonic_regression)

#ifdef __cplusplus
}
#endif
#endif
