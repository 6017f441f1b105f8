"""Host-side mirror of the reference's PCA expression builders (/root/reference/python/polars_ds/exprs/num.py:369-463)
and of its isotonic regression (num.py:1106-1136).

Same names, arguments, defaults and validation; the same symbols and inputs cross the plugin ABI: the features (centred
as ``f - f.mean()`` when ``center``), preceded for ``principal_components`` by ``pl.lit(k, dtype=pl.UInt32)``.  The
PCA symbols take no kwargs.  The results are always Float64.

``isotonic_regression`` sends ``y`` (and the weights, if given) cast to Float64 with the kwargs
``{"has_weights": ..., "increasing": ...}``; the result is Float64 with the input's length.
"""
from __future__ import annotations

from typing import Optional, Union

from ..frame import ColExpr, PluginExpr, col, lit_u32

__all__ = ["singular_values", "pca", "principal_components", "isotonic_regression"]

ExprLike = Union[str, ColExpr]


def to_expr(f: ExprLike) -> ColExpr:
    if isinstance(f, str):
        return col(f)
    if isinstance(f, ColExpr):
        return f
    raise ValueError("Input can only be a column name or a column expression.")


def _inputs(features, center: bool):
    feats = [to_expr(f) for f in features]
    return [f.center() for f in feats] if center else feats


def singular_values(
    *features: ExprLike,
    center: bool = True,
    as_explained_var: bool = False,
    as_ratio: bool = False,
) -> PluginExpr:
    """All singular values of the matrix of `features` in descending order; rows with a null are dropped.
    `as_explained_var`: singular_value ^ 2 / (n - 1) as the reference's list.eval computes it (n = the number of values);
    `as_ratio`: normalised to sum to 1."""
    post = (("explained_var",) if as_explained_var else ()) + (("ratio",) if as_ratio else ())
    return PluginExpr("pl_singular_values", _inputs(features, center), None, returns_scalar=True, list_post=post)


def pca(*features: ExprLike, center: bool = True) -> PluginExpr:
    """Singular values and the principal (weight) vectors: a struct of min(n, p) rows {singular_value, weight_vector}."""
    return PluginExpr("pl_pca", _inputs(features, center), None, changes_length=True, pass_name_to_apply=True)


def principal_components(*features: ExprLike, k: int = 2, center: bool = True) -> PluginExpr:
    """The first k principal components of every row (a struct pc1..pck); NaN when there are fewer rows than `k`."""
    if k > len(features) or k <= 0:
        raise ValueError("Input `k` should be between 1 and the number of features inclusive.")
    return PluginExpr("pl_principal_components", [lit_u32(k)] + _inputs(features, center), None,
                      pass_name_to_apply=True)


def isotonic_regression(y: ExprLike, weights: Optional[ExprLike] = None, increasing: bool = True) -> PluginExpr:
    """The least-squares monotone fit of `y` (the same as scipy.optimize.isotonic_regression): non-decreasing if
    `increasing`, else non-increasing.  `weights` (positive) weight each row's squared error.  The device runs
    pool-adjacent-violators on partitions and joins them with a tree of merges that pool only around each junction."""
    args = [to_expr(y).cast("f64")]
    has_weights = weights is not None
    if has_weights:
        args.append(to_expr(weights).cast("f64"))
    return PluginExpr("pl_isotonic_regression", args, {"has_weights": has_weights, "increasing": increasing})
