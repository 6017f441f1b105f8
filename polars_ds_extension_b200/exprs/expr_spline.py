"""Host-side mirror of the reference's smoothing-spline expression builder (python/polars_ds/exprs/expr_spline.py).

Same name, arguments and validation; the same symbol and inputs cross the plugin ABI: ``x`` and ``y`` cast to Float64
and rechunked, with the kwargs ``{"lambda": lambda_}``.  The result is Float64 with the input's length.
"""
from __future__ import annotations

from typing import Union

from ..frame import ColExpr, PluginExpr, col

__all__ = ["smooth_spline"]

ExprLike = Union[str, ColExpr]


def to_expr(f: ExprLike) -> ColExpr:
    if isinstance(f, str):
        return col(f)
    if isinstance(f, ColExpr):
        return f
    raise ValueError("Input can only be a column name or a column expression.")


def smooth_spline(x: ExprLike, y: ExprLike, lambda_: float) -> PluginExpr:
    """Fits a smoothing cubic spline f and returns f(x).  x must be sorted and strictly increasing.

    `lambda_` is the regularization factor: the larger, the smoother the curve (0 interpolates, g = y).  The device
    solves the Reinsch band system (R + lambda Q'Q) gamma = Q'y, g = y - lambda Q gamma in O(n)."""
    if lambda_ < 0.0:
        raise ValueError("Input `lambda_` must be nonnegative.")
    xx, yy = to_expr(x), to_expr(y)
    return PluginExpr("pl_smooth_spline", [xx.cast("f64").rechunk(), yy.cast("f64").rechunk()],
                      {"lambda": lambda_})
