"""polars_ds_extension_b200 — B200-native engine behind the polars_ds `lin_reg` expression family.

The product is the shared library `_polars_ds_b200.so` (hand-written sm_90a CUDA behind the Polars plugin C ABI and
the `pdsb_*` C API, see include/).  This package holds the host-side mirror of the reference's Python wrappers
(`pds.lin_reg`, `logistic_reg`, `simple_lin_reg`, `lin_reg_report`, `rolling_lin_reg`, `recursive_lin_reg`, `lin_reg_w_rcond`,
`singular_values`, `pca`, `principal_components`, `smooth_spline`, `isotonic_regression`), the
numpy-facing model classes (`linear_models.LR / ElasticNet / OnlineLR / GLM / MixedModel`) and a Polars-free harness that calls the plugin
symbols exactly the way Polars does.
"""
from . import config  # noqa: F401
from .exprs.expr_linear import (  # noqa: F401
    lin_reg,
    lin_reg_report,
    lin_reg_w_rcond,
    linear_impute,
    logistic_reg,
    query_ar_coeffs,
    recursive_lin_reg,
    rolling_lin_reg,
    simple_lin_reg,
)
from .exprs.num import isotonic_regression, pca, principal_components, singular_values  # noqa: F401
from .exprs.expr_spline import smooth_spline  # noqa: F401
from .frame import Frame, col  # noqa: F401
from ._lib import PdsbError, lib  # noqa: F401

__version__ = "0.1.0"
