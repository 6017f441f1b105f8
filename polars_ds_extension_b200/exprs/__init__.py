from .expr_spline import smooth_spline  # noqa: F401
