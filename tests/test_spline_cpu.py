"""CPU checks of smooth_spline: the dense restatement of the reference against the long-double band solve and SciPy's
make_smoothing_spline, lambda = 0, linear data, the non-finite cases of the dense form, the wrapper, the schema twin,
the required kwarg and the loud failure without a GPU."""
import numpy as np
import pyarrow as pa
import pytest

import polars_ds_extension_b200 as pds
from polars_ds_extension_b200 import _harness
from polars_ds_extension_b200.frame import Frame
from tests import spline_oracle as so
from tests.helpers import has_gpu


def _xs(n, kind, seed):
    x = np.linspace(0.0, 10.0, n)
    if kind == "jitter":
        x = x + np.random.default_rng(seed).uniform(-0.3, 0.3, n) * (10.0 / (n - 1))
    return x


CASES = [(n, kind, lam) for n in (5, 37, 200, 500) for kind in ("even", "jitter") for lam in (1e-3, 1e-1, 10.0, 100.0)]


@pytest.mark.parametrize("n,kind,lam", CASES)
def test_dense_band_and_scipy_agree(n, kind, lam):
    from scipy.interpolate import make_smoothing_spline

    x = _xs(n, kind, n)
    y = np.sin(x) + 0.1 * np.random.default_rng(n + 1).standard_normal(n)
    g_ld = so.reinsch_ld(x, y, lam)
    assert so.rel_err(so.dense_smooth_spline(x, y, lam), g_ld, y) < 1e-8
    assert so.rel_err(so.reinsch_f64(x, y, lam), g_ld, y) < 1e-8
    assert so.rel_err(make_smoothing_spline(x, y, lam=lam)(x), g_ld, y) < 1e-8


@pytest.mark.parametrize("n", [3, 4, 5])
def test_smallest_inputs(n):
    x = np.array([0.0, 0.7, 1.9, 2.2, 4.0])[:n]
    y = np.array([1.0, -2.0, 0.5, 3.0, 1.5])[:n]
    for lam in (1e-3, 1.0, 1e3):
        g = so.dense_smooth_spline(x, y, lam)
        assert so.rel_err(g, so.reinsch_ld(x, y, lam), y) < 1e-10
        assert so.rel_err(so.reinsch_f64(x, y, lam), so.reinsch_ld(x, y, lam), y) < 1e-12


def test_lambda_zero_returns_y():
    x = _xs(40, "jitter", 3)
    y = np.cos(x)
    for f in (so.dense_smooth_spline, so.reinsch_ld, so.reinsch_f64):
        np.testing.assert_array_equal(f(x, y, 0.0), y)


@pytest.mark.parametrize("lam", [1e-6, 1e-2, 1.0, 1e2, 1e6])
def test_linear_data_is_in_the_null_space(lam):
    x = _xs(300, "jitter", 5)
    y = 2.5 - 0.75 * x
    # the dense form rounds Q R^-1 Q' y (exactly 0) to ~eps lambda / h^3 relative: loose for it, tight for the band form
    assert so.rel_err(so.dense_smooth_spline(x, y, lam), y, y) < 1e-10 * max(1.0, lam)
    for f in (so.reinsch_ld, so.reinsch_f64):
        assert so.rel_err(f(x, y, lam), y, y) < 1e-12


def test_errors_in_the_reference_order():
    with pytest.raises(so.SplineError, match="Input x or y has nulls."):
        so.dense_smooth_spline([0.0, None, 2.0], [1.0, 2.0], 1.0)
    with pytest.raises(so.SplineError, match="Input lengths are not the same."):
        so.dense_smooth_spline([0.0, 1.0, 2.0], [1.0, 2.0], 1.0)
    with pytest.raises(so.SplineError, match="Must have >= 3 points."):
        so.dense_smooth_spline([0.0, 1.0], [1.0, 2.0], 1.0)
    for x in ([0.0, 1.0, 1.0, 2.0], [0.0, 2.0, 1.0, 3.0]):
        with pytest.raises(so.SplineError, match="Input is not increasing."):
            so.dense_smooth_spline(x, [1.0, 2.0, 3.0, 4.0], 0.0)


def test_non_finite_inputs_of_the_dense_form():
    """What the dense restatement gives: a NaN or inf y, or a NaN x, makes every output NaN (M^-1 is dense).  An
    infinite x at either end passes the increasing check and gives finite values: the device returns all NaN there
    (DESIGN §5)."""
    x = np.linspace(0.0, 10.0, 40)
    y = np.sin(x)
    for lam in (1e-3, 1.0):
        for bad in (np.nan, np.inf, -np.inf):
            yb = y.copy()
            yb[7] = bad
            assert np.isnan(so.dense_smooth_spline(x, yb, lam)).all()
        xb = x.copy()
        xb[10] = np.nan
        assert np.isnan(so.dense_smooth_spline(xb, y, lam)).all()
        xb = x.copy()
        xb[-1] = np.inf
        assert np.isfinite(so.dense_smooth_spline(xb, y, lam)).all()


def test_wrapper_symbol_inputs_and_validation():
    e = pds.smooth_spline("x", "y", 0.5)
    assert e.symbol == "pl_smooth_spline" and e.kwargs == {"lambda": 0.5}
    assert [a.name for a in e.args] == ["x", "y"]
    assert all(a.cast_to == "f64" and a.rechunked for a in e.args)
    assert not e.returns_scalar and not e.changes_length
    assert pds.smooth_spline(pds.col("a"), "b", 0.0).kwargs == {"lambda": 0.0}
    with pytest.raises(ValueError, match="Input `lambda_` must be nonnegative."):
        pds.smooth_spline("x", "y", -1e-9)
    from polars_ds_extension_b200.exprs import smooth_spline

    assert smooth_spline is pds.smooth_spline


def test_wrapper_casts_integer_and_float32_columns():
    f = Frame({"x": pa.array([1, 2, 4], type=pa.int32()), "y": pa.array([1.0, 2.0, 5.0], type=pa.float32())})
    e = pds.smooth_spline("x", "y", 1.0)
    xs = f._eval_arg(e.args[0])
    ys = f._eval_arg(e.args[1])
    assert xs.type == pa.float64() and ys.type == pa.float64() and xs.num_chunks == 1


def test_schema_twin_is_float64():
    f = _harness.field_of("pl_smooth_spline", [pa.field("x", pa.float64()), pa.field("y", pa.float64())])
    assert f.type == pa.float64() and f.name == "x"
    assert set(_harness.SPLINE_SYMBOLS).isdisjoint(_harness.PLUGIN_SYMBOLS + _harness.PCA_SYMBOLS)


def test_missing_lambda_kwarg_is_an_error():
    x = pa.chunked_array([pa.array([0.0, 1.0, 2.0])])
    with pytest.raises(pds.PdsbError, match="kwargs: missing field `lambda`"):
        _harness.call_plugin("pl_smooth_spline", [x, x], ["x", "y"], {})


@pytest.mark.skipif(has_gpu(), reason="checks the loud failure on a box without a GPU")
def test_spline_symbol_fails_loudly_without_gpu():
    df = Frame({"x": np.linspace(0.0, 1.0, 20), "y": np.arange(20.0)})
    with pytest.raises(pds.PdsbError, match="no CPU fallback"):
        df.select(pds.smooth_spline("x", "y", 1.0))
