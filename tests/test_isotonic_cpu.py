"""CPU checks of isotonic_regression: the restatement of the reference against SciPy bit for bit, the long-double and
exact oracles, the reference's errors and passthrough, what the restatement gives on NaN and inf, the wrapper, the
schema twin, the required kwargs and the loud failure without a GPU."""
import numpy as np
import pyarrow as pa
import pytest
from scipy.optimize import isotonic_regression as sp_iso

import polars_ds_extension_b200 as pds
from polars_ds_extension_b200 import _harness
from polars_ds_extension_b200.frame import Frame
from tests import isotonic_oracle as io
from tests.helpers import has_gpu

SEEDS = range(40)


def _case(seed):
    rng = np.random.default_rng(seed)
    n = int(rng.integers(2, 600))
    kind = io.SHAPES[seed % len(io.SHAPES)]
    y = io.shape(kind, n, seed) if kind != "runs" else np.repeat(rng.integers(-3, 4, n // 7 + 1), 7)[:n] * 1.0
    w = rng.uniform(0.1, 3.0, n) if seed % 2 else None
    return y, w


@pytest.mark.parametrize("seed", SEEDS)
@pytest.mark.parametrize("increasing", [True, False])
def test_restatement_equals_scipy_bit_for_bit(seed, increasing):
    y, w = _case(seed)
    for ww in (w, None):
        np.testing.assert_array_equal(io.reference_pava(y, ww, increasing), sp_iso(y, weights=ww, increasing=increasing).x)


@pytest.mark.parametrize("seed", SEEDS)
@pytest.mark.parametrize("increasing", [True, False])
def test_long_double_oracles_agree_with_scipy(seed, increasing):
    y, w = _case(seed)
    ref = sp_iso(y, weights=w, increasing=increasing).x
    ld = io.pava_ld(y, w, increasing)
    assert io.rel_err(ref, ld, y) < 1e-13
    assert io.rel_err(io.blocks_ld(y, w, increasing), ld, y) < 1e-15
    assert np.all(np.diff(ld) >= 0) if increasing else np.all(np.diff(ld) <= 0)


@pytest.mark.parametrize("increasing", [True, False])
def test_exact_oracle_on_integer_data(increasing):
    rng = np.random.default_rng(5)
    y = rng.integers(-100, 100, 700)
    w = rng.integers(1, 10, 700)
    ex = io.exact_f64(y, w, increasing)
    assert io.rel_err(sp_iso(y.astype(float), weights=w.astype(float), increasing=increasing).x, ex, y) < 1e-14
    assert io.rel_err(io.pava_ld(y, w, increasing), ex, y) < 1e-16      # ex is rounded to f64


def test_errors_in_the_reference_order():
    with pytest.raises(io.IsotonicError, match="Input should not contain nulls."):
        io.reference_pava([1.0, None, 2.0], [1.0, 2.0])            # y's nulls come before the weights' length
    with pytest.raises(io.IsotonicError, match="must be the same length as y"):
        io.reference_pava([1.0, 0.0, 2.0], [1.0, None])
    with pytest.raises(io.IsotonicError, match="Weight should not contain nulls."):
        io.reference_pava([1.0, 0.0, 2.0], [1.0, None, -1.0])
    for w in ([1.0, 0.0, 2.0], [1.0, -2.0, 2.0]):
        with pytest.raises(io.IsotonicError, match="Weight should not contain negative values."):
            io.reference_pava([1.0, 0.0, 2.0], w)
    # a NaN weight passes the w <= 0 check
    io.reference_pava([1.0, 0.0, 2.0], [1.0, np.nan, 2.0])


def test_short_columns_pass_through():
    assert io.reference_pava([], None) == []
    assert io.reference_pava([None], [1.0, 2.0]) == [None]          # before any check
    assert io.reference_pava([3.5], [-1.0]) == [3.5]


def test_non_finite_in_the_restatement():
    """What the sequential loop gives; the device returns all NaN for any non-finite y or w instead (DESIGN §5)."""
    out = io.reference_pava([1.0, np.nan, 0.5, 2.0])
    np.testing.assert_array_equal(out, [1.0, np.nan, 0.5, 2.0])   # unchanged and not monotone
    out = io.reference_pava([1.0, np.inf, 0.5, 2.0, 3.0])
    np.testing.assert_array_equal(out, [1.0] + [np.inf] * 4)       # inf spreads to the rows after it
    out = io.reference_pava([0.0, 1.0, 2.0], [1.0, np.nan, 1.0])
    np.testing.assert_array_equal(out, [0.0, 1.0, 2.0])            # a NaN weight is never pooled here
    out = io.reference_pava([2.0, 1.0, 0.0], [1.0, np.nan, 1.0])
    np.testing.assert_array_equal(out, [np.nan, np.nan, 0.0])       # it poisons the pool it enters, and stops it


def test_wrapper_symbol_casts_and_kwargs():
    e = pds.isotonic_regression("y")
    assert e.symbol == "pl_isotonic_regression" and e.kwargs == {"has_weights": False, "increasing": True}
    assert [a.name for a in e.args] == ["y"] and e.args[0].cast_to == "f64"
    assert not e.returns_scalar and not e.changes_length
    e = pds.isotonic_regression(pds.col("a"), weights="w", increasing=False)
    assert e.kwargs == {"has_weights": True, "increasing": False}
    assert [a.name for a in e.args] == ["a", "w"] and all(a.cast_to == "f64" for a in e.args)
    from polars_ds_extension_b200.exprs.num import isotonic_regression

    assert isotonic_regression is pds.isotonic_regression
    f = Frame({"y": pa.array([3, 1, 2], type=pa.int32()), "w": pa.array([1.0, 2.0, 5.0], type=pa.float32())})
    assert all(f._eval_arg(a).type == pa.float64() for a in pds.isotonic_regression("y", "w").args)


def test_schema_twin_is_float64():
    f = _harness.field_of("pl_isotonic_regression", [pa.field("y", pa.float64())])
    assert f.type == pa.float64() and f.name == "y"
    f = _harness.field_of("pl_isotonic_regression", [pa.field("v", pa.float64()), pa.field("w", pa.float64())])
    assert f.type == pa.float64() and f.name == "v"
    others = _harness.PLUGIN_SYMBOLS + _harness.PCA_SYMBOLS + _harness.SPLINE_SYMBOLS
    assert set(_harness.ISOTONIC_SYMBOLS).isdisjoint(others)


@pytest.mark.parametrize("kw,missing", [({"increasing": True}, "has_weights"), ({"has_weights": False}, "increasing")])
def test_missing_kwarg_is_an_error(kw, missing):
    y = pa.chunked_array([pa.array([0.0, 1.0, 2.0])])
    with pytest.raises(pds.PdsbError, match=f"kwargs: missing field `{missing}`"):
        _harness.call_plugin("pl_isotonic_regression", [y], ["y"], kw)


@pytest.mark.skipif(has_gpu(), reason="checks the loud failure on a box without a GPU")
def test_isotonic_symbol_fails_loudly_without_gpu():
    df = Frame({"y": np.arange(20.0)[::-1].copy()})
    with pytest.raises(pds.PdsbError, match="no CPU fallback"):
        df.select(pds.isotonic_regression("y"))
