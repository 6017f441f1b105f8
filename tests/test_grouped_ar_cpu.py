"""CPU-side checks of group_by().agg(query_ar_coeffs(...), fast=True): the pl_ar_coeffs_by schema twins, the fast path
sends [offsets, x] in group order with pl_lr's kwargs plus "lag", the f32 expression calls the f32 symbol, a
hand-written lin_reg with the same arguments takes the same path, near misses with a shift or slice are refused, and
without a GPU the call fails loudly."""
import numpy as np
import pyarrow as pa
import pytest

import polars_ds_extension_b200 as pds
import polars_ds_extension_b200.config as cfg
from polars_ds_extension_b200 import _harness
from polars_ds_extension_b200 import frame as frame_mod
from polars_ds_extension_b200.frame import col
from tests.helpers import capture_plugin, has_gpu

REFUSED_SHIFT = "an argument with shift or slice is only batched as query_ar_coeffs"
REFUSED_OVER = "fast over is only available for lin_reg predictions"


@pytest.mark.parametrize("sfx", ["", "_f32"])
def test_field_equals_the_single_calls(sfx):
    by = _harness.field_of(f"pl_ar_coeffs_by{sfx}", [pa.field("__offsets__", pa.int64()), pa.field("x", pa.float64())])
    ins = [pa.field("x", pa.float64()), pa.field("1", pa.float64()), pa.field("2", pa.float64())]
    single = _harness.field_of(f"pl_lr{sfx}", ins)
    assert by.type == single.type and by.name == single.name
    assert by.type == pa.large_list(pa.float32() if sfx else pa.float64())


def _frame():
    # g = [1, 0, 1, 0, ...]: group 1 (first seen) holds the even rows, group 0 the odd ones
    return pds.Frame({"x": np.arange(10.0) ** 2, "z": np.arange(10.0), "g": np.arange(10) % 2 == 0})


def _capture(monkeypatch, n_groups, q, f32=False):
    t = pa.float32() if f32 else pa.float64()
    return capture_plugin(monkeypatch, pa.array([[float(g)] * q for g in range(n_groups)], type=pa.large_list(t)))


@pytest.mark.parametrize("f64", [True, False])
@pytest.mark.parametrize("lag,bias,policy", [(1, True, "raise"), (3, False, "zero"), (2, True, "0.5")])
def test_fast_agg_sends_offsets_x_and_kwargs(monkeypatch, f64, lag, bias, policy):
    monkeypatch.setattr(cfg, "LIN_REG_EXPR_F64", f64)
    calls = _capture(monkeypatch, 2, lag + bias, not f64)
    e = pds.query_ar_coeffs("x", lag=lag, add_bias=bias, null_policy=policy)
    before = (e.symbol, list(e.args), dict(e.kwargs))
    out = _frame().group_by("g").agg(e, fast=True)
    assert (e.symbol, list(e.args), dict(e.kwargs)) == before            # e itself is unchanged
    (symbol, inputs, names, kwargs), = calls
    assert symbol == "pl_ar_coeffs_by" + ("" if f64 else "_f32")
    assert names == ["__offsets__", "x"]
    assert kwargs == dict(e.kwargs, lag=lag) and set(kwargs) == set(e.kwargs) | {"lag"}
    assert inputs[0].to_pylist() == [0, 5, 10]
    assert inputs[1].type == (pa.float64() if f64 else pa.float32())    # cast as the target is, in the single call
    assert inputs[1].to_pylist() == [0.0, 4.0, 16.0, 36.0, 64.0, 1.0, 9.0, 25.0, 49.0, 81.0]    # stable group order
    assert list(out["g"]) == [True, False]
    assert out[e.out_name].to_pylist() == [[0.0] * (lag + bias), [1.0] * (lag + bias)]


def test_hand_written_lin_reg_takes_the_same_path(monkeypatch):
    monkeypatch.setattr(cfg, "LIN_REG_EXPR_F64", True)
    calls = _capture(monkeypatch, 2, 3)
    e = pds.lin_reg(*[col("x").shift(i).slice(2) for i in (1, 2)], target=col("x").slice(2), add_bias=True)
    _frame().group_by("g").agg(e, fast=True)
    (symbol, inputs, names, kwargs), = calls
    assert symbol == "pl_ar_coeffs_by" and names == ["__offsets__", "x"]
    assert kwargs == dict(e.kwargs, lag=2)
    assert frame_mod._ar_pattern(e) == ("x", "f64", 2)
    assert frame_mod._ar_pattern(pds.query_ar_coeffs("x", lag=5)) == ("x", "f64", 5)


def _near_misses():
    x = col("x")
    return {
        "lags not 1..L": pds.lin_reg(x.shift(2).slice(2), x.shift(1).slice(2), target=x.slice(2)),
        "a lag missing": pds.lin_reg(x.shift(1).slice(2), target=x.slice(2)),
        "two columns": pds.lin_reg(x.shift(1).slice(2), col("z").shift(2).slice(2), target=x.slice(2)),
        "an extra feature": pds.lin_reg(x.shift(1).slice(1), col("z").slice(1), target=x.slice(1)),
        "shift without slice": pds.lin_reg(x.shift(1), target=x),
        "slice of the wrong length": pds.lin_reg(x.shift(1).slice(2), target=x.slice(2).slice(1)),
        "weighted": pds.lin_reg(x.shift(1).slice(1), target=x.slice(1), weights="z"),
        "lin_reg_report": pds.lin_reg_report(x.shift(1).slice(1), target=x.slice(1)),
    }


@pytest.mark.parametrize("case", sorted(_near_misses()))
def test_near_misses_are_refused(monkeypatch, case):
    calls = _capture(monkeypatch, 2, 2)
    e = _near_misses()[case]
    assert frame_mod._ar_pattern(e) is None
    with pytest.raises(ValueError, match=REFUSED_SHIFT):
        _frame().group_by("g").agg(e, fast=True)
    assert calls == []


def test_shifted_arguments_are_refused_under_fast_over(monkeypatch):
    calls = _capture(monkeypatch, 2, 2)
    x = col("x")
    e = pds.lin_reg(x.shift(1), target=x, return_pred=True)
    with pytest.raises(ValueError, match=REFUSED_SHIFT):
        _frame().select(e.over("g", fast=True))
    with pytest.raises(ValueError, match=REFUSED_OVER):          # no over for the AR coefficients
        pds.query_ar_coeffs("x", lag=2).over("g", fast=True)
    assert calls == []


def test_unshifted_lin_reg_still_goes_to_pl_lr_by(monkeypatch):
    calls = _capture(monkeypatch, 2, 1)
    e = pds.lin_reg("z", target="x")
    assert frame_mod._ar_pattern(e) is None
    _frame().group_by("g").agg(e, fast=True)
    assert calls[0][0] == "pl_lr_by" and calls[0][2] == ["__offsets__", "x", "z"]


@pytest.mark.skipif(has_gpu(), reason="checks the loud failure on a box without a GPU")
@pytest.mark.parametrize("sfx", ["", "_f32"])
def test_fails_loudly_without_gpu(monkeypatch, sfx):
    monkeypatch.setattr(cfg, "LIN_REG_EXPR_F64", not sfx)          # the expression calls pl_ar_coeffs_by{sfx}
    with pytest.raises(pds.PdsbError, match="no CPU fallback"):
        _frame().group_by("g").agg(pds.query_ar_coeffs("x", lag=2), fast=True)
