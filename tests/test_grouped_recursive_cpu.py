"""CPU-side checks of recursive_lin_reg(...).over(key) on the device: the pl_recursive_lr_by schema twins, the fast path
sends [offsets, y, x...] in group order with the expression's kwargs, the f32 expression calls the f32 symbol, the
rolling refusal still holds, and without a GPU the call fails loudly."""
import numpy as np
import pyarrow as pa
import pytest

import polars_ds_extension_b200 as pds
import polars_ds_extension_b200.config as cfg
from polars_ds_extension_b200 import _harness
from tests.helpers import capture_plugin, has_gpu

REFUSED_OVER = "fast over is only available for lin_reg predictions"
REFUSED_AGG = "fast group_by is only available for lin_reg coefficients"
KWARGS = {"null_policy": "skip", "n": 3, "bias": True, "lambda": 0.5, "min_size": 0}


@pytest.mark.parametrize("sfx", ["", "_f32"])
def test_field_equals_the_single_calls(sfx):
    ins = [pa.field("y", pa.float64()), pa.field("x0", pa.float64()), pa.field("x1", pa.float64())]
    by = _harness.field_of(f"pl_recursive_lr_by{sfx}", [pa.field("__offsets__", pa.int64())] + ins)
    single = _harness.field_of(f"pl_recursive_lr{sfx}", ins)
    assert by.type == single.type and by.name == single.name
    t = pa.float32() if sfx else pa.float64()
    assert by.type == pa.struct([pa.field("coeffs", pa.large_list(t)), pa.field("pred", t)])


def _frame():
    return pds.Frame({"y": np.arange(8.0) ** 2, "a": np.arange(8.0), "b": np.arange(8, dtype=np.int64) % 3,
                      "g": np.array([1, 0, 1, 0, 1, 0, 1, 0])})


def _result(n, f32=False):
    t = pa.float32() if f32 else pa.float64()
    return pa.StructArray.from_arrays([pa.array([[float(i)] for i in range(n)], type=pa.large_list(t)),
                                       pa.array(np.arange(float(n)), type=t)], names=["coeffs", "pred"])


@pytest.mark.parametrize("f64", [True, False])
def test_fast_over_sends_offsets_args_and_kwargs(monkeypatch, f64):
    monkeypatch.setattr(cfg, "LIN_REG_EXPR_F64", f64)
    calls = capture_plugin(monkeypatch, _result(8, not f64))
    e = pds.recursive_lin_reg("a", "b", target="y", start_with=3, add_bias=True, l2_reg=-0.5, null_policy="skip")
    before = (e.symbol, list(e.args), dict(e.kwargs), e.over_key, e.over_fast)
    out = _frame().select(e.over("g", fast=True))[e.symbol]
    assert (e.symbol, list(e.args), dict(e.kwargs), e.over_key, e.over_fast) == before    # e itself is unchanged
    (symbol, inputs, names, kwargs), = calls
    assert symbol == "pl_recursive_lr_by" + ("" if f64 else "_f32")
    assert names == ["__offsets__", "y", "a", "b"]
    assert kwargs == KWARGS == e.kwargs
    assert inputs[0].to_pylist() == [0, 4, 8]
    assert inputs[1].type == (pa.float64() if f64 else pa.float32())              # the target is cast, as in the single call
    assert inputs[1].to_pylist() == [0.0, 4.0, 16.0, 36.0, 1.0, 9.0, 25.0, 49.0]     # stable group order
    assert inputs[2].to_pylist() == [0.0, 2.0, 4.0, 6.0, 1.0, 3.0, 5.0, 7.0]
    assert inputs[3].type == pa.int64() and inputs[3].to_pylist() == [0, 2, 1, 0, 1, 0, 2, 1]
    # the per-row results go back to the frame's row order: row r of group order is frame row order[r]
    order = [0, 2, 4, 6, 1, 3, 5, 7]
    back = out.field("pred").to_pylist()
    assert [back[order[r]] for r in range(8)] == list(np.arange(8.0))


def test_refusals():
    df = pds.Frame({"y": np.arange(6.0), "a": np.arange(6.0), "g": np.arange(6) % 2})
    with pytest.raises(ValueError, match=REFUSED_OVER) as ei:
        pds.rolling_lin_reg("a", target="y", window_size=3).over("g", fast=True)
    assert "recursive_lin_reg" in str(ei.value)
    with pytest.raises(ValueError, match=REFUSED_AGG):
        df.group_by("g").agg(pds.recursive_lin_reg("a", target="y", start_with=2), fast=True)


@pytest.mark.skipif(has_gpu(), reason="checks the loud failure on a box without a GPU")
@pytest.mark.parametrize("sfx", ["", "_f32"])
def test_fails_loudly_without_gpu(monkeypatch, sfx):
    monkeypatch.setattr(cfg, "LIN_REG_EXPR_F64", not sfx)          # the expression calls pl_recursive_lr_by{sfx}
    df = pds.Frame({"y": np.arange(10.0), "a": np.ones(10), "g": np.arange(10) % 2})
    with pytest.raises(pds.PdsbError, match="no CPU fallback"):
        df.select(pds.recursive_lin_reg("a", target="y", start_with=2).over("g", fast=True))
