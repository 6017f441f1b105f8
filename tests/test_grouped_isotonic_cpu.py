"""CPU-side checks of isotonic_regression(...).over(key) on the device: the pl_isotonic_regression_by schema twin, the
fast path sends [offsets, y (, w)] in group order with the expression's kwargs, the group_by refusal still holds, and
without a GPU the call fails loudly."""
import numpy as np
import pyarrow as pa
import pytest

import polars_ds_extension_b200 as pds
from polars_ds_extension_b200 import _harness
from tests.helpers import capture_plugin, has_gpu

REFUSED_AGG = "fast group_by is only available for lin_reg coefficients"
REFUSED_OVER = "fast over is only available for lin_reg predictions"


@pytest.mark.parametrize("weighted", [False, True])
def test_field_is_float64_named_after_y(weighted):
    ins = [pa.field("__offsets__", pa.int64()), pa.field("target", pa.float64())]
    if weighted:
        ins.append(pa.field("w", pa.float64()))
    f = _harness.field_of("pl_isotonic_regression_by", ins)
    assert f.type == pa.float64() and f.name == "target"
    single = _harness.field_of("pl_isotonic_regression", ins[1:])
    assert single.type == f.type and single.name == f.name


def _frame():
    return pds.Frame({"y": np.arange(8.0) ** 2, "w": np.arange(1.0, 9.0), "g": np.array([1, 0, 1, 0, 1, 0, 1, 0])})


@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("increasing", [True, False])
def test_fast_over_sends_offsets_args_and_kwargs(monkeypatch, weighted, increasing):
    calls = capture_plugin(monkeypatch, pa.array(np.arange(8.0)))
    e = pds.isotonic_regression("y", "w" if weighted else None, increasing=increasing)
    before = (e.symbol, list(e.args), dict(e.kwargs), e.over_key, e.over_fast)
    out = _frame().select(e.over("g", fast=True))["pl_isotonic_regression"]
    assert (e.symbol, list(e.args), dict(e.kwargs), e.over_key, e.over_fast) == before    # e itself is unchanged
    (symbol, inputs, names, kwargs), = calls
    assert symbol == "pl_isotonic_regression_by"
    assert names == ["__offsets__", "y"] + (["w"] if weighted else [])
    assert kwargs == {"has_weights": weighted, "increasing": increasing}
    assert inputs[0].to_pylist() == [0, 4, 8]
    assert inputs[1].type == pa.float64()
    assert inputs[1].to_pylist() == [0.0, 4.0, 16.0, 36.0, 1.0, 9.0, 25.0, 49.0]     # stable group order
    if weighted:
        assert inputs[2].to_pylist() == [1.0, 3.0, 5.0, 7.0, 2.0, 4.0, 6.0, 8.0]
    # the per-row results go back to the frame's row order: row r of group order is frame row order[r]
    order = [0, 2, 4, 6, 1, 3, 5, 7]
    back = out.to_pylist()
    assert [back[order[r]] for r in range(8)] == list(np.arange(8.0))


def test_integer_columns_are_cast_before_the_call(monkeypatch):
    calls = capture_plugin(monkeypatch, pa.array(np.zeros(6)))
    df = pds.Frame({"y": np.arange(6), "w": np.ones(6, dtype=np.float32), "g": np.arange(6) % 2})
    df.select(pds.isotonic_regression("y", "w").over("g", fast=True))
    (_, inputs, _, _), = calls
    assert inputs[1].type == pa.float64() and inputs[2].type == pa.float64()


def test_refusals():
    df = pds.Frame({"y": np.arange(6.0), "g": np.arange(6) % 2})
    with pytest.raises(ValueError, match=REFUSED_AGG):
        df.group_by("g").agg(pds.isotonic_regression("y"), fast=True)
    with pytest.raises(ValueError, match=REFUSED_OVER):
        pds.smooth_spline("y", "y", 1.0).over("g", fast=True)


@pytest.mark.skipif(has_gpu(), reason="checks the loud failure on a box without a GPU")
def test_fails_loudly_without_gpu():
    df = pds.Frame({"y": np.arange(10.0), "w": np.ones(10), "g": np.arange(10) % 2})
    with pytest.raises(pds.PdsbError, match="no CPU fallback"):
        df.select(pds.isotonic_regression("y", "w").over("g", fast=True))
