"""CPU-side checks of group_by().agg(lin_reg_w_rcond) on the device that are particular to it: the schema twins are a
LargeList of pl_lr_w_rcond's struct; the fast path sends [offsets, y, x...] with the kwargs unchanged; over(fast=True)
is still refused; and without a GPU the Frame call fails loudly.  The checks every batched symbol shares (exports,
declaration, symbol list, entries, input messages, routing) are in test_grouped_abi_cpu.py."""
import numpy as np
import pyarrow as pa
import pytest

import polars_ds_extension_b200 as pds
import polars_ds_extension_b200.config as cfg
from polars_ds_extension_b200 import _harness
from tests.helpers import capture_plugin, has_gpu


@pytest.mark.parametrize("f32", [False, True])
def test_field_twin_is_a_large_list_of_the_single_call_struct(f32):
    sfx = "_f32" if f32 else ""
    f = _harness.field_of(f"pl_lr_w_rcond_by{sfx}")
    single = _harness.field_of(f"pl_lr_w_rcond{sfx}").type
    assert f.type == pa.large_list(pa.field("item", single))
    T = pa.float32() if f32 else pa.float64()
    assert [single.field(i).name for i in range(single.num_fields)] == ["coeffs", "singular_values"]
    assert all(single.field(i).type == pa.large_list(pa.field("item", T)) for i in range(2))


@pytest.mark.parametrize("f64", [True, False])
def test_fast_agg_sends_offsets_y_x_and_the_kwargs_unchanged(monkeypatch, f64):
    monkeypatch.setattr(cfg, "LIN_REG_EXPR_F64", f64)
    calls = capture_plugin(monkeypatch, pa.array([None, None], type=pa.large_list(
        pa.struct([("coeffs", pa.large_list(pa.float64()))]))))
    df = pds.Frame({"a": np.arange(8.0), "b": np.arange(8.0) ** 2, "y": np.arange(8.0) % 3, "g": np.arange(8) % 2})
    e = pds.lin_reg_w_rcond("a", "b", target="y", add_bias=True, rcond=-1e-3, l2_reg=0.5, null_policy="skip")
    df.group_by("g").agg(e, fast=True)
    (symbol, inputs, names, kwargs), = calls
    assert symbol == "pl_lr_w_rcond_by" + ("" if f64 else "_f32")
    assert names == ["__offsets__", "y", "a", "b"]
    assert kwargs == e.kwargs
    assert kwargs["tol"] == 1e-3 and kwargs["l2_reg"] == 0.5 and kwargs["bias"] and kwargs["null_policy"] == "skip"
    assert inputs[0].to_pylist() == [0, 4, 8]
    assert inputs[1].type == (pa.float64() if f64 else pa.float32())
    assert inputs[1].to_pylist() == [0.0, 2.0, 1.0, 0.0, 1.0, 0.0, 2.0, 1.0]       # y's rows in group order
    assert inputs[2].to_pylist() == [0.0, 2.0, 4.0, 6.0, 1.0, 3.0, 5.0, 7.0]


def test_over_fast_and_other_symbols_are_still_refused():
    df = pds.Frame({"a": np.arange(6.0), "w": np.ones(6), "y": np.arange(6.0) % 2, "g": np.arange(6) % 2})
    with pytest.raises(ValueError, match="fast over is only available for lin_reg predictions"):
        pds.lin_reg_w_rcond("a", target="y").over("g", fast=True)
    with pytest.raises(ValueError, match="fast group_by is only available for lin_reg coefficients.*lin_reg_w_rcond"):
        df.group_by("g").agg(pds.rolling_lin_reg("a", target="y", window_size=3), fast=True)


@pytest.mark.skipif(has_gpu(), reason="checks the loud failure on a box without a GPU")
@pytest.mark.parametrize("sym", ["pl_lr_w_rcond_by", "pl_lr_w_rcond_by_f32"])
def test_well_formed_call_fails_loudly_without_gpu(monkeypatch, sym):
    monkeypatch.setattr(cfg, "LIN_REG_EXPR_F64", not sym.endswith("_f32"))
    df = pds.Frame({"x1": np.arange(10.0), "y": np.arange(10.0) % 3, "g": np.arange(10) % 2})
    with pytest.raises(pds.PdsbError, match="no CPU fallback"):
        df.group_by("g").agg(pds.lin_reg_w_rcond("x1", target="y", add_bias=True), fast=True)
