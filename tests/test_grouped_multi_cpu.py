"""CPU-side checks of group_by().agg(lin_reg(target=[...])) on the device that are particular to it: the schema twins
are pl_lr_multi's; the fast path sends [offsets, target_0.., x...] with pl_lr_multi's kwargs unchanged; the plugin
layer checks last_target_idx; the multi-target predictions stay refused under over(fast=True); and without a GPU the
Frame call fails loudly.  The checks every batched symbol shares (exports, declaration, symbol list, entries, input
messages, routing) are in test_grouped_abi_cpu.py."""
import numpy as np
import pyarrow as pa
import pytest

import polars_ds_extension_b200 as pds
import polars_ds_extension_b200.config as cfg
from polars_ds_extension_b200 import _harness
from tests.helpers import capture_plugin, has_gpu

SYMBOLS = ["pl_lr_multi_by", "pl_lr_multi_by_f32"]
KW = {"bias": True, "null_policy": "raise", "solver": "qr", "last_target_idx": 2, "l2_reg": 0.0,
      "singular_x_tol": 1e-12}
OFFSETS = pa.array(np.array([0, 5, 10], dtype=np.int64))


def _col(f32, k=0):
    return pa.array((np.arange(10) * (k + 1) % 3).astype(np.float32 if f32 else np.float64))


@pytest.mark.parametrize("f32", [False, True])
def test_field_twin_is_the_single_calls(f32):
    sfx = "_f32" if f32 else ""
    f = _harness.field_of(f"pl_lr_multi_by{sfx}")
    assert f == _harness.field_of(f"pl_lr_multi{sfx}")
    assert f.name == "coeffs" and f.type == pa.large_list(pa.field("item", pa.float32() if f32 else pa.float64()))


@pytest.mark.parametrize("f64", [True, False])
def test_fast_agg_sends_offsets_targets_x_and_the_kwargs_unchanged(monkeypatch, f64):
    monkeypatch.setattr(cfg, "LIN_REG_EXPR_F64", f64)
    calls = capture_plugin(monkeypatch,
                           pa.array([None, None], type=pa.struct([("target_0", pa.large_list(pa.float64()))])))
    df = pds.Frame({"a": np.arange(8.0), "b": np.arange(8.0) ** 2, "y": np.arange(8) % 3, "z": -np.arange(8.0),
                    "g": np.arange(8) % 2})
    e = pds.lin_reg("a", "b", target=["y", "z"], add_bias=True, l2_reg=0.5, solver="choleskey", null_policy="zero")
    df.group_by("g").agg(e, fast=True)
    (symbol, inputs, names, kwargs), = calls
    assert symbol == "pl_lr_multi_by" + ("" if f64 else "_f32")
    assert names == ["__offsets__", "target_0", "target_1", "a", "b"]
    assert kwargs == e.kwargs
    assert kwargs["last_target_idx"] == 2 and kwargs["l2_reg"] == 0.5 and kwargs["solver"] == "choleskey"
    assert kwargs["bias"] and kwargs["null_policy"] == "zero"
    assert inputs[0].to_pylist() == [0, 4, 8]
    T = pa.float64() if f64 else pa.float32()
    assert inputs[1].type == T and inputs[2].type == T                 # the targets are cast, as pl_lr_multi's are
    assert inputs[1].to_pylist() == [0.0, 2.0, 1.0, 0.0, 1.0, 0.0, 2.0, 1.0]       # y's rows in group order
    assert inputs[2].to_pylist() == [-0.0, -2.0, -4.0, -6.0, -1.0, -3.0, -5.0, -7.0]
    assert inputs[3].to_pylist() == [0.0, 2.0, 4.0, 6.0, 1.0, 3.0, 5.0, 7.0]
    assert inputs[4].to_pylist() == [0.0, 4.0, 16.0, 36.0, 1.0, 9.0, 25.0, 49.0]


def _fails_with(sym, inputs, names, msg, kw=KW):
    with pytest.raises(pds.PdsbError) as ei:
        _harness.call_plugin(sym, inputs, names, kw)
    assert str(ei.value) == f"the plugin failed with message: {msg}"


@pytest.mark.parametrize("t", [0, -1, 3, 4])
@pytest.mark.parametrize("sym", SYMBOLS)
def test_last_target_idx_out_of_range(sym, t):
    f32 = sym.endswith("_f32")
    _fails_with(sym, [OFFSETS, _col(f32), _col(f32, 1), _col(f32, 2)], ["__offsets__", "target_0", "target_1", "x1"],
                "last_target_idx out of range", dict(KW, last_target_idx=t))


def test_missing_multi_kwarg():
    _fails_with("pl_lr_multi_by", [OFFSETS, _col(False), _col(False, 1), _col(False, 2)],
                ["__offsets__", "target_0", "target_1", "x1"], "kwargs: missing field `last_target_idx`",
                {k: v for k, v in KW.items() if k != "last_target_idx"})


def test_multi_target_predictions_and_other_symbols_stay_refused():
    df = pds.Frame({"a": np.arange(6.0), "y": np.arange(6.0) % 2, "z": np.arange(6.0), "g": np.arange(6) % 2})
    with pytest.raises(ValueError, match="fast over is only available for lin_reg predictions"):
        pds.lin_reg("a", target=["y", "z"], return_pred=True).over("g", fast=True)
    with pytest.raises(ValueError, match="fast over is only available for lin_reg predictions"):
        pds.lin_reg("a", target=["y", "z"]).over("g", fast=True)
    with pytest.raises(ValueError, match="fast group_by is only available for lin_reg coefficients.*lin_reg_w_rcond"):
        df.group_by("g").agg(pds.lin_reg("a", target=["y", "z"], return_pred=True), fast=True)


@pytest.mark.skipif(has_gpu(), reason="checks the loud failure on a box without a GPU")
@pytest.mark.parametrize("sym", SYMBOLS)
def test_well_formed_call_fails_loudly_without_gpu(monkeypatch, sym):
    monkeypatch.setattr(cfg, "LIN_REG_EXPR_F64", not sym.endswith("_f32"))
    df = pds.Frame({"x1": np.arange(10.0), "y": np.arange(10.0) % 3, "z": np.arange(10.0) % 4, "g": np.arange(10) % 2})
    with pytest.raises(pds.PdsbError, match="no CPU fallback"):
        df.group_by("g").agg(pds.lin_reg("x1", target=["y", "z"], add_bias=True), fast=True)
