"""CPU-side checks of group_by().agg(lin_reg(target=[...])) on the device: pl_lr_multi_by and its f32 twin are exported
and declared once, in include/polars_plugin_group_multi_abi.h only; their schema twins are pl_lr_multi's; the host and
device entries are declared in pdsb.h; the fast path sends [offsets, target_0.., x...] with pl_lr_multi's kwargs
unchanged; the plugin layer's input checks give their exact messages; the multi-target predictions stay refused under
over(fast=True); and without a GPU the call fails loudly."""
import re
from pathlib import Path

import numpy as np
import pyarrow as pa
import pytest

import polars_ds_extension_b200 as pds
import polars_ds_extension_b200.config as cfg
from polars_ds_extension_b200 import _harness
from polars_ds_extension_b200 import frame as frame_mod
from polars_ds_extension_b200._lib import lib

ROOT = Path(__file__).resolve().parent.parent
MULTI_HEADER = ROOT / "include" / "polars_plugin_group_multi_abi.h"
SYMBOLS = ["pl_lr_multi_by", "pl_lr_multi_by_f32"]
ENTRIES = ["pdsb_host_grouped_lin_reg_multi", "pdsb_dev_grouped_lin_reg_multi_f32", "pdsb_dev_grouped_lin_reg_multi_f64"]
KW = {"bias": True, "null_policy": "raise", "solver": "qr", "last_target_idx": 2, "l2_reg": 0.0,
      "singular_x_tol": 1e-12}
OFFSETS = pa.array(np.array([0, 5, 10], dtype=np.int64))


def _has_gpu():
    try:
        import torch

        return torch.cuda.is_available()
    except Exception:
        return False


def _code(header):
    return re.sub(r"/\*.*?\*/", "", header.read_text(), flags=re.S)


def _col(f32, k=0):
    return pa.array((np.arange(10) * (k + 1) % 3).astype(np.float32 if f32 else np.float64))


def test_symbol_list():
    assert _harness.GROUPED_MULTI_SYMBOLS == SYMBOLS


@pytest.mark.parametrize("sym", SYMBOLS)
def test_symbol_and_twin_exported(sym):
    L = lib()
    assert hasattr(L, f"_polars_plugin_{sym}") and hasattr(L, f"_polars_plugin_field_{sym}"), sym


@pytest.mark.parametrize("sym", SYMBOLS)
def test_declared_once_in_the_multi_header_only(sym):
    assert re.findall(r"PDSB_DECLARE_EXPR\((\w+)\)", _code(MULTI_HEADER)).count(sym) == 1
    for h in sorted((ROOT / "include").glob("*.h")):
        if h != MULTI_HEADER:
            assert not re.search(rf"\b{sym}\b", _code(h)), (h.name, sym)


def test_the_multi_header_declares_nothing_else():
    assert sorted(re.findall(r"PDSB_DECLARE_EXPR\((\w+)\)", _code(MULTI_HEADER))) == SYMBOLS
    assert "rcond" not in MULTI_HEADER.read_text()


@pytest.mark.parametrize("sym", SYMBOLS)
def test_symbol_is_in_no_other_list(sym):
    others = (_harness.PLUGIN_SYMBOLS + _harness.PCA_SYMBOLS + _harness.SPLINE_SYMBOLS + _harness.ISOTONIC_SYMBOLS
              + _harness.GROUPED_SYMBOLS + _harness.GROUPED_RCOND_SYMBOLS)
    assert sym not in others and _harness.GROUPED_MULTI_SYMBOLS.count(sym) == 1


def test_host_and_device_entries_exported_and_declared():
    L = lib()
    pdsb_h = (ROOT / "include" / "pdsb.h").read_text()
    for fn in ENTRIES:
        assert hasattr(L, fn), fn
        assert f"int {fn}(" in pdsb_h, fn


@pytest.mark.parametrize("f32", [False, True])
def test_field_twin_is_the_single_calls(f32):
    sfx = "_f32" if f32 else ""
    f = _harness.field_of(f"pl_lr_multi_by{sfx}")
    assert f == _harness.field_of(f"pl_lr_multi{sfx}")
    assert f.name == "coeffs" and f.type == pa.large_list(pa.field("item", pa.float32() if f32 else pa.float64()))


def test_batched_symbol_table():
    assert frame_mod._by_group("pl_lr_multi", per_row=False) == "pl_lr_multi_by"
    assert frame_mod._by_group("pl_lr_multi_f32", per_row=False) == "pl_lr_multi_by"
    assert frame_mod._by_group("pl_lr_multi", per_row=True) is None
    assert frame_mod._by_group("pl_lr_multi_pred", per_row=True) is None
    assert frame_mod._by_group("pl_lr_multi_pred", per_row=False) is None


@pytest.mark.parametrize("f64", [True, False])
def test_fast_agg_sends_offsets_targets_x_and_the_kwargs_unchanged(monkeypatch, f64):
    monkeypatch.setattr(cfg, "LIN_REG_EXPR_F64", f64)
    calls = []

    def fake(symbol, inputs, names, kwargs, raw_kwargs=None):
        calls.append((symbol, inputs, list(names), kwargs))
        return pa.array([None, None], type=pa.struct([("target_0", pa.large_list(pa.float64()))]))

    monkeypatch.setattr(_harness, "call_plugin", fake)
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


@pytest.mark.parametrize("sym", SYMBOLS)
def test_too_few_inputs(sym):
    _fails_with(sym, [OFFSETS, _col(sym.endswith("_f32"))], ["__offsets__", "target_0"],
                f"{sym}: need offsets, target and at least one feature")


@pytest.mark.parametrize("offsets", [pa.array(np.array([0, 5, 10], dtype=np.int32)),
                                     pa.array([0, None, 10], type=pa.int64())], ids=["int32", "null"])
@pytest.mark.parametrize("sym", SYMBOLS)
def test_offsets_must_be_one_non_null_int64_chunk(sym, offsets):
    f32 = sym.endswith("_f32")
    _fails_with(sym, [offsets, _col(f32), _col(f32, 1), _col(f32, 2)], ["__offsets__", "target_0", "target_1", "x1"],
                f"{sym}: offsets must be one non-null Int64 chunk")


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


@pytest.mark.skipif(_has_gpu(), reason="checks the loud failure on a box without a GPU")
@pytest.mark.parametrize("sym", SYMBOLS)
def test_well_formed_call_fails_loudly_without_gpu(sym):
    f32 = sym.endswith("_f32")
    with pytest.raises(pds.PdsbError, match="no CPU fallback"):
        _harness.call_plugin(sym, [OFFSETS, _col(f32), _col(f32, 1), _col(f32, 2)],
                             ["__offsets__", "target_0", "target_1", "x1"], KW)
    df = pds.Frame({"x1": np.arange(10.0), "y": np.arange(10.0) % 3, "z": np.arange(10.0) % 4, "g": np.arange(10) % 2})
    with pytest.raises(pds.PdsbError, match="no CPU fallback"):
        df.group_by("g").agg(pds.lin_reg("x1", target=["y", "z"], add_bias=True), fast=True)
