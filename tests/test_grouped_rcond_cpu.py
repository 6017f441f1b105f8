"""CPU-side checks of group_by().agg(lin_reg_w_rcond) on the device: pl_lr_w_rcond_by and its f32 twin are exported and
declared once, in include/polars_plugin_group_rcond_abi.h only; the schema twins are a LargeList of pl_lr_w_rcond's
struct; the fast path sends [offsets, y, x...] with the kwargs unchanged; the plugin layer's input checks give their exact
messages; over(fast=True) is still refused; and without a GPU the call fails loudly."""
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
RCOND_HEADER = ROOT / "include" / "polars_plugin_group_rcond_abi.h"
SYMBOLS = ["pl_lr_w_rcond_by", "pl_lr_w_rcond_by_f32"]
ENTRIES = ["pdsb_host_grouped_lin_reg_rcond", "pdsb_dev_grouped_lin_reg_rcond_f32", "pdsb_dev_grouped_lin_reg_rcond_f64"]
KW = {"bias": True, "null_policy": "skip", "l1_reg": 0.0, "l2_reg": 0.0, "solver": "", "tol": 1e-5}
OFFSETS = pa.array(np.array([0, 5, 10], dtype=np.int64))


def _has_gpu():
    try:
        import torch

        return torch.cuda.is_available()
    except Exception:
        return False


def _code(header):
    return re.sub(r"/\*.*?\*/", "", header.read_text(), flags=re.S)


def _col(f32):
    return pa.array(np.arange(10, dtype=np.float32 if f32 else np.float64) % 3)


def test_symbol_list():
    assert _harness.GROUPED_RCOND_SYMBOLS == SYMBOLS


@pytest.mark.parametrize("sym", SYMBOLS)
def test_symbol_and_twin_exported(sym):
    L = lib()
    assert hasattr(L, f"_polars_plugin_{sym}") and hasattr(L, f"_polars_plugin_field_{sym}"), sym


@pytest.mark.parametrize("sym", SYMBOLS)
def test_declared_once_in_the_rcond_header_only(sym):
    assert re.findall(r"PDSB_DECLARE_EXPR\((\w+)\)", _code(RCOND_HEADER)).count(sym) == 1
    for h in sorted((ROOT / "include").glob("*.h")):
        if h != RCOND_HEADER:
            assert not re.search(rf"\b{sym}\b", _code(h)), (h.name, sym)


def test_the_rcond_header_declares_nothing_else():
    assert sorted(re.findall(r"PDSB_DECLARE_EXPR\((\w+)\)", _code(RCOND_HEADER))) == SYMBOLS


@pytest.mark.parametrize("sym", SYMBOLS)
def test_symbol_is_in_no_other_list(sym):
    others = (_harness.PLUGIN_SYMBOLS + _harness.PCA_SYMBOLS + _harness.SPLINE_SYMBOLS + _harness.ISOTONIC_SYMBOLS
              + _harness.GROUPED_SYMBOLS)
    assert sym not in others and _harness.GROUPED_RCOND_SYMBOLS.count(sym) == 1


def test_host_and_device_entries_exported_and_declared():
    L = lib()
    pdsb_h = (ROOT / "include" / "pdsb.h").read_text()
    for fn in ENTRIES:
        assert hasattr(L, fn), fn
        assert f"int {fn}(" in pdsb_h, fn


@pytest.mark.parametrize("f32", [False, True])
def test_field_twin_is_a_large_list_of_the_single_call_struct(f32):
    sfx = "_f32" if f32 else ""
    f = _harness.field_of(f"pl_lr_w_rcond_by{sfx}")
    single = _harness.field_of(f"pl_lr_w_rcond{sfx}").type
    assert f.type == pa.large_list(pa.field("item", single))
    T = pa.float32() if f32 else pa.float64()
    assert [single.field(i).name for i in range(single.num_fields)] == ["coeffs", "singular_values"]
    assert all(single.field(i).type == pa.large_list(pa.field("item", T)) for i in range(2))


def test_batched_symbol_table():
    assert frame_mod._by_group("pl_lr_w_rcond", per_row=False) == "pl_lr_w_rcond_by"
    assert frame_mod._by_group("pl_lr_w_rcond_f32", per_row=False) == "pl_lr_w_rcond_by"
    assert frame_mod._by_group("pl_lr_w_rcond", per_row=True) is None


@pytest.mark.parametrize("f64", [True, False])
def test_fast_agg_sends_offsets_y_x_and_the_kwargs_unchanged(monkeypatch, f64):
    monkeypatch.setattr(cfg, "LIN_REG_EXPR_F64", f64)
    calls = []

    def fake(symbol, inputs, names, kwargs, raw_kwargs=None):
        calls.append((symbol, inputs, list(names), kwargs))
        return pa.array([None, None], type=pa.large_list(pa.struct([("coeffs", pa.large_list(pa.float64()))])))

    monkeypatch.setattr(_harness, "call_plugin", fake)
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


def _fails_with(sym, inputs, names, msg):
    with pytest.raises(pds.PdsbError) as ei:
        _harness.call_plugin(sym, inputs, names, KW)
    assert str(ei.value) == f"the plugin failed with message: {msg}"


@pytest.mark.parametrize("sym", SYMBOLS)
def test_too_few_inputs(sym):
    _fails_with(sym, [OFFSETS, _col(sym.endswith("_f32"))], ["__offsets__", "y"],
                f"{sym}: need offsets, target and at least one feature")


@pytest.mark.parametrize("offsets", [pa.array(np.array([0, 5, 10], dtype=np.int32)),
                                     pa.array([0, None, 10], type=pa.int64())], ids=["int32", "null"])
@pytest.mark.parametrize("sym", SYMBOLS)
def test_offsets_must_be_one_non_null_int64_chunk(sym, offsets):
    f32 = sym.endswith("_f32")
    _fails_with(sym, [offsets, _col(f32), _col(f32)], ["__offsets__", "y", "x1"],
                f"{sym}: offsets must be one non-null Int64 chunk")


def test_over_fast_and_other_symbols_are_still_refused():
    df = pds.Frame({"a": np.arange(6.0), "w": np.ones(6), "y": np.arange(6.0) % 2, "g": np.arange(6) % 2})
    with pytest.raises(ValueError, match="fast over is only available for lin_reg predictions"):
        pds.lin_reg_w_rcond("a", target="y").over("g", fast=True)
    with pytest.raises(ValueError, match="fast group_by is only available for lin_reg coefficients.*lin_reg_w_rcond"):
        df.group_by("g").agg(pds.rolling_lin_reg("a", target="y", window_size=3), fast=True)


@pytest.mark.skipif(_has_gpu(), reason="checks the loud failure on a box without a GPU")
@pytest.mark.parametrize("sym", SYMBOLS)
def test_well_formed_call_fails_loudly_without_gpu(sym):
    f32 = sym.endswith("_f32")
    with pytest.raises(pds.PdsbError, match="no CPU fallback"):
        _harness.call_plugin(sym, [OFFSETS, _col(f32), _col(f32)], ["__offsets__", "y", "x1"], KW)
    df = pds.Frame({"x1": np.arange(10.0), "y": np.arange(10.0) % 3, "g": np.arange(10) % 2})
    with pytest.raises(pds.PdsbError, match="no CPU fallback"):
        df.group_by("g").agg(pds.lin_reg_w_rcond("x1", target="y", add_bias=True), fast=True)
