"""CPU-side checks of weighted lin_reg over groups (pl_wls_by, pl_wls_pred_by and their _f32 twins): the symbols and
their schema twins are exported and declared once, in include/polars_plugin_wls_abi.h only; the host and device entries
are exported and declared in pdsb.h; the frame sends [offsets, w, y, x...] with the expression's kwargs to them when the
expression is weighted, and unweighted ones still to pl_lr_by / pl_lr_pred_by; the argument, offset and group errors
come before any device work; a well-formed call fails loudly without a GPU."""
import re
from pathlib import Path

import numpy as np
import pyarrow as pa
import pytest

import polars_ds_extension_b200 as pds
from polars_ds_extension_b200 import _harness
from polars_ds_extension_b200 import frame as frame_mod
from polars_ds_extension_b200._lib import lib
from tests.helpers import capture_plugin, has_gpu

ROOT = Path(__file__).resolve().parent.parent
WLS_HEADER = ROOT / "include" / "polars_plugin_wls_abi.h"
SYMBOLS = ["pl_wls_by", "pl_wls_by_f32", "pl_wls_pred_by", "pl_wls_pred_by_f32"]
ENTRIES = ["pdsb_host_grouped_wls", "pdsb_dev_grouped_wls_lin_reg_f32", "pdsb_dev_grouped_wls_lin_reg_f64"]
LR_KW = {"bias": True, "null_policy": "skip", "l1_reg": 0.0, "l2_reg": 0.0, "solver": "qr", "tol": 1e-5,
         "max_iter": 200, "weighted": True, "positive": False, "singular_x_tol": 1e-12}
OFFSETS = pa.array(np.array([0, 5, 10], dtype=np.int64))


def _code(header):
    """The header without its comments: prose may name a symbol, only code declares one."""
    return re.sub(r"/\*.*?\*/", "", header.read_text(), flags=re.S)


def test_symbol_list():
    assert _harness.WLS_GROUP_SYMBOLS == SYMBOLS


@pytest.mark.parametrize("sym", SYMBOLS)
def test_symbol_and_twin_exported(sym):
    L = lib()
    assert hasattr(L, f"_polars_plugin_{sym}") and hasattr(L, f"_polars_plugin_field_{sym}"), sym


@pytest.mark.parametrize("sym", SYMBOLS)
def test_declared_once_in_the_wls_header_only(sym):
    assert re.findall(r"PDSB_DECLARE_EXPR\((\w+)\)", _code(WLS_HEADER)).count(sym) == 1
    for h in sorted((ROOT / "include").glob("*.h")):
        if h != WLS_HEADER:
            assert not re.search(rf"\b{sym}\b", _code(h)), (h.name, sym)


def test_the_wls_header_declares_nothing_else():
    assert sorted(re.findall(r"PDSB_DECLARE_EXPR\((\w+)\)", _code(WLS_HEADER))) == sorted(SYMBOLS)


@pytest.mark.parametrize("sym", SYMBOLS)
def test_symbol_is_in_one_list_once(sym):
    every = (_harness.PLUGIN_SYMBOLS + _harness.PCA_SYMBOLS + _harness.SPLINE_SYMBOLS + _harness.ISOTONIC_SYMBOLS
             + _harness.GROUPED_SYMBOLS + _harness.WLS_GROUP_SYMBOLS)
    assert every.count(sym) == 1


def test_header_compiles_as_c99_next_to_the_others(tmp_path):
    import shutil
    import subprocess

    if shutil.which("gcc") is None:
        pytest.skip("gcc not available")
    src = tmp_path / "hdr.c"
    src.write_text('#include "pdsb.h"\n#include "polars_plugin_group_abi.h"\n#include "polars_plugin_wls_abi.h"\n'
                   "int main(void) { return pdsb_version() < 0; }\n")
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", f"-I{ROOT / 'include'}",
                    "-fsyntax-only", str(src)], check=True)


@pytest.mark.parametrize("fn", ENTRIES)
def test_host_and_device_entries_exported_and_declared(fn):
    assert hasattr(lib(), fn), fn
    assert f"int {fn}(" in (ROOT / "include" / "pdsb.h").read_text(), fn


@pytest.mark.parametrize("sym", SYMBOLS)
def test_schema_twin_is_the_single_calls(sym):
    sfx = "_f32" if sym.endswith("_f32") else ""
    single = "pl_lr_pred" if "pred" in sym else "pl_lr"
    assert _harness.field_of(sym).type == _harness.field_of(single + sfx).type
    T = pa.float32() if sfx else pa.float64()
    f = _harness.field_of(sym)
    if "pred" in sym:
        assert [c.name for c in f.type] == ["pred", "resid"] and f.type.field(0).type == T
    else:
        assert f.name == "coeffs" and f.type == pa.large_list(pa.field("item", T))


def _frame():
    rng = np.random.default_rng(1)
    return pds.Frame({"a": rng.standard_normal(9), "b": rng.standard_normal(9), "y": rng.standard_normal(9),
                      "w": rng.uniform(0.5, 2.0, 9), "g": np.array([3, 1, 3, 2, 1, 3, 2, 2, 1])})


ORDER = [0, 2, 5, 1, 4, 8, 3, 6, 7]      # rows sorted stably by key, keys in first-seen order 3, 1, 2


@pytest.mark.parametrize("f64", [True, False])
def test_group_by_sends_offsets_w_y_x_to_pl_wls_by(monkeypatch, f64):
    import polars_ds_extension_b200.config as cfg

    monkeypatch.setattr(cfg, "LIN_REG_EXPR_F64", f64)
    calls = capture_plugin(monkeypatch, pa.array([None, None, None], type=pa.large_list(pa.float64())))
    df = _frame()
    e = pds.lin_reg("a", "b", target="y", add_bias=True, weights="w", l2_reg=0.5)
    df.group_by("g").agg(e, fast=True)
    (sym, inputs, names, kwargs), = calls
    assert sym == "pl_wls_by" + ("" if f64 else "_f32")
    assert names == ["__offsets__", "w", "y", "a", "b"]
    assert kwargs == e.kwargs and kwargs["weighted"] is True and kwargs["l2_reg"] == 0.5
    assert inputs[0].to_pylist() == [0, 3, 6, 9]
    for k, name in enumerate(["w", "y", "a", "b"], 1):
        want = df[name].to_numpy()[ORDER].astype(np.float64 if f64 else np.float32)
        assert np.array_equal(np.asarray(inputs[k].to_numpy(), dtype=want.dtype), want), name


@pytest.mark.parametrize("f64", [True, False])
def test_over_sends_the_same_inputs_to_pl_wls_pred_by(monkeypatch, f64):
    import polars_ds_extension_b200.config as cfg

    monkeypatch.setattr(cfg, "LIN_REG_EXPR_F64", f64)
    T = pa.float64() if f64 else pa.float32()
    res = pa.StructArray.from_arrays([pa.array(np.arange(9.0), type=T), pa.array(np.zeros(9), type=T)], ["pred", "resid"])
    calls = capture_plugin(monkeypatch, res)
    e = pds.lin_reg("a", target="y", weights="w", return_pred=True)
    out = _frame().select(e.over("g", fast=True))[e.out_name]
    (sym, inputs, names, kwargs), = calls
    assert sym == "pl_wls_pred_by" + ("" if f64 else "_f32")
    assert names == ["__offsets__", "w", "y", "a"] and kwargs == e.kwargs
    assert inputs[0].to_pylist() == [0, 3, 6, 9]
    # row ORDER[i] of the frame gets the i-th output row
    assert out.field("pred").to_numpy().tolist() == np.argsort(ORDER).astype(float).tolist()


def test_simple_lin_reg_with_weights_follows_lin_reg(monkeypatch):
    calls = capture_plugin(monkeypatch, pa.array([None, None, None], type=pa.large_list(pa.float64())))
    _frame().group_by("g").agg(pds.simple_lin_reg("a", target="y", weights="w"), fast=True)
    assert [c[0] for c in calls] == ["pl_wls_by"] and calls[0][2] == ["__offsets__", "w", "y", "a"]


def test_unweighted_expressions_still_go_to_pl_lr_by(monkeypatch):
    df = _frame()
    calls = capture_plugin(monkeypatch, pa.array([None, None, None], type=pa.large_list(pa.float64())))
    df.group_by("g").agg(pds.lin_reg("a", target="y"), fast=True)
    res = pa.StructArray.from_arrays([pa.array(np.zeros(9)), pa.array(np.zeros(9))], ["pred", "resid"])
    pred_calls = capture_plugin(monkeypatch, res)
    df.select(pds.lin_reg("a", target="y", return_pred=True).over("g", fast=True))
    assert [c[0] for c in calls + pred_calls] == ["pl_lr_by", "pl_lr_pred_by"]
    assert [c[2] for c in calls + pred_calls] == [["__offsets__", "y", "a"]] * 2


def test_weighted_routes_and_refusals():
    e = pds.lin_reg("a", target="y", weights="w")
    ep = pds.lin_reg("a", target="y", weights="w", return_pred=True)
    assert frame_mod._wls_by_group(e, per_row=False) == "pl_wls_by"
    assert frame_mod._wls_by_group(e, per_row=True) is None
    assert frame_mod._wls_by_group(ep, per_row=True) == "pl_wls_pred_by"
    assert frame_mod._wls_by_group(ep, per_row=False) is None
    assert frame_mod._wls_by_group(pds.lin_reg("a", target="y"), per_row=False) is None
    with pytest.raises(ValueError, match="fast over is only available for lin_reg predictions"):
        e.over("g", fast=True)
    with pytest.raises(ValueError, match="fast group_by is only available for lin_reg coefficients"):
        _frame().group_by("g").agg(pds.lin_reg_report("a", target="y", weights="w"), fast=True)


def _col(f32=False, n=10, seed=0):
    return pa.array(np.random.default_rng(seed).uniform(0.5, 2.0, n).astype(np.float32 if f32 else np.float64))


def _fails_with(sym, inputs, kwargs, msg, names=None):
    names = names or ["__offsets__", "w", "y"] + [f"x{i}" for i in range(len(inputs) - 3)]
    with pytest.raises(pds.PdsbError) as ei:
        _harness.call_plugin(sym, inputs, names[:len(inputs)], kwargs)
    assert str(ei.value) == f"the plugin failed with message: {msg}"


@pytest.mark.parametrize("sym", SYMBOLS)
def test_too_few_inputs(sym):
    f32 = sym.endswith("_f32")
    _fails_with(sym, [OFFSETS, _col(f32), _col(f32)], LR_KW,
                f"{sym}: need offsets, weights, target and at least one feature")


@pytest.mark.parametrize("offsets", [pa.array(np.array([0, 5, 10], dtype=np.int32)),
                                     pa.array([0, None, 10], type=pa.int64())], ids=["int32", "null"])
@pytest.mark.parametrize("sym", SYMBOLS)
def test_offsets_must_be_one_non_null_int64_chunk(sym, offsets):
    f32 = sym.endswith("_f32")
    _fails_with(sym, [offsets, _col(f32), _col(f32), _col(f32)], LR_KW, f"{sym}: offsets must be one non-null Int64 chunk")


@pytest.mark.parametrize("sym", SYMBOLS)
def test_unweighted_call_points_to_pl_lr_by(sym):
    f32 = sym.endswith("_f32")
    target = "pl_lr_pred_by" if "pred" in sym else "pl_lr_by"
    _fails_with(sym, [OFFSETS, _col(f32), _col(f32), _col(f32)], dict(LR_KW, weighted=False),
                f"{sym}: weighted is false; an unweighted fit goes to {target}")


# The host checks read host data only and come before the device check, so they give their messages on any machine
@pytest.mark.parametrize("offsets,msg", [([0, 5, 9], "grouped weighted lin_reg: bad group offsets"),
                                         ([1, 5, 10], "grouped weighted lin_reg: bad group offsets"),
                                         ([0, 6, 5, 10], "grouped weighted lin_reg: group offsets must be non-decreasing "
                                                         "and within [0, n] (group 1)")])
def test_bad_offsets(offsets, msg):
    off = pa.array(np.array(offsets, dtype=np.int64))
    _fails_with("pl_wls_by", [off, _col(), _col(), _col()], LR_KW, msg)


def test_weights_must_be_as_long_as_the_data():
    _fails_with("pl_wls_by", [OFFSETS, _col(n=9), _col(), _col()], LR_KW, "Shape of weights is not the same as the data.")


def test_data_columns_must_agree():
    _fails_with("pl_wls_by", [OFFSETS, _col(), _col(), _col(n=9)], LR_KW, "Seires don't have the same length.")


def test_at_most_64_features():
    cols = [pa.array(np.arange(70.0))] * 67
    off = pa.array(np.array([0, 70], dtype=np.int64))
    _fails_with("pl_wls_by", [off] + cols, LR_KW, "grouped weighted lin_reg: 65 features; at most 64 are supported")


def _with_null(a, rows):
    v = a.to_numpy(zero_copy_only=False).copy()
    mask = np.zeros(len(v), bool)
    mask[rows] = True
    return pa.array(v, mask=mask)


@pytest.mark.parametrize("col", [2, 3], ids=["y", "x"])
def test_raise_with_a_null(col):
    cols = [_col(seed=1), _col(seed=2), _col(seed=3)]
    cols[col - 1] = _with_null(cols[col - 1], [7])
    _fails_with("pl_wls_by", [OFFSETS] + cols, dict(LR_KW, null_policy="raise"), "Nulls found in data")


@pytest.mark.parametrize("policy,col", [("skip", 2), ("skip", 3), ("0.0", 2)], ids=["skip-y", "skip-x", "fill-y"])
def test_a_masked_row_fails_as_the_single_call_does(policy, col):
    # w = 1 everywhere: the single call counts llround(sum w over kept rows) = 4 rows in a group of 5
    w = pa.array(np.ones(10))
    cols = [w, _col(seed=2), _col(seed=3)]
    cols[col - 1] = _with_null(cols[col - 1], [7])
    _fails_with("pl_wls_by", [OFFSETS] + cols, dict(LR_KW, null_policy=policy),
                "Shape of weights is not the same as the data.")
    # weights summing to fewer rows than coefficients, and a NaN weight anywhere in the group
    for wv, msg in ((np.full(10, 0.1), "#Data < #features. No conclusive result."),
                    (np.where(np.arange(10) == 9, np.nan, 1.0), "#Data < #features. No conclusive result.")):
        _fails_with("pl_wls_by", [OFFSETS, pa.array(wv)] + cols[1:], dict(LR_KW, null_policy=policy), msg)


def test_a_masked_row_passes_when_the_weights_count_the_group():
    # kept weights summing to the group's length: the single call runs, and so does the batched call
    w = np.ones(10)
    w[5] = 2.0                                     # row 7 (null y) drops; 2 + 1 + 1 + 1 = 5 rows in group 1
    cols = [pa.array(w), _with_null(_col(seed=2), [7]), _col(seed=3)]
    call = lambda: _harness.call_plugin("pl_wls_by", [OFFSETS] + cols, ["__offsets__", "w", "y", "x"], LR_KW)
    if has_gpu():
        assert call().null_count == 0
    else:
        with pytest.raises(pds.PdsbError, match="no CPU fallback"):
            call()


def test_first_failing_group_decides_the_message():
    # group 0 has a null y under "skip" with weights of a small sum, group 1 with weights that count the group
    off = pa.array(np.array([0, 5, 10], dtype=np.int64))
    w = np.concatenate([np.full(5, 0.1), np.full(5, 1.5)])
    y = _with_null(_col(seed=2), [1, 7])
    _fails_with("pl_wls_by", [off, pa.array(w), y, _col(seed=3)], LR_KW, "#Data < #features. No conclusive result.")
    off = pa.array(np.array([0, 5, 10], dtype=np.int64))
    w = np.concatenate([np.full(5, 1.5), np.full(5, 0.1)])
    _fails_with("pl_wls_by", [off, pa.array(w), y, _col(seed=3)], LR_KW, "Shape of weights is not the same as the data.")


@pytest.mark.skipif(has_gpu(), reason="checks the loud failure on a box without a GPU")
@pytest.mark.parametrize("sym", SYMBOLS)
def test_well_formed_call_fails_loudly_without_gpu(sym):
    f32 = sym.endswith("_f32")
    with pytest.raises(pds.PdsbError, match="no CPU fallback"):
        _harness.call_plugin(sym, [OFFSETS, _col(f32), _col(f32), _col(f32)], ["__offsets__", "w", "y", "x"], LR_KW)


@pytest.mark.skipif(has_gpu(), reason="checks the loud failure on a box without a GPU")
def test_frame_call_fails_loudly_without_gpu():
    with pytest.raises(pds.PdsbError, match="no CPU fallback"):
        _frame().group_by("g").agg(pds.lin_reg("a", target="y", weights="w"), fast=True)
