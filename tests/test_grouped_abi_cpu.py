"""CPU-side checks shared by every batched group symbol (`pl_*_by`): each is exported with its schema twin and declared
once, in include/polars_plugin_group_abi.h only; the symbol lists do not overlap; every family's host and device entries
are exported and declared in pdsb.h; the plugin layer's input checks give each symbol's exact message before any device
work, and a well-formed call fails loudly without a GPU; frame._BY_GROUP routes each single-call symbol to its batched
symbol for over (per row) or group_by().agg (per group) only."""
import re
from pathlib import Path

import numpy as np
import pyarrow as pa
import pytest

import polars_ds_extension_b200 as pds
from polars_ds_extension_b200 import _harness
from polars_ds_extension_b200 import frame as frame_mod
from polars_ds_extension_b200._lib import lib
from tests.helpers import has_gpu

ROOT = Path(__file__).resolve().parent.parent
GROUP_HEADER = ROOT / "include" / "polars_plugin_group_abi.h"

# each family's entries in include/pdsb.h: the host entry its symbols call and the device entries behind it
ENTRIES = {
    "lin_reg": ["pdsb_host_grouped_lin_reg", "pdsb_dev_grouped_lin_reg_f32", "pdsb_dev_grouped_lin_reg_f64"],
    "predict": ["pdsb_host_grouped_lin_reg_pred", "pdsb_dev_grouped_predict_f32", "pdsb_dev_grouped_predict_f64"],
    "logistic": ["pdsb_host_grouped_logistic", "pdsb_dev_grouped_logistic_f64"],
    "report": ["pdsb_host_grouped_report", "pdsb_dev_grouped_report_f32", "pdsb_dev_grouped_report_f64"],
    "pca": ["pdsb_host_pca_by", "pdsb_dev_grouped_pca_f32", "pdsb_dev_grouped_pca_f64", "pdsb_dev_grouped_project_f32",
            "pdsb_dev_grouped_project_f64"],
    "isotonic": ["pdsb_host_grouped_isotonic", "pdsb_dev_grouped_isotonic_f64"],
    "recursive": ["pdsb_host_grouped_recursive", "pdsb_dev_grouped_recursive_lin_reg_f32",
                  "pdsb_dev_grouped_recursive_lin_reg_f64"],
    "ar": ["pdsb_host_grouped_ar", "pdsb_dev_grouped_ar_lin_reg_f32", "pdsb_dev_grouped_ar_lin_reg_f64"],
    "rcond": ["pdsb_host_grouped_lin_reg_rcond", "pdsb_dev_grouped_lin_reg_rcond_f32",
              "pdsb_dev_grouped_lin_reg_rcond_f64"],
    "multi": ["pdsb_host_grouped_lin_reg_multi", "pdsb_dev_grouped_lin_reg_multi_f32",
              "pdsb_dev_grouped_lin_reg_multi_f64"],
    "glm": ["pdsb_glm_fit_by", "pdsb_dev_grouped_glm_f64"],
}

OFFSETS = pa.array(np.array([0, 5, 10], dtype=np.int64))
LR_KW = {"bias": True, "null_policy": "skip", "solver": "qr", "l1_reg": 0.0, "l2_reg": 0.0, "tol": 1e-5}
ONLINE_KW = {"null_policy": "skip", "n": 2, "bias": True, "lambda": 1.0, "min_size": 0}
PCA_KW = {"center": True}
ISO_KW = {"has_weights": False, "increasing": True}
RCOND_KW = {"bias": True, "null_policy": "skip", "l1_reg": 0.0, "l2_reg": 0.0, "solver": "", "tol": 1e-5}
MULTI_KW = {"bias": True, "null_policy": "raise", "solver": "qr", "last_target_idx": 2, "l2_reg": 0.0,
            "singular_x_tol": 1e-12}


def _col(f32=False):
    return pa.array(np.arange(10, dtype=np.float32 if f32 else np.float64) % 3)


def _k(value=1, type=pa.uint32()):
    return pa.array([value], type=type)


# symbol -> (well-formed inputs after the offsets, their names, kwargs, how many inputs are one too few, the message's
# tail for that).  The lin_reg and report twins name the f64 fit in their messages.
MSG_NAME = {"pl_lr_by_f32": "pl_lr_by", "pl_lr_pred_by": "pl_lr_by", "pl_lr_pred_by_f32": "pl_lr_by",
            "pl_lin_reg_report_by_f32": "pl_lin_reg_report_by"}
FEATURES = "need offsets, target and at least one feature"


def _lr(kw, f32=False):
    return [_col(f32), _col(f32)], ["y", "x1"], kw, 2, FEATURES


CALLS = {
    "pl_lr_by": _lr(LR_KW),
    "pl_lr_by_f32": _lr(LR_KW, True),
    "pl_lr_pred_by": _lr(LR_KW),
    "pl_lr_pred_by_f32": _lr(LR_KW, True),
    "pl_logistic_by": _lr(LR_KW),
    "pl_logistic_pred_by": _lr(LR_KW),
    "pl_lin_reg_report_by": _lr(dict(LR_KW, std_err="hc1")),
    "pl_lin_reg_report_by_f32": _lr(dict(LR_KW, std_err="hc1"), True),
    "pl_recursive_lr_by": _lr(ONLINE_KW),
    "pl_recursive_lr_by_f32": _lr(ONLINE_KW, True),
    "pl_singular_values_by": ([_col(), _col()], ["x1", "x2"], PCA_KW, 1, "need offsets and at least one feature"),
    "pl_pca_by": ([_col(), _col()], ["x1", "x2"], PCA_KW, 1, "need offsets and at least one feature"),
    "pl_principal_components_by": ([_k(), _col(), _col()], ["literal", "x1", "x2"], PCA_KW, 2,
                                   "need offsets, k and at least one feature"),
    "pl_isotonic_regression_by": ([_col()], ["y"], ISO_KW, 1, "need offsets and y"),
    "pl_ar_coeffs_by": ([_col()], ["x"], dict(LR_KW, lag=2), 1, "the inputs are the offsets and one column"),
    "pl_ar_coeffs_by_f32": ([_col(True)], ["x"], dict(LR_KW, lag=2), 1, "the inputs are the offsets and one column"),
    "pl_lr_w_rcond_by": _lr(RCOND_KW),
    "pl_lr_w_rcond_by_f32": _lr(RCOND_KW, True),
    "pl_lr_multi_by": ([_col(), _col(), _col()], ["target_0", "target_1", "x1"], MULTI_KW, 2, FEATURES),
    "pl_lr_multi_by_f32": ([_col(True), _col(True), _col(True)], ["target_0", "target_1", "x1"], MULTI_KW, 2, FEATURES),
}
SYMBOLS = sorted(CALLS)

# frame._BY_GROUP, row by row: single-call symbol -> (its batched symbol, whether that gives one value per row)
BY_GROUP = {
    "pl_lr": ("pl_lr_by", False),
    "pl_lr_pred": ("pl_lr_pred_by", True),
    "pl_logistic_coeffs": ("pl_logistic_by", False),
    "pl_logistic_pred": ("pl_logistic_pred_by", True),
    "pl_lin_reg_report": ("pl_lin_reg_report_by", False),
    "pl_singular_values": ("pl_singular_values_by", False),
    "pl_pca": ("pl_pca_by", False),
    "pl_principal_components": ("pl_principal_components_by", True),
    "pl_isotonic_regression": ("pl_isotonic_regression_by", True),
    "pl_recursive_lr": ("pl_recursive_lr_by", True),
    "pl_lr_w_rcond": ("pl_lr_w_rcond_by", False),
    "pl_lr_multi": ("pl_lr_multi_by", False),
}
# (symbol, its batched symbol or None, per_row): both spellings of every row, then single-call symbols with none
BY_GROUP_CASES = ([(single + sfx, batched, per_row) for single, (batched, per_row) in BY_GROUP.items()
                   for sfx in ("", "_f32")]
                  + [("pl_rolling_lr", None, True), ("pl_wls_report", None, False), ("pl_lr_multi_pred", None, False)])


def _code(header):
    """The header without its comments: prose may name a symbol, only code declares one."""
    return re.sub(r"/\*.*?\*/", "", header.read_text(), flags=re.S)


def test_all_20_batched_symbols_are_listed_and_checked():
    assert len(_harness.GROUPED_SYMBOLS) == 20
    assert SYMBOLS == sorted(_harness.GROUPED_SYMBOLS)
    assert BY_GROUP == frame_mod._BY_GROUP


@pytest.mark.parametrize("sym", _harness.GROUPED_SYMBOLS)
def test_symbol_and_twin_exported(sym):
    L = lib()
    assert hasattr(L, f"_polars_plugin_{sym}") and hasattr(L, f"_polars_plugin_field_{sym}"), sym


@pytest.mark.parametrize("sym", _harness.GROUPED_SYMBOLS)
def test_declared_once_in_the_group_header_only(sym):
    declared = re.findall(r"PDSB_DECLARE_EXPR\((\w+)\)", _code(GROUP_HEADER))
    assert declared.count(sym) == 1
    for h in sorted((ROOT / "include").glob("*.h")):
        if h != GROUP_HEADER:
            assert not re.search(rf"\b{sym}\b", _code(h)), (h.name, sym)


def test_the_group_header_declares_nothing_else():
    declared = re.findall(r"PDSB_DECLARE_EXPR\((\w+)\)", _code(GROUP_HEADER))
    assert sorted(declared) == sorted(_harness.GROUPED_SYMBOLS)


@pytest.mark.parametrize("sym", _harness.GROUPED_SYMBOLS)
def test_symbol_is_in_one_list_once(sym):
    every = (_harness.PLUGIN_SYMBOLS + _harness.PCA_SYMBOLS + _harness.SPLINE_SYMBOLS + _harness.ISOTONIC_SYMBOLS
             + _harness.GROUPED_SYMBOLS)
    assert every.count(sym) == 1


@pytest.mark.parametrize("family", sorted(ENTRIES))
def test_host_and_device_entries_exported_and_declared(family):
    L = lib()
    pdsb_h = (ROOT / "include" / "pdsb.h").read_text()
    for fn in ENTRIES[family]:
        assert hasattr(L, fn), fn
        assert f"int {fn}(" in pdsb_h, fn


def _fails_with(sym, inputs, names, kwargs, msg):
    with pytest.raises(pds.PdsbError) as ei:
        _harness.call_plugin(sym, inputs, names, kwargs)
    assert str(ei.value) == f"the plugin failed with message: {msg}"


@pytest.mark.parametrize("sym", SYMBOLS)
def test_too_few_inputs(sym):
    cols, names, kw, n_few, tail = CALLS[sym]
    _fails_with(sym, ([OFFSETS] + cols)[:n_few], (["__offsets__"] + names)[:n_few], kw,
                f"{MSG_NAME.get(sym, sym)}: {tail}")


@pytest.mark.parametrize("offsets", [pa.array(np.array([0, 5, 10], dtype=np.int32)),
                                     pa.array([0, None, 10], type=pa.int64())], ids=["int32", "null"])
@pytest.mark.parametrize("sym", SYMBOLS)
def test_offsets_must_be_one_non_null_int64_chunk(sym, offsets):
    cols, names, kw, _, _ = CALLS[sym]
    _fails_with(sym, [offsets] + cols, ["__offsets__"] + names, kw,
                f"{MSG_NAME.get(sym, sym)}: offsets must be one non-null Int64 chunk")


@pytest.mark.parametrize("k,msg", [(_k(1, pa.int64()), "invalid series dtype: expected `UInt32` for k"),
                                   (_k(None), "principal_components: k is null")], ids=["int64", "null"])
def test_principal_components_k_literal(k, msg):
    cols, names, kw, _, _ = CALLS["pl_principal_components_by"]
    _fails_with("pl_principal_components_by", [OFFSETS, k] + cols[1:], ["__offsets__"] + names, kw, msg)


@pytest.mark.parametrize("lag", [0, 65])
@pytest.mark.parametrize("sym", ["pl_ar_coeffs_by", "pl_ar_coeffs_by_f32"])
def test_ar_lag_range(sym, lag):
    cols, names, kw, _, _ = CALLS[sym]
    _fails_with(sym, [OFFSETS] + cols, ["__offsets__"] + names, dict(kw, lag=lag),
                f"{sym}: lag={lag}; the batched fit takes 1 to 64 lags (use the per-group loop)")


@pytest.mark.parametrize("symbol,batched,per_row", BY_GROUP_CASES)
def test_by_group_table(symbol, batched, per_row):
    assert frame_mod._by_group(symbol, per_row=per_row) == batched
    assert frame_mod._by_group(symbol, per_row=not per_row) is None
    assert batched is None or batched in _harness.GROUPED_SYMBOLS


@pytest.mark.skipif(has_gpu(), reason="checks the loud failure on a box without a GPU")
@pytest.mark.parametrize("sym", SYMBOLS)
def test_well_formed_call_fails_loudly_without_gpu(sym):
    cols, names, kw, _, _ = CALLS[sym]
    with pytest.raises(pds.PdsbError, match="no CPU fallback"):
        _harness.call_plugin(sym, [OFFSETS] + cols, ["__offsets__"] + names, kw)
