"""CPU-side checks of group_by().agg(logistic_reg) and logistic_reg(return_pred=True).over(key) on the device: the
pl_logistic_by / pl_logistic_pred_by symbols and their schema twins are exported, the Python expressions carry
logistic_reg's kwargs, the fast paths are refused for every other symbol, and without a GPU the calls fail loudly."""
import re
from pathlib import Path

import numpy as np
import pyarrow as pa
import pytest

import polars_ds_extension_b200 as pds
from polars_ds_extension_b200 import _harness
from polars_ds_extension_b200._lib import lib

ROOT = Path(__file__).resolve().parent.parent


def _has_gpu():
    try:
        import torch

        return torch.cuda.is_available()
    except Exception:
        return False


def test_symbols_and_twins_exported():
    L = lib()
    text = (ROOT / "include" / "polars_plugin_group_logistic_abi.h").read_text()
    declared = re.findall(r"PDSB_DECLARE_GROUP_LOGISTIC_EXPR\((\w+)\)", text)
    assert sorted(n for n in declared if n != "name") == sorted(_harness.GROUPED_LOGISTIC_SYMBOLS)
    for sym in _harness.GROUPED_LOGISTIC_SYMBOLS:
        assert hasattr(L, f"_polars_plugin_{sym}") and hasattr(L, f"_polars_plugin_field_{sym}"), sym
    for fn in ("pdsb_dev_grouped_logistic_f64", "pdsb_host_grouped_logistic"):
        assert hasattr(L, fn), fn


def test_field_twins_match_the_single_fit_symbols():
    f = _harness.field_of("pl_logistic_by")
    assert f.type == _harness.field_of("pl_logistic_coeffs").type == pa.large_list(pa.field("item", pa.float64()))
    g = _harness.field_of("pl_logistic_pred_by")
    assert g.type == _harness.field_of("pl_logistic_pred").type == pa.float64()
    assert g.name == "pred"


def test_symbol_lists_are_disjoint():
    others = (_harness.PLUGIN_SYMBOLS + _harness.PCA_SYMBOLS + _harness.SPLINE_SYMBOLS + _harness.ISOTONIC_SYMBOLS
              + _harness.GROUPED_PRED_SYMBOLS)
    assert not set(others) & set(_harness.GROUPED_LOGISTIC_SYMBOLS)
    assert len(set(_harness.GROUPED_LOGISTIC_SYMBOLS)) == len(_harness.GROUPED_LOGISTIC_SYMBOLS)


def test_new_symbols_are_not_in_the_other_headers():
    for h in ("polars_plugin_abi.h", "polars_plugin_group_abi.h", "polars_plugin_num_abi.h"):
        text = (ROOT / "include" / h).read_text()
        for sym in _harness.GROUPED_LOGISTIC_SYMBOLS:
            assert sym not in text, (h, sym)


@pytest.mark.parametrize("pred", [False, True])
def test_expressions_carry_logistic_reg_kwargs(pred):
    base = pds.logistic_reg("a", "b", target="y", add_bias=False, l1_reg=0.01, l2_reg=0.1, tol=1e-9, max_iter=7,
                            null_policy="zero", return_pred=pred)
    assert base.symbol == ("pl_logistic_pred" if pred else "pl_logistic_coeffs")
    assert base.kwargs == {"bias": False, "null_policy": "zero", "l1_reg": 0.01, "l2_reg": 0.1, "solver": "",
                           "tol": 1e-9, "max_iter": 7}
    assert [c.out_name for c in base.args] == ["y", "a", "b"]
    if pred:
        e = base.over("g", fast=True)
        assert e.symbol == base.symbol and e.kwargs == base.kwargs and e.over_key == "g" and e.over_fast
        assert base.over_key is None and not base.over_fast
    else:
        with pytest.raises(ValueError, match="fast over is only available for lin_reg predictions"):
            base.over("g", fast=True)


def test_batched_symbol_table():
    from polars_ds_extension_b200.frame import _by_group

    assert _by_group("pl_logistic_coeffs", per_row=False) == "pl_logistic_by"
    assert _by_group("pl_logistic_pred", per_row=True) == "pl_logistic_pred_by"
    assert _by_group("pl_lr", per_row=False) == "pl_lr_by"
    assert _by_group("pl_lr_pred_f32", per_row=True) == "pl_lr_pred_by"
    assert _by_group("pl_logistic_pred", per_row=False) is None
    assert _by_group("pl_logistic_coeffs", per_row=True) is None
    assert _by_group("pl_rolling_lr", per_row=True) is None


def test_fast_paths_still_refuse_other_symbols():
    with pytest.raises(ValueError, match="fast over is only available for lin_reg predictions"):
        pds.lin_reg("a", target="y").over("g", fast=True)
    with pytest.raises(ValueError, match="fast over is only available for lin_reg predictions"):
        pds.rolling_lin_reg("a", target="y", window_size=3).over("g", fast=True)
    with pytest.raises(ValueError, match="fast over is only available for lin_reg predictions"):
        pds.lin_reg("a", "b", target=["y", "z"], return_pred=True).over("g", fast=True)
    df = pds.Frame({"a": np.arange(6.0), "y": np.arange(6.0) % 2, "g": np.arange(6) % 2})
    with pytest.raises(ValueError, match="fast group_by is only available for lin_reg coefficients"):
        df.group_by("g").agg(pds.logistic_reg("a", target="y", return_pred=True), fast=True)
    with pytest.raises(ValueError, match="fast group_by is only available for lin_reg coefficients"):
        df.group_by("g").agg(pds.rolling_lin_reg("a", target="y", window_size=3), fast=True)


@pytest.mark.skipif(_has_gpu(), reason="checks the loud failure on a box without a GPU")
def test_fails_loudly_without_gpu():
    df = pds.Frame({"x1": np.arange(10.0), "y": (np.arange(10) % 3 == 0).astype(np.float64), "g": np.arange(10) % 2})
    with pytest.raises(pds.PdsbError, match="no CPU fallback"):
        df.select(pds.logistic_reg("x1", target="y", return_pred=True).over("g", fast=True))
    with pytest.raises(pds.PdsbError, match="no CPU fallback"):
        df.group_by("g").agg(pds.logistic_reg("x1", target="y"), fast=True)
    kw = pds.logistic_reg("x1", target="y").kwargs
    for sym in _harness.GROUPED_LOGISTIC_SYMBOLS:
        with pytest.raises(pds.PdsbError, match="no CPU fallback"):
            _harness.call_plugin(sym, [pa.array(np.array([0, 5, 10], dtype=np.int64)), pa.array(np.arange(10.0) % 2),
                                       pa.array(np.arange(10.0))], ["__offsets__", "y", "x1"], kw)
