"""CPU-side checks of group_by().agg(lin_reg_report) on the device: the pl_lin_reg_report_by schema twins, the fast path
sends [offsets, y, x...] with the report's kwargs and no var(y) argument, weighted reports and other symbols are still
refused, and without a GPU the call fails loudly."""
import numpy as np
import pyarrow as pa
import pytest

import polars_ds_extension_b200 as pds
import polars_ds_extension_b200.config as cfg
from polars_ds_extension_b200 import _harness
from tests.helpers import capture_plugin, has_gpu

REFUSED = "fast group_by is only available for lin_reg coefficients"


@pytest.mark.parametrize("f32", [False, True])
def test_field_twin_is_a_large_list_of_the_report_struct(f32):
    sfx = "_f32" if f32 else ""
    f = _harness.field_of(f"pl_lin_reg_report_by{sfx}")
    single = _harness.field_of(f"pl_lin_reg_report{sfx}").type
    assert f.type == pa.large_list(pa.field("item", single))
    assert [single.field(i).name for i in range(single.num_fields)] == \
        ["features", "beta", "std_err", "t", "p>|t|", "0.025", "0.975", "r2", "adj_r2"]
    assert single.field(0).type == pa.large_string()
    assert all(single.field(i).type == (pa.float32() if f32 else pa.float64()) for i in range(1, 9))


@pytest.mark.parametrize("f64", [True, False])
@pytest.mark.parametrize("se", ["se", "hc0", "hc3"])
def test_fast_agg_sends_offsets_y_x_and_the_report_kwargs(monkeypatch, f64, se):
    monkeypatch.setattr(cfg, "LIN_REG_EXPR_F64", f64)
    calls = capture_plugin(monkeypatch, pa.array([None, None], type=pa.large_list(pa.struct([("beta", pa.float64())]))))
    df = pds.Frame({"a": np.arange(8.0), "b": np.arange(8.0) ** 2, "y": np.arange(8.0) % 3, "g": np.arange(8) % 2})
    e = pds.lin_reg_report("a", "b", target="y", add_bias=True, null_policy="skip", std_err=se)
    df.group_by("g").agg(e, fast=True)
    (symbol, inputs, names, kwargs), = calls
    assert symbol == "pl_lin_reg_report_by" + ("" if f64 else "_f32")
    assert names == ["__offsets__", "y", "a", "b"]
    assert kwargs == e.kwargs and kwargs["std_err"] == se and kwargs["bias"] and kwargs["null_policy"] == "skip"
    assert inputs[0].to_pylist() == [0, 4, 8]
    assert inputs[1].type == (pa.float64() if f64 else pa.float32())
    assert len(inputs[1]) == 8                        # the target's rows, not the one-row var(y)
    assert inputs[2].to_pylist() == [0.0, 2.0, 4.0, 6.0, 1.0, 3.0, 5.0, 7.0]       # rows in group order


def test_weighted_reports_and_other_symbols_are_still_refused():
    df = pds.Frame({"a": np.arange(6.0), "w": np.ones(6), "y": np.arange(6.0) % 2, "g": np.arange(6) % 2})
    with pytest.raises(ValueError, match=REFUSED):
        df.group_by("g").agg(pds.lin_reg_report("a", target="y", weights="w"), fast=True)
    with pytest.raises(ValueError, match=REFUSED):
        df.group_by("g").agg(pds.rolling_lin_reg("a", target="y", window_size=3), fast=True)
    with pytest.raises(ValueError, match=REFUSED):
        df.group_by("g").agg(pds.lin_reg("a", target="y", return_pred=True), fast=True)
    with pytest.raises(ValueError, match="fast over is only available for lin_reg predictions"):
        pds.lin_reg_report("a", target="y").over("g", fast=True)


@pytest.mark.skipif(has_gpu(), reason="checks the loud failure on a box without a GPU")
def test_fails_loudly_without_gpu():
    df = pds.Frame({"x1": np.arange(10.0), "y": np.arange(10.0) % 3, "g": np.arange(10) % 2})
    with pytest.raises(pds.PdsbError, match="no CPU fallback"):
        df.group_by("g").agg(pds.lin_reg_report("x1", target="y", add_bias=True), fast=True)
