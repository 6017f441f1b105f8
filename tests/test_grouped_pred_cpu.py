"""CPU-side checks of lin_reg(return_pred=True).over(key): the pl_lr_pred_by schema twins, the Python expression carries
pl_lr_pred's kwargs, the fast path is refused for other symbols, and without a GPU the call fails loudly."""
import numpy as np
import pyarrow as pa
import pytest

import polars_ds_extension_b200 as pds
from polars_ds_extension_b200 import _harness
from tests.helpers import has_gpu


@pytest.mark.parametrize("sym", ["pl_lr_pred_by", "pl_lr_pred_by_f32"])
def test_field_twin_is_pred_struct(sym):
    T = pa.float32() if sym.endswith("_f32") else pa.float64()
    f = _harness.field_of(sym)
    assert pa.types.is_struct(f.type)
    assert [c.name for c in f.type] == ["pred", "resid"]
    assert f.type.field(0).type == T and f.type.field(1).type == T
    assert f.type == _harness.field_of("pl_lr_pred" + ("_f32" if sym.endswith("_f32") else "")).type


@pytest.mark.parametrize("f64", [True, False])
def test_over_carries_lin_reg_pred_kwargs(monkeypatch, f64):
    import polars_ds_extension_b200.config as cfg

    monkeypatch.setattr(cfg, "LIN_REG_EXPR_F64", f64)
    base = pds.lin_reg("a", "b", target="y", add_bias=True, l2_reg=0.1, return_pred=True)
    e = base.over("g", fast=True)
    assert e.symbol == base.symbol == ("pl_lr_pred" if f64 else "pl_lr_pred_f32")
    assert e.kwargs == base.kwargs
    assert [c.out_name for c in e.args] == [c.out_name for c in base.args] == ["y", "a", "b"]
    assert e.over_key == "g" and e.over_fast
    assert base.over_key is None and not base.over_fast          # the expression it came from is unchanged
    slow = base.over("g")
    assert slow.over_key == "g" and not slow.over_fast and slow.kwargs == base.kwargs


def test_fast_over_refuses_other_symbols():
    with pytest.raises(ValueError, match="fast over is only available for lin_reg predictions"):
        pds.lin_reg("a", target="y").over("g", fast=True)
    with pytest.raises(ValueError, match="fast over is only available for lin_reg predictions"):
        pds.rolling_lin_reg("a", target="y", window_size=3).over("g", fast=True)
    with pytest.raises(ValueError, match="fast over is only available for lin_reg predictions"):
        pds.lin_reg("a", "b", target=["y", "z"], return_pred=True).over("g", fast=True)
    pds.rolling_lin_reg("a", target="y", window_size=3).over("g")     # any row-shaped symbol works without fast


def test_group_order_helpers():
    from polars_ds_extension_b200.frame import _group_ids, _key_order

    keys = np.array([5, 3, 5, 9, 3, 3, 9, 1])
    uniq, gid = _group_ids(keys)
    assert uniq == [5, 3, 9, 1]                                   # first-seen order
    assert gid.tolist() == [0, 1, 0, 2, 1, 1, 2, 3]
    order, offsets = _key_order(gid, len(uniq))
    assert order.tolist() == [0, 2, 1, 4, 5, 3, 6, 7]             # stable within each group
    assert offsets.tolist() == [0, 2, 5, 7, 8]


@pytest.mark.skipif(has_gpu(), reason="checks the loud failure on a box without a GPU")
@pytest.mark.parametrize("fast", [True, False])
def test_fails_loudly_without_gpu(fast):
    df = pds.Frame({"x1": np.arange(10.0), "y": np.arange(10.0) * 2, "g": np.arange(10) % 2})
    with pytest.raises(pds.PdsbError, match="no CPU fallback"):
        df.select(pds.lin_reg("x1", target="y", return_pred=True).over("g", fast=fast))
