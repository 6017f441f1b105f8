"""CPU-side checks of grouped PCA on the device: the pl_singular_values_by / pl_pca_by / pl_principal_components_by
schema twins, the fast paths send [offsets, (k), raw features...] in group order with {"center": ...}, singular_values'
list steps run per group, a mix of centred and un-centred features is refused, the other refusals still hold, and
without a GPU the call fails loudly."""
import numpy as np
import pyarrow as pa
import pytest

import polars_ds_extension_b200 as pds
from polars_ds_extension_b200 import _harness
from polars_ds_extension_b200 import frame as frame_mod
from polars_ds_extension_b200.frame import col
from tests.helpers import capture_plugin, has_gpu

REFUSED_AGG = "fast group_by is only available for lin_reg coefficients"
REFUSED_OVER = "fast over is only available for lin_reg predictions"


def test_field_twins():
    assert _harness.field_of("pl_singular_values_by").type == _harness.field_of("pl_singular_values").type
    single = _harness.field_of("pl_pca").type
    assert _harness.field_of("pl_pca_by").type == pa.large_list(pa.field("pca", single))
    ins = [pa.field("__offsets__", pa.int64()), pa.field("literal", pa.uint32())] + \
        [pa.field(f"x{i}", pa.float64()) for i in range(3)]
    t = _harness.field_of("pl_principal_components_by", ins).type
    assert [t.field(i).name for i in range(t.num_fields)] == ["pc1", "pc2", "pc3"]
    assert all(t.field(i).type == pa.float64() for i in range(t.num_fields))


def _frame():
    return pds.Frame({"a": np.arange(8.0), "b": np.arange(8.0) ** 2, "c": np.arange(8, dtype=np.float32),
                      "g": np.array([1, 0, 1, 0, 1, 0, 1, 0])})


@pytest.mark.parametrize("center", [True, False])
def test_fast_agg_sends_offsets_and_raw_columns(monkeypatch, center):
    calls = capture_plugin(monkeypatch, pa.array([[3.0, 1.0], [4.0, 1.0]], type=pa.large_list(pa.float64())))
    e = pds.singular_values("a", "b", center=center)
    out = _frame().group_by("g").agg(e, fast=True)
    (symbol, inputs, names, kwargs), = calls
    assert symbol == "pl_singular_values_by"
    assert names == ["__offsets__", "a", "b"]
    assert kwargs == {"center": center}
    assert inputs[0].to_pylist() == [0, 4, 8]
    assert inputs[1].to_pylist() == [0.0, 2.0, 4.0, 6.0, 1.0, 3.0, 5.0, 7.0]     # stable group order, un-centred
    assert inputs[2].to_pylist() == [0.0, 4.0, 16.0, 36.0, 1.0, 9.0, 25.0, 49.0]
    assert list(out["g"]) == [1, 0]
    assert out["pl_singular_values"].to_pylist() == [[3.0, 1.0], [4.0, 1.0]]


def test_pca_agg_and_f32_column(monkeypatch):
    calls = capture_plugin(monkeypatch,
                           pa.array([None, None], type=pa.large_list(pa.struct([("singular_value", pa.float64())]))))
    _frame().group_by("g").agg(pds.pca("c", "a"), fast=True)
    (symbol, inputs, names, kwargs), = calls
    assert symbol == "pl_pca_by" and names == ["__offsets__", "c", "a"] and kwargs == {"center": True}
    assert inputs[1].type == pa.float32()                       # the column's own dtype: centring happens on the device
    assert inputs[1].to_pylist() == [0.0, 2.0, 4.0, 6.0, 1.0, 3.0, 5.0, 7.0]


def test_list_post_is_applied_per_group(monkeypatch):
    capture_plugin(monkeypatch, pa.array([[3.0, 1.0], [2.0, 2.0, 4.0], []], type=pa.large_list(pa.float64())))
    df = pds.Frame({"a": np.arange(6.0), "b": np.arange(6.0), "g": np.arange(6) % 3})
    ev = df.group_by("g").agg(pds.singular_values("a", "b", as_explained_var=True), fast=True)["pl_singular_values"]
    assert ev.to_pylist() == [[9.0, 1.0], [2.0, 2.0, 8.0], []]
    r = df.group_by("g").agg(pds.singular_values("a", "b", as_ratio=True), fast=True)["pl_singular_values"]
    assert r.to_pylist() == [[0.75, 0.25], [0.25, 0.25, 0.5], []]
    both = df.group_by("g").agg(pds.singular_values("a", "b", as_explained_var=True, as_ratio=True),
                                fast=True)["pl_singular_values"]
    np.testing.assert_allclose(both.to_pylist()[0], [0.9, 0.1])


def test_fast_over_passes_k_unpermuted(monkeypatch):
    pcs = pa.StructArray.from_arrays([pa.array(np.arange(8.0)), pa.array(-np.arange(8.0))], names=["pc1", "pc2"])
    calls = capture_plugin(monkeypatch, pcs)
    e = pds.principal_components("a", "b", "c", k=2, center=False)
    out = _frame().select(e.over("g", fast=True))["pl_principal_components"]
    (symbol, inputs, names, kwargs), = calls
    assert symbol == "pl_principal_components_by"
    assert names == ["__offsets__", "literal", "a", "b", "c"]
    assert kwargs == {"center": False}
    assert inputs[1].type == pa.uint32() and inputs[1].to_pylist() == [2]
    assert inputs[2].to_pylist() == [0.0, 2.0, 4.0, 6.0, 1.0, 3.0, 5.0, 7.0]
    # the per-row results go back to the frame's row order: row r of group order is frame row order[r]
    order = [0, 2, 4, 6, 1, 3, 5, 7]
    back = out.field("pc1").to_pylist()
    assert [back[order[r]] for r in range(8)] == list(np.arange(8.0))


def test_mixed_centring_is_refused():
    df = _frame()
    e = pds.singular_values("a", col("b").center(), center=False)
    with pytest.raises(ValueError, match="either every feature is centred or none is"):
        df.group_by("g").agg(e, fast=True)
    e = pds.principal_components(col("a").center(), "b", k=1, center=False)
    with pytest.raises(ValueError, match="either every feature is centred or none is"):
        df.select(e.over("g", fast=True))


def test_other_refusals_still_hold():
    df = pds.Frame({"a": np.arange(6.0), "w": np.ones(6), "y": np.arange(6.0) % 2, "g": np.arange(6) % 2})
    with pytest.raises(ValueError, match=REFUSED_AGG):
        df.group_by("g").agg(pds.rolling_lin_reg("a", target="y", window_size=3), fast=True)
    with pytest.raises(ValueError, match=REFUSED_AGG):
        df.group_by("g").agg(pds.lin_reg_report("a", target="y", weights="w"), fast=True)
    with pytest.raises(ValueError, match=REFUSED_AGG):
        df.group_by("g").agg(pds.principal_components("a", "y", k=1), fast=True)
    with pytest.raises(ValueError, match=REFUSED_OVER):
        pds.rolling_lin_reg("a", target="y", window_size=3).over("g", fast=True)
    with pytest.raises(ValueError, match=REFUSED_OVER):
        pds.singular_values("a", "y").over("g", fast=True)
    with pytest.raises(ValueError, match=REFUSED_OVER):
        pds.pca("a", "y").over("g", fast=True)
    assert frame_mod._by_group("pl_rolling_lr", per_row=True) is None


@pytest.mark.skipif(has_gpu(), reason="checks the loud failure on a box without a GPU")
def test_fails_loudly_without_gpu():
    df = pds.Frame({"x1": np.arange(10.0), "x2": np.arange(10.0) % 3, "g": np.arange(10) % 2})
    with pytest.raises(pds.PdsbError, match="no CPU fallback"):
        df.group_by("g").agg(pds.singular_values("x1", "x2"), fast=True)
    with pytest.raises(pds.PdsbError, match="no CPU fallback"):
        df.select(pds.principal_components("x1", "x2", k=1).over("g", fast=True))
