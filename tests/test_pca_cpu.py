"""CPU checks of the PCA expressions: the NumPy oracle against sklearn (the reference's test_pca with a seeded RNG), the
sign rule against sklearn's svd_flip, the explained-variance / ratio post-steps, the wrappers' symbols and inputs,
centring and the k literal, the schema twins, and the loud failure without a GPU."""
import numpy as np
import pyarrow as pa
import pytest

import polars_ds_extension_b200 as pds
from polars_ds_extension_b200 import _harness
from polars_ds_extension_b200.frame import Frame, _list_post
from tests import pca_oracle as po
from tests.helpers import has_gpu


def _uniform_frame(n=2000, seed=52):
    rng = np.random.default_rng(seed)
    return {f"x{i}": rng.random(n) for i in (1, 2, 3)}


def test_oracle_matches_sklearn_pca():
    # tests/test_many.py:52-86 of the reference, pds.random replaced by a seeded numpy RNG
    from sklearn.decomposition import PCA

    d = _uniform_frame()
    X = np.column_stack([d["x1"], d["x2"], d["x3"]])
    Xc = X - X.mean(axis=0)
    sk = PCA().fit(X)
    s = po.singular_values([Xc[:, i] for i in range(3)])
    assert np.isclose(s, sk.singular_values_).all()
    s2, W = po.pca([Xc[:, i] for i in range(3)])
    np.testing.assert_allclose(s2, sk.singular_values_, rtol=1e-12)
    np.testing.assert_allclose(W, sk.components_, rtol=1e-9, atol=1e-12)   # signs included


def test_sign_rule_is_svd_flip():
    from sklearn.utils.extmath import svd_flip

    rng = np.random.default_rng(3)
    for p in (1, 2, 5, 17):
        X = rng.standard_normal((50, p))
        u, s, vt = np.linalg.svd(X, full_matrices=False)
        _, vt_flip = svd_flip(u.copy(), vt.copy(), u_based_decision=False)
        np.testing.assert_array_equal(po.sign_fix(vt.T).T, vt_flip)
    V = np.array([[0.6, -0.8], [-0.6, 0.6]])          # |max| tie in column 0: the first entry decides
    np.testing.assert_array_equal(po.sign_fix(V)[:, 0], [0.6, -0.6])


def test_post_steps_mirror_the_list_eval():
    s = np.array([4.0, 2.0, 1.0])
    arr = pa.array([s.tolist()], type=pa.large_list(pa.float64()))
    ev = np.asarray(_list_post(arr, "explained_var")[0].as_py())
    # quirk kept: pl.count() inside list.eval counts the list's elements (3), not the rows (n - 1 in sklearn)
    np.testing.assert_allclose(ev, s ** 2 / 2.0)
    np.testing.assert_allclose(ev, po.explained_var(s))
    r = np.asarray(_list_post(_list_post(arr, "explained_var"), "ratio")[0].as_py())
    np.testing.assert_allclose(r, po.ratio(po.explained_var(s)))
    assert pds.singular_values("a", "b", as_explained_var=True, as_ratio=True).list_post == ("explained_var", "ratio")
    assert pds.singular_values("a", "b", as_ratio=True).list_post == ("ratio",)


def test_wrappers_symbols_inputs_and_validation():
    e = pds.singular_values("a", "b")
    assert e.symbol == "pl_singular_values" and e.returns_scalar and e.kwargs is None
    assert [a.name for a in e.args] == ["a", "b"] and all(a.centered for a in e.args)
    assert not any(a.centered for a in pds.singular_values("a", "b", center=False).args)
    e = pds.pca("a", "b", "c", center=False)
    assert e.symbol == "pl_pca" and e.changes_length and e.pass_name_to_apply and e.kwargs is None
    e = pds.principal_components("a", "b", "c", k=2)
    assert e.symbol == "pl_principal_components" and e.pass_name_to_apply and not e.returns_scalar
    assert e.args[0].lit_u32 == 2 and [a.name for a in e.args[1:]] == ["a", "b", "c"]
    assert all(a.centered for a in e.args[1:]) and not e.args[0].centered
    for k in (0, 4, -1):
        with pytest.raises(ValueError, match="Input `k` should be between 1 and the number of features inclusive."):
            pds.principal_components("a", "b", "c", k=k)


def test_centring_and_literal_evaluation():
    f = Frame({"a": pa.array([1.0, None, 3.0, 8.0]), "b": pa.array([1, 2, 3, 6], type=pa.int32()),
               "c": pa.array([1.0, 2.0, 4.0, 5.0], type=pa.float32())})
    a = f._eval_arg(pds.col("a").center()).combine_chunks()
    assert a.null_count == 1 and a.type == pa.float64()
    np.testing.assert_allclose(a.fill_null(0).to_numpy(), [-3.0, 0.0, -1.0, 4.0])     # mean over non-null = 4
    b = f._eval_arg(pds.col("b").center()).combine_chunks()
    assert b.type == pa.float64()
    np.testing.assert_allclose(b.to_numpy(), [-2.0, -1.0, 0.0, 3.0])
    c = f._eval_arg(pds.col("c").center()).combine_chunks()
    assert c.type == pa.float32()
    np.testing.assert_allclose(c.to_numpy(), [-2.0, -1.0, 1.0, 2.0])
    k = f._eval_arg(pds.principal_components("a", "b", k=2).args[0])
    assert k.type == pa.uint32() and k.to_pylist() == [2]


def test_schema_twins_of_the_pca_symbols():
    f = _harness.field_of("pl_singular_values")
    assert f.name == "singular_values" and f.type == pa.large_list(pa.field("item", pa.float64()))
    f = _harness.field_of("pl_pca")
    assert f.name == "pca" and [c.name for c in f.type] == ["singular_value", "weight_vector"]
    assert f.type.field(0).type == pa.float64() and f.type.field(1).type == pa.large_list(pa.field("item", pa.float64()))
    ins = [pa.field("literal", pa.uint32())] + [pa.field(n, pa.float64()) for n in ("a", "b", "c")]
    f = _harness.field_of("pl_principal_components", ins)
    # the reference declares one pc field per input, the k literal included (pca.rs:28-37)
    assert f.name == "principal_components" and [c.name for c in f.type] == ["pc1", "pc2", "pc3", "pc4"]
    assert all(c.type == pa.float64() for c in f.type)
    assert set(_harness.PCA_SYMBOLS).isdisjoint(_harness.PLUGIN_SYMBOLS)


@pytest.mark.skipif(has_gpu(), reason="checks the loud failure on a box without a GPU")
def test_pca_symbols_fail_loudly_without_gpu():
    # also shows the empty kwargs buffer is accepted: the call gets past the kwargs to the device check
    df = Frame(_uniform_frame(20))
    for e in (pds.singular_values("x1", "x2"), pds.pca("x1", "x2"), pds.principal_components("x1", "x2", k=1)):
        with pytest.raises(pds.PdsbError, match="no CPU fallback"):
            df.select(e)
