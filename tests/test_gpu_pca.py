"""PCA expressions on the H100 through the plugin C ABI, against the NumPy oracle (tests/pca_oracle.py) and sklearn."""
import numpy as np
import pyarrow as pa
import pytest

import polars_ds_extension_b200 as pds
from polars_ds_extension_b200.frame import Frame
from tests import pca_oracle as po

pytestmark = pytest.mark.gpu
EPS = np.finfo(np.float64).eps


def _sv(res):
    return np.asarray(res[0].as_py(), dtype=np.float64)


def _pca(res):
    return (res.field("singular_value").to_numpy(zero_copy_only=False),
            np.array([np.asarray(v) for v in res.field("weight_vector").to_pylist()]).reshape(len(res), -1))


def _pcs(res):
    return np.column_stack([res.field(i).to_numpy(zero_copy_only=False) for i in range(res.type.num_fields)])


def _inputs(df, e):
    """The evaluated plugin inputs (centred as the wrapper asks) as f64 columns and validity, for the oracle."""
    cols, valid = [], []
    for a in e.args:
        if a.lit_u32 is not None:
            continue
        arr = df._eval_arg(a).combine_chunks()
        valid.append(np.asarray(arr.is_valid().to_numpy(zero_copy_only=False), dtype=bool))
        cols.append(arr.cast(pa.float64()).fill_null(0).to_numpy(zero_copy_only=False))
    return cols, (valid if any((~v).any() for v in valid) else None)


def _frame(X, dtype=np.float64):
    return Frame({f"x{i}": X[:, i].astype(dtype) for i in range(X.shape[1])})


def _check_vs_oracle(df, names, center=True):
    e = pds.singular_values(*names, center=center)
    cols, valid = _inputs(df, e)
    s_ref = po.singular_values(cols, valid)
    s = _sv(df.select(e)["pl_singular_values"])
    big = s_ref >= 1e-3 * s_ref[0]
    np.testing.assert_allclose(s[big], s_ref[big], rtol=1e-9)
    s2, W = _pca(df.select(pds.pca(*names, center=center))["pl_pca"])
    s_ref2, W_ref = po.pca(cols, valid)
    np.testing.assert_array_equal(s2, s)
    lam = s_ref2 ** 2
    gap = np.full(len(lam), np.inf)
    gap[:-1] = np.minimum(gap[:-1], lam[:-1] - lam[1:])
    gap[1:] = np.minimum(gap[1:], lam[:-1] - lam[1:])
    ok = gap >= 1e-2 * lam[0]
    np.testing.assert_allclose(W[ok], W_ref[ok], rtol=0, atol=1e-9)
    return s, W


def _spread(n, p, seed):
    rng = np.random.default_rng(seed)
    return rng.standard_normal((n, p)) * np.linspace(3.0, 0.2, p) + rng.standard_normal(p)


def test_lifted_reference_test_pca():
    from sklearn.decomposition import PCA

    rng = np.random.default_rng(52)
    df = Frame({f"x{i}": rng.random(2000) for i in (1, 2, 3)})
    s = _sv(df.select(pds.singular_values("x1", "x2", "x3").alias("res"))["res"])
    X = np.column_stack([df[f"x{i}"].to_numpy() for i in (1, 2, 3)])
    sk = PCA().fit(X)
    assert np.isclose(s, sk.singular_values_).all()
    _, W = _pca(df.select(pds.pca("x1", "x2", "x3").alias("vectors"))["vectors"])
    for i in range(len(W)):
        assert np.isclose(np.abs(W[i]), np.abs(sk.components_[i]), rtol=1e-5).all()
    np.testing.assert_allclose(W, sk.components_, atol=1e-9)           # the sign rule is sklearn's


@pytest.mark.parametrize("p", [1, 2, 3, 8, 31, 32, 33, 64, 65, 100, 259])
@pytest.mark.parametrize("dtype", ["f64", "f32", "i64"])
def test_matches_oracle(p, dtype):
    n = 3000 if p < 100 else 4000
    X = _spread(n, p, p)
    if dtype == "i64":
        df = _frame(np.rint(X * 100), np.int64)
    else:
        df = _frame(X, np.float32 if dtype == "f32" else np.float64)
    names = [f"x{i}" for i in range(p)]
    _check_vs_oracle(df, names)
    if p in (3, 32, 100):
        _check_vs_oracle(df, names, center=False)


def test_multi_chunk_and_sliced_inputs():
    X = _spread(5003, 12, 7)
    chunked = Frame({f"x{i}": pa.chunked_array([X[:1000, i], X[1000:1001, i], X[1001:, i]]) for i in range(12)})
    _check_vs_oracle(chunked, [f"x{i}" for i in range(12)])
    sliced = Frame({f"x{i}": pa.chunked_array([pa.array(X[:, i].astype(np.float32)).slice(3)]) for i in range(12)})
    _check_vs_oracle(sliced, [f"x{i}" for i in range(12)])


def test_uncentred_large_mean():
    X = _spread(4000, 6, 11) + 1e4
    df = _frame(X)
    names = [f"x{i}" for i in range(6)]
    s, _ = _check_vs_oracle(df, names, center=False)
    s_c, _ = _check_vs_oracle(df, names, center=True)
    assert s[0] > 1e4 * s_c[-1]


def _designed(n, sig, seed):
    rng = np.random.default_rng(seed)
    p = len(sig)
    U, _ = np.linalg.qr(rng.standard_normal((n, p)))
    V, _ = np.linalg.qr(rng.standard_normal((p, p)))
    return (U * sig) @ V.T


def test_designed_spectrum_meets_the_documented_bound():
    sig = np.logspace(0, -6, 8)
    X = _designed(4096, sig, 5)
    df = _frame(X)
    names = [f"x{i}" for i in range(8)]
    s = _sv(df.select(pds.singular_values(*names, center=False))["pl_singular_values"])
    s_ref = po.singular_values([X[:, i] for i in range(8)])
    rel = np.abs(s - s_ref) / s_ref
    bound = 64 * EPS * (s_ref[0] / s_ref) ** 2 + 4 * EPS * s_ref[0] / s_ref
    resolved = s_ref >= 1.5e-8 * s_ref[0]
    assert np.all(rel[resolved] <= bound[resolved]), (rel, bound)


def test_duplicated_column_trailing_value():
    X = _spread(3000, 5, 9)
    X = np.column_stack([X, X[:, 2]])
    df = _frame(X)
    s = _sv(df.select(pds.singular_values(*[f"x{i}" for i in range(6)]))["pl_singular_values"])
    assert s[-1] <= 1e-7 * s[0]


def test_null_rows_dropped():
    X = _spread(2000, 5, 13)
    cols = {f"x{i}": pa.array(X[:, i], mask=(np.arange(2000) % (7 + i) == 3)) for i in range(5)}
    df = Frame(cols)
    names = list(cols)
    _check_vs_oracle(df, names)
    _check_vs_oracle(df, names, center=False)


def test_principal_components_matches_projection():
    X = _spread(20000, 10, 17)
    df = _frame(X)
    names = [f"x{i}" for i in range(10)]
    for k in (1, 3, 10):
        pcs = _pcs(df.select(pds.principal_components(*names, k=k))["pl_principal_components"])
        _, W = _pca(df.select(pds.pca(*names))["pl_pca"])
        Xc = np.column_stack(_inputs(df, pds.pca(*names))[0])
        ref_dev = Xc @ W[:k].T
        np.testing.assert_allclose(pcs, ref_dev, rtol=1e-12, atol=1e-12 * np.abs(ref_dev).max())
        ref = po.principal_components(list(Xc.T), k)
        np.testing.assert_allclose(pcs, ref, rtol=1e-9, atol=1e-9 * np.abs(ref).max())
    Xf = X.astype(np.float32)
    dff = _frame(Xf)
    pcs = _pcs(dff.select(pds.principal_components(*names, k=4, center=False))["pl_principal_components"])
    ref = po.principal_components([Xf[:, i].astype(np.float64) for i in range(10)], 4)
    np.testing.assert_allclose(pcs, ref, rtol=1e-9, atol=1e-9 * np.abs(ref).max())


def test_edge_cases():
    X = _spread(50, 4, 19)
    names = [f"x{i}" for i in range(4)]
    nulls = Frame({n: pa.array(X[:, i], mask=(np.arange(50) == 7)) for i, n in enumerate(names)})
    with pytest.raises(pds.PdsbError, match="Nulls are found in data and this method doesn't allow nulls."):
        nulls.select(pds.principal_components(*names, k=2))
    small = _frame(X[:2])
    pcs = _pcs(small.select(pds.principal_components(*names, k=3))["pl_principal_components"])
    assert pcs.shape == (2, 3) and np.isnan(pcs).all()
    # n < p: singular values follow the reference; pca and k <= n < p components are errors
    s = _sv(small.select(pds.singular_values(*names))["pl_singular_values"])
    Xc = X[:2] - X[:2].mean(axis=0)
    np.testing.assert_allclose(s[:1], po.singular_values(list(Xc.T))[:1], rtol=1e-9)
    assert len(s) == 2
    with pytest.raises(pds.PdsbError, match="rows < 4 features is not supported"):
        small.select(pds.pca(*names))
    with pytest.raises(pds.PdsbError, match="rows < 4 features is not supported"):
        small.select(pds.principal_components(*names, k=2))
    empty = _frame(X[:0])
    assert len(_sv(empty.select(pds.singular_values(*names, center=False))["pl_singular_values"])) == 0
    bad = X.copy()
    bad[10, 1] = np.nan
    for e in (pds.singular_values(*names, center=False), pds.pca(*names, center=False),
              pds.principal_components(*names, k=2, center=False)):
        with pytest.raises(pds.PdsbError, match="SVD algorithm did not converge."):
            _frame(bad).select(e)
    wide = _frame(_spread(300, 260, 1))
    with pytest.raises(pds.PdsbError, match="at most 259"):
        wide.select(pds.singular_values(*[f"x{i}" for i in range(260)]))


def test_device_layer_unaligned_f32():
    import torch

    X = _spread(1001, 5, 23).astype(np.float32)
    buf = torch.zeros(5 * 1002 + 1, dtype=torch.float32, device="cuda")
    view = buf[1:].view(5, 1002)
    view[:, :1001] = torch.from_numpy(np.ascontiguousarray(X.T)).cuda()
    sig = torch.zeros(5, dtype=torch.float64, device="cuda")
    V = torch.zeros(25, dtype=torch.float64, device="cuda")
    st = torch.zeros(2, dtype=torch.int32, device="cuda")
    L = pds.lib()
    assert L.pdsb_dev_pca_f32(view.data_ptr(), 1002, None, 1001, 5, sig.data_ptr(), V.data_ptr(), st.data_ptr(), None) == 0
    torch.cuda.synchronize()
    assert st.tolist() == [0, 5]
    s_ref, W_ref = po.pca([X[:, i].astype(np.float64) for i in range(5)])
    np.testing.assert_allclose(sig.cpu().numpy(), s_ref, rtol=1e-12)
    np.testing.assert_allclose(V.cpu().numpy().reshape(5, 5), W_ref, atol=1e-10)
    out = torch.zeros(1001 * 2, dtype=torch.float64, device="cuda")
    assert L.pdsb_dev_project_f32(view.data_ptr(), 1002, 1001, 5, V.data_ptr(), 2, out.data_ptr(), 1001, None) == 0
    torch.cuda.synchronize()
    ref = X.astype(np.float64) @ W_ref[:2].T
    np.testing.assert_allclose(out.cpu().numpy().reshape(2, 1001).T, ref, rtol=1e-9, atol=1e-9 * np.abs(ref).max())


def test_full_size_and_reproducible():
    rng = np.random.default_rng(29)
    X = (rng.standard_normal((1_000_000, 32)) * np.linspace(2.0, 0.1, 32)).astype(np.float32)
    df = _frame(X, np.float32)
    names = [f"x{i}" for i in range(32)]
    s, W = _check_vs_oracle(df, names)
    s2, W2 = _pca(df.select(pds.pca(*names))["pl_pca"])
    np.testing.assert_array_equal(s2, s)
    np.testing.assert_array_equal(W2, W)
    a = _pcs(df.select(pds.principal_components(*names, k=8))["pl_principal_components"])
    b = _pcs(df.select(pds.principal_components(*names, k=8))["pl_principal_components"])
    np.testing.assert_array_equal(a, b)
