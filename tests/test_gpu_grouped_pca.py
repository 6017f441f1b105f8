"""Grouped PCA on the H100 (K18): group_by().agg(singular_values / pca, fast=True) and
principal_components(...).over(key, fast=True) against Polars' per-group loop (fast=False) and against the NumPy oracle
(tests/pca_oracle.py) on each group's centred inputs, with test_gpu_pca.py's accuracy rule.  One CPU test shows that the
rule catches the S - n mu mu^T shortcut the device must not take."""
import numpy as np
import pyarrow as pa
import pytest

import polars_ds_extension_b200 as pds
from polars_ds_extension_b200 import _harness
from polars_ds_extension_b200.frame import Frame
from tests import pca_oracle as po

gpu = pytest.mark.gpu
SIZES = lambda p: sorted({1, 2, max(p - 1, 1), p, p + 1, 127, 128, 129, 1000, 8191, 8192, 8193, 16385, 20000})


def _dev():
    import torch

    from polars_ds_extension_b200 import device as dev
    return torch, dev


def _data(sizes, p, seed, mean_scale=1.0):
    """Rows of len(sizes) groups (group g: its own mean and column scales), interleaved in the frame."""
    rng = np.random.default_rng(seed)
    blocks, keys = [], []
    for g, n in enumerate(sizes):
        scale = np.linspace(3.0, 0.2, p) * (1.0 + 0.1 * g)
        blocks.append(rng.standard_normal((n, p)) * scale + mean_scale * rng.standard_normal(p) * (g + 1))
        keys.append(np.full(n, g))
    X, key = np.concatenate(blocks), np.concatenate(keys)
    perm = rng.permutation(len(key))
    return X[perm], key[perm]


def _frame(X, key, dtype):
    if dtype == "i64":
        cols = {f"x{i}": np.rint(X[:, i] * 100).astype(np.int64) for i in range(X.shape[1])}
    else:
        cols = {f"x{i}": X[:, i].astype(np.float32 if dtype == "f32" else np.float64) for i in range(X.shape[1])}
    return Frame(cols | {"g": key})


def _names(p):
    return [f"x{i}" for i in range(p)]


def _inputs(df, e):
    """The loop's (centred) plugin inputs of one group's frame as f64 columns and validity, for the oracle."""
    cols, valid = [], []
    for a in e.args:
        if a.lit_u32 is not None:
            continue
        arr = df._eval_arg(a).combine_chunks()
        valid.append(np.asarray(arr.is_valid().to_numpy(zero_copy_only=False), dtype=bool))
        cols.append(arr.cast(pa.float64()).fill_null(0).to_numpy(zero_copy_only=False))
    return cols, (valid if any((~v).any() for v in valid) else None)


def _sv_rule(s, ref):
    assert len(s) == len(ref)
    if len(ref) == 0:
        return
    big = ref >= 1e-3 * ref[0]
    np.testing.assert_allclose(s[big], ref[big], rtol=1e-9)


def _vec_rule(W, s_ref, W_ref):
    lam = s_ref ** 2
    gap = np.full(len(lam), np.inf)
    gap[:-1] = np.minimum(gap[:-1], lam[:-1] - lam[1:])
    gap[1:] = np.minimum(gap[1:], lam[:-1] - lam[1:])
    ok = gap >= 1e-2 * lam[0]
    np.testing.assert_allclose(W[ok], W_ref[ok], rtol=0, atol=1e-9)
    return ok


def _pca_lists(arr):
    """LargeList<Struct{singular_value, weight_vector}> -> per group (sigma [p], W [p x p])."""
    out = []
    for v in arr.to_pylist():
        out.append((np.array([d["singular_value"] for d in v]), np.array([d["weight_vector"] for d in v])))
    return out


def _pcs(res):
    return np.column_stack([res.field(i).to_numpy(zero_copy_only=False) for i in range(res.type.num_fields)])


def _loop_means_f32(sub, names):
    return np.array([np.float32(sub[c].drop_null().to_numpy().astype(np.float64).mean()) for c in names])


def _device_means(df, names, dtype):
    """The device's group means of the frame's rows in key order (first-seen), through the device entry."""
    torch, dev = _dev()
    uniq, gid = pds.frame._group_ids(df["g"].to_numpy())
    order, offsets = pds.frame._key_order(gid, len(uniq))
    td = torch.float32 if dtype == "f32" else torch.float64
    X = torch.tensor(np.stack([df[c].to_numpy()[order] for c in names]), dtype=td, device="cuda")
    mean, *_ = dev.grouped_pca(X, torch.tensor(offsets, device="cuda"), center=True)
    return mean.cpu().numpy()


@gpu
@pytest.mark.parametrize("center", [True, False])
@pytest.mark.parametrize("dtype", ["f64", "f32", "i64"])
@pytest.mark.parametrize("p", [1, 2, 3, 8, 31, 32, 33, 64])
def test_against_loop_and_oracle(p, dtype, center):
    sizes = SIZES(p)
    X, key = _data(sizes, p, seed=100 + p)
    df = _frame(X, key, dtype)
    names = _names(p)
    gb = df.group_by("g")
    uniq, gid = pds.frame._group_ids(key)
    if dtype == "f32" and center:
        dm = _device_means(df, names, dtype)
        for g in range(len(uniq)):
            np.testing.assert_array_equal(dm[g].astype(np.float32), _loop_means_f32(df.filter(gid == g), names))
    e = pds.singular_values(*names, center=center)
    fast = gb.agg(e, fast=True)["pl_singular_values"].to_pylist()
    loop = gb.agg(e, fast=False)["pl_singular_values"]
    assert len(fast) == len(uniq)
    full = [g for g in range(len(uniq)) if (gid == g).sum() >= p]
    for g in range(len(uniq)):
        s = np.asarray(fast[g])
        _sv_rule(s, np.asarray(loop[g][0].as_py()))
        cols, valid = _inputs(df.filter(gid == g), e)
        _sv_rule(s, po.singular_values(cols, valid))
    # pca on the groups with at least p rows (any other group is the loop's error, tested below)
    sub = df.filter(np.isin(gid, full))
    sgid = pds.frame._group_ids(sub["g"].to_numpy())[1]
    ep = pds.pca(*names, center=center)
    fp = _pca_lists(sub.group_by("g").agg(ep, fast=True)["pl_pca"])
    lp = sub.group_by("g").agg(ep, fast=False)["pl_pca"]
    fs = sub.group_by("g").agg(e, fast=True)["pl_singular_values"].to_pylist()
    for g in range(len(fp)):
        s, W = fp[g]
        np.testing.assert_array_equal(s, np.asarray(fs[g]))          # pca's sigma = singular_values', bit for bit
        ls = lp[g].field("singular_value").to_numpy(zero_copy_only=False)
        lW = np.array(lp[g].field("weight_vector").to_pylist())
        _sv_rule(s, ls)
        _vec_rule(W, ls, lW)
        cols, valid = _inputs(sub.filter(sgid == g), ep)
        s_ref, W_ref = po.pca(cols, valid)
        _sv_rule(s, s_ref)
        _vec_rule(W, s_ref, W_ref)


def _pc_check(df, names, key, k, center):
    e = pds.principal_components(*names, k=k, center=center)
    fast = _pcs(df.select(e.over("g", fast=True))["pl_principal_components"])
    loop = _pcs(df.select(e.over("g", fast=False))["pl_principal_components"])
    assert fast.shape == (len(key), k)
    uniq, gid = pds.frame._group_ids(key)
    for g in range(len(uniq)):
        rows = gid == g
        cols, _ = _inputs(df.filter(rows), e)
        if rows.sum() < k:
            assert np.isnan(fast[rows]).all() and np.isnan(loop[rows]).all()
            continue
        s_ref, W_ref = po.pca(cols)
        lam = s_ref ** 2
        if k < len(lam) and lam[k - 1] - lam[k] < 1e-2 * lam[0]:
            continue                                                # pc_k is not determined to the rule's accuracy
        if any(lam[j] - lam[j + 1] < 1e-2 * lam[0] for j in range(k - 1)):
            continue
        ref = po.principal_components(cols, k)
        for other in (ref, loop[rows]):
            tol = 1e-9 * np.max(np.abs(other))
            np.testing.assert_allclose(fast[rows], other, rtol=1e-9, atol=tol)


@gpu
@pytest.mark.parametrize("center", [True, False])
@pytest.mark.parametrize("dtype", ["f64", "f32", "i64"])
@pytest.mark.parametrize("p", [1, 2, 3, 8, 31, 32, 33, 64])
def test_principal_components_over(p, dtype, center):
    k = min(2, p)
    sizes = sorted({1, p, p + 1, 128, 1000, 8193, 16385}) if k > 1 else [1, 2, 128, 8193]
    X, key = _data(sizes, p, seed=200 + p)
    _pc_check(_frame(X, key, dtype), _names(p), key, k, center)


@gpu
def test_large_group_means():
    p, n_g = 6, 3000
    rng = np.random.default_rng(5)
    X = np.concatenate([rng.standard_normal((n_g, p)) * np.linspace(1.0, 0.1, p) + 1e4 * (g + 1) for g in range(6)])
    key = np.repeat(np.arange(6), n_g)
    df = _frame(X, key, "f64")
    e = pds.singular_values(*_names(p), center=True)
    fast = df.group_by("g").agg(e, fast=True)["pl_singular_values"].to_pylist()
    for g in range(6):
        cols, _ = _inputs(df.filter(key == g), e)
        _sv_rule(np.asarray(fast[g]), po.singular_values(cols))
    _pc_check(df, _names(p), key, 2, True)


def test_shortcut_gram_fails_the_rule_cpu():
    """S - n mu mu^T in f64 on the large-mean data: the error the two-pass centred Gram exists to avoid."""
    p, n_g = 6, 3000
    rng = np.random.default_rng(5)
    X = np.concatenate([rng.standard_normal((n_g, p)) * np.linspace(1.0, 0.1, p) + 1e4 * (g + 1) for g in range(6)])
    failed = 0
    for g in range(6):
        Z = X[g * n_g:(g + 1) * n_g]
        mu = Z.mean(axis=0)
        G = Z.T @ Z - n_g * np.outer(mu, mu)
        s = np.sqrt(np.maximum(np.linalg.eigvalsh(G)[::-1], 0.0))
        ref = po.singular_values([Z[:, c] - mu[c] for c in range(p)])
        try:
            _sv_rule(s, ref)
        except AssertionError:
            failed += 1
    assert failed == 6


@gpu
@pytest.mark.parametrize("dtype", ["f64", "f32"])
def test_nulls(dtype):
    p = 4
    X, key = _data([50, 300, 9000], p, seed=9)
    df = _frame(X, key, dtype)
    rng = np.random.default_rng(3)
    cols = {}
    for i, c in enumerate(_names(p)):
        v = df[c].combine_chunks().to_numpy(zero_copy_only=False)
        cols[c] = pa.array(v, mask=rng.random(len(v)) < 0.05 * (i + 1))
    dn = Frame(cols | {"g": key})
    uniq, gid = pds.frame._group_ids(key)
    for center in (True, False):
        e = pds.singular_values(*_names(p), center=center)
        fast = dn.group_by("g").agg(e, fast=True)["pl_singular_values"].to_pylist()
        loop = dn.group_by("g").agg(e, fast=False)["pl_singular_values"]
        ep = pds.pca(*_names(p), center=center)
        fp = _pca_lists(dn.group_by("g").agg(ep, fast=True)["pl_pca"])
        for g in range(len(uniq)):
            _sv_rule(np.asarray(fast[g]), np.asarray(loop[g][0].as_py()))
            c_, v_ = _inputs(dn.filter(gid == g), e)
            _sv_rule(np.asarray(fast[g]), po.singular_values(c_, v_))
            s_ref, W_ref = po.pca(c_, v_)
            _vec_rule(fp[g][1], s_ref, W_ref)
    with pytest.raises(pds.PdsbError, match="Nulls are found in data and this method doesn't allow nulls."):
        dn.select(pds.principal_components(*_names(p), k=2).over("g", fast=True))


@gpu
def test_device_layer_mask():
    """A masked row leaves the Gram; its NaN values are nulls for the means, its other values count."""
    torch, dev = _dev()
    rng = np.random.default_rng(4)
    X = rng.standard_normal((3, 500)) + 5.0
    m = rng.random(500) > 0.2
    nulls = (rng.random((3, 500)) < 0.1) & ~m
    Xn = np.where(nulls, np.nan, X)
    offs = np.array([0, 200, 500])
    mean, sigma, V, st = dev.grouped_pca(torch.tensor(Xn, device="cuda"), torch.tensor(offs, device="cuda"), True,
                                         mask=torch.tensor(m.astype(np.float64), device="cuda"))
    st = st.cpu().numpy()
    for g in range(2):
        sl = slice(offs[g], offs[g + 1])
        mu = np.array([np.nanmean(Xn[c, sl]) for c in range(3)])
        np.testing.assert_allclose(mean.cpu().numpy()[g], mu, rtol=1e-14)
        keep = m[sl]
        ref = po.singular_values([X[c, sl][keep] - mu[c] for c in range(3)])
        _sv_rule(sigma.cpu().numpy()[g], ref)
        assert st[g, 0] == 0 and st[g, 1] == 3


def _err(fn):
    with pytest.raises(pds.PdsbError) as ei:
        fn()
    return str(ei.value)


@gpu
def test_semantics_table():
    p = 3
    X, key = _data([10, 2, 40], p, seed=1)         # group 1: 2 rows < 3 features
    df = _frame(X, key, "f64")
    names = _names(p)
    # pca with fewer rows than features in a group: the loop's error, for the whole call
    ep = pds.pca(*names)
    msg = _err(lambda: df.group_by("g").agg(ep, fast=True))
    assert "pca: 2 rows < 3 features is not supported" in msg
    assert msg == _err(lambda: df.group_by("g").agg(ep, fast=False))
    # principal_components: k <= n < p is the single call's error; n < k gives NaN rows
    msg = _err(lambda: df.select(pds.principal_components(*names, k=2).over("g", fast=True)))
    assert "principal_components: 2 rows < 3 features is not supported" in msg
    assert msg == _err(lambda: df.select(pds.principal_components(*names, k=2).over("g", fast=False)))
    X1, key1 = _data([10, 1, 40], p, seed=2)
    d1 = _frame(X1, key1, "f64")
    pcs = _pcs(d1.select(pds.principal_components(*names, k=2).over("g", fast=True))["pl_principal_components"])
    uniq, gid = pds.frame._group_ids(key1)
    lone = gid == gid[key1 == 1][0]
    assert np.isnan(pcs[lone]).all() and np.isfinite(pcs[~lone]).all()
    # singular_values of an empty group: an empty list
    cols = [pa.array(X[:12, c]) for c in range(p)]
    out = _harness.call_plugin("pl_singular_values_by", [pa.array(np.array([0, 0, 12, 12], dtype=np.int64))] + cols,
                               ["__offsets__"] + names, {"center": True})
    v = out.to_pylist()
    assert v[0] == [] and len(v[1]) == 3 and v[2] == []
    # a NaN or inf in a kept row: "SVD algorithm did not converge.", as the loop raises it (K5's moments would drop it)
    for bad in (np.nan, np.inf):
        Xb = X.copy()
        Xb[np.flatnonzero(key == 2)[3], 1] = bad
        db = _frame(Xb, key, "f64")
        e = pds.singular_values(*names)
        msg = _err(lambda: db.group_by("g").agg(e, fast=True))
        assert "SVD algorithm did not converge." in msg
        assert "SVD algorithm did not converge." in _err(lambda: db.group_by("g").agg(e, fast=False))
    # more than 64 features
    wide = Frame({f"x{i}": np.arange(100.0) * (i + 1) % 7 for i in range(65)} | {"g": np.arange(100) % 2})
    assert "at most 64" in _err(lambda: wide.group_by("g").agg(pds.singular_values(*_names(65)), fast=True))


@gpu
@pytest.mark.parametrize("dtype", ["f64", "f32"])
def test_explained_var_and_ratio(dtype):
    p = 5
    X, key = _data([3, 40, 1000, 9000], p, seed=8)
    df = _frame(X, key, dtype)
    for kw in ({"as_explained_var": True}, {"as_ratio": True}, {"as_explained_var": True, "as_ratio": True}):
        e = pds.singular_values(*_names(p), **kw)
        fast = df.group_by("g").agg(e, fast=True)["pl_singular_values"].to_pylist()
        loop = df.group_by("g").agg(e, fast=False)["pl_singular_values"]
        for g in range(len(fast)):
            ref = np.asarray(loop[g][0].as_py())
            np.testing.assert_allclose(fast[g], ref, rtol=1e-9, atol=1e-9 * np.max(np.abs(ref)))


@gpu
@pytest.mark.parametrize("dtype", ["f64", "f32"])
def test_group_independent_of_batch(dtype):
    p, k = 5, 2
    sizes = [7, 300, 9000, 20000, 128]
    X, key = _data(sizes, p, seed=12)
    order = np.argsort(key, kind="stable")
    Xs = X[order].astype(np.float32 if dtype == "f32" else np.float64)
    offs = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    names = ["__offsets__"] + _names(p)

    def run(sym, rows, offsets):
        ins = [pa.array(offsets)] + ([pa.array([k], type=pa.uint32())] if sym == "pl_principal_components_by" else [])
        ins += [pa.array(Xs[rows, c]) for c in range(p)]
        nm = names[:1] + (["literal"] if sym == "pl_principal_components_by" else []) + names[1:]
        return _harness.call_plugin(sym, ins, nm, {"center": True})

    whole = slice(0, len(key))
    sv = run("pl_singular_values_by", whole, offs).to_pylist()
    pc = _pcs(run("pl_principal_components_by", whole, offs))
    pca = _pca_lists(run("pl_pca_by", whole, offs))
    # the same groups in another order inside the batch
    perm = [3, 0, 4, 2, 1]
    rows2 = np.concatenate([np.arange(offs[g], offs[g + 1]) for g in perm])
    offs2 = np.concatenate([[0], np.cumsum([sizes[g] for g in perm])]).astype(np.int64)
    sv2 = run("pl_singular_values_by", rows2, offs2).to_pylist()
    for g in range(len(sizes)):
        rows = slice(offs[g], offs[g + 1])
        one = np.array([0, sizes[g]], dtype=np.int64)
        assert run("pl_singular_values_by", rows, one).to_pylist()[0] == sv[g]
        assert sv2[perm.index(g)] == sv[g]
        s1, W1 = _pca_lists(run("pl_pca_by", rows, one))[0]
        np.testing.assert_array_equal(s1, pca[g][0])
        np.testing.assert_array_equal(W1, pca[g][1])
        np.testing.assert_array_equal(_pcs(run("pl_principal_components_by", rows, one)), pc[rows])


@gpu
@pytest.mark.parametrize("center", [True, False])
def test_device_layer_f32_odd_ld(center):
    torch, dev = _dev()
    p, k = 7, 3
    sizes = [1, 9, 700, 8200]
    n = sum(sizes)
    X, _ = _data(sizes, p, seed=21)
    Xs = X.astype(np.float32)          # rows cut into groups of `sizes` in frame order
    store = torch.zeros((p, n + 3), dtype=torch.float32, device="cuda")
    store[:, :n] = torch.tensor(Xs.T, device="cuda")
    Xt = store[:, :n]
    assert Xt.stride(0) % 4 != 0
    offs = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    doffs = torch.tensor(offs, device="cuda")
    mean, sigma, V, st = dev.grouped_pca(Xt, doffs, center=center)
    out = dev.grouped_project(Xt, doffs, V, k, mean=mean).cpu().numpy().T
    sigma, V, st = sigma.cpu().numpy(), V.cpu().numpy(), st.cpu().numpy()
    for g in range(len(sizes)):
        Z = Xs[offs[g]:offs[g + 1]].astype(np.float64)
        if center:
            mu = np.float32(Z.mean(axis=0))
            np.testing.assert_array_equal(mean.cpu().numpy()[g].astype(np.float32), mu)
            Z = (Xs[offs[g]:offs[g + 1]] - mu).astype(np.float64)
        cols = [Z[:, c] for c in range(p)]
        dim = min(sizes[g], p)
        assert st[g, 0] == 0 and st[g, 1] == dim
        ref = po.singular_values(cols)
        _sv_rule(sigma[g][:dim], ref)
        if sizes[g] < k:
            assert np.isnan(out[offs[g]:offs[g + 1]]).all()
        elif sizes[g] >= p:
            s_ref, W_ref = po.pca(cols)
            ok = _vec_rule(V[g].T, s_ref, W_ref)
            if ok[:k].all():
                ref_pc = po.principal_components(cols, k)
                np.testing.assert_allclose(out[offs[g]:offs[g + 1]], ref_pc, rtol=1e-9,
                                           atol=1e-9 * np.max(np.abs(ref_pc)))


@gpu
def test_scale():
    torch, dev = _dev()
    rng = np.random.default_rng(31)
    # 1e5 groups of 3 rows at p = 2, through the plugin
    ng, p = 100_000, 2
    X = rng.standard_normal((3 * ng, p)) * [2.0, 0.5] + rng.standard_normal((ng, 1)).repeat(3, axis=0)
    offs = np.arange(0, 3 * ng + 1, 3, dtype=np.int64)
    sv = _harness.call_plugin("pl_singular_values_by", [pa.array(offs)] + [pa.array(X[:, c]) for c in range(p)],
                              ["__offsets__", "x0", "x1"], {"center": True}).to_pylist()
    assert len(sv) == ng
    for g in rng.choice(ng, 200, replace=False):
        Z = X[3 * g:3 * g + 3]
        _sv_rule(np.asarray(sv[g]), po.singular_values([Z[:, c] - Z[:, c].mean() for c in range(p)]))
    # one call over 1e7 rows (the item count read back from the device), f32 on the device entry
    sizes = [5_000_000, 3, 2_999_990, 7, 2_000_000]
    n = sum(sizes)
    Xb = (rng.standard_normal((p, n)) * np.array([[3.0], [0.3]]) + 1e3).astype(np.float32)
    offs = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    mean, sigma, V, st = dev.grouped_pca(torch.tensor(Xb, device="cuda"), torch.tensor(offs, device="cuda"), True)
    mean, sigma, st = mean.cpu().numpy(), sigma.cpu().numpy(), st.cpu().numpy()
    for g in range(len(sizes)):
        Z = Xb[:, offs[g]:offs[g + 1]]
        mu = mean[g].astype(np.float32)
        assert st[g, 0] == 0 and st[g, 1] == min(sizes[g], p)
        ref = po.singular_values([(Z[c] - mu[c]).astype(np.float64) for c in range(p)])
        _sv_rule(sigma[g][:len(ref)], ref)
