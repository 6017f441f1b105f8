"""MixedModel without a GPU: the REML oracle (tests/mixed_oracle.py) against closed forms and an independent dense
REML, the lifted reference test's assertions on the oracle, `fit_df`'s data preparation against a per-group loop,
and the report's p-values against SciPy."""
import numpy as np
import pytest
import scipy.optimize as so
import scipy.stats as st

from tests.mixed_oracle import fit_reml, lifted_case


def test_oracle_balanced_anova_closed_form():
    rng = np.random.default_rng(3)
    G, m = 20, 8
    g = np.repeat(np.arange(G), m)
    y = 2.0 + rng.normal(0.0, 1.5, G)[g] + rng.normal(size=G * m)
    means = np.bincount(g, weights=y) / m
    msb = m * np.sum((means - y.mean()) ** 2) / (G - 1)
    msw = np.sum((y - means[g]) ** 2) / (G * (m - 1))
    assert msb > msw
    r = fit_reml(np.ones((G * m, 1)), y, g, G, [0])
    assert r["gamma"] == pytest.approx((msb - msw) / (m * msw), rel=1e-6)
    assert r["resid_variance"] == pytest.approx(msw, rel=1e-6)
    assert r["std_errors"][0] ** 2 == pytest.approx(msb / (G * m), rel=1e-6)
    assert r["coeffs"][0] == pytest.approx(y.mean(), rel=1e-12)
    assert r["dfs"].tolist() == [G - 1]


def test_oracle_against_dense_reml():
    rng = np.random.default_rng(4)
    G = 30
    g = np.repeat(np.arange(G), rng.integers(5, 16, G))
    n = g.size
    X = np.column_stack([np.ones(n), rng.normal(size=n), rng.normal(size=n)])
    y = X @ np.array([1.0, 0.5, -0.3]) + rng.normal(0.0, 0.8, G)[g] + rng.normal(size=n)
    Zd = np.zeros((n, G))
    Zd[np.arange(n), g] = 1.0
    p = X.shape[1]

    def dense(gam):
        V = np.eye(n) + gam * Zd @ Zd.T
        Vi = np.linalg.inv(V)
        A = X.T @ Vi @ X
        beta = np.linalg.solve(A, X.T @ Vi @ y)
        r = y - X @ beta
        s2 = r @ Vi @ r / (n - p)
        return (n - p) * np.log(s2) + np.linalg.slogdet(V)[1] + np.linalg.slogdet(A)[1], beta, s2, A

    opt = so.minimize_scalar(lambda t: dense(t)[0], bounds=(0.0, 100.0), method="bounded",
                             options={"xatol": 1e-12})
    _, beta, s2, A = dense(opt.x)
    r = fit_reml(X, y, g, G, [0])
    assert r["gamma"] == pytest.approx(opt.x, rel=1e-5)
    np.testing.assert_allclose(r["coeffs"], beta, rtol=1e-6)
    assert r["resid_variance"] == pytest.approx(s2, rel=1e-6)
    np.testing.assert_allclose(r["std_errors"], np.sqrt(s2 * np.diag(np.linalg.inv(A))), rtol=1e-5)
    assert r["dfs"].tolist() == [G - 1, n - G - 2, n - G - 2]


def test_oracle_meets_lifted_reference_test():
    d = lifted_case()
    n = d["y"].size
    X = np.column_stack([np.ones(n), d["x"], d["noise"]])
    r = fit_reml(X, d["y"], d["group"], 40, [0])
    assert abs(r["coeffs"][0] - 1.5) < 0.5 and abs(r["coeffs"][1] - 2.0) < 0.2
    t = r["coeffs"] / r["std_errors"]
    pv = 2.0 * st.t.sf(np.abs(t), r["dfs"])
    assert pv[1] < 1e-6 and pv[2] > 0.05
    assert r["gamma"] > 0.0 and np.all(r["dfs"] > 0)


def _naive_prepare(F, y, keys, null_policy):
    rows = []
    for i in range(len(y)):
        f = F[i].copy()
        if keys[i] is None:
            continue
        if null_policy == "skip" and (np.isnan(f).any() or np.isnan(y[i])):
            continue
        if null_policy in ("zero", "one", "2.5"):
            if np.isnan(y[i]):
                continue
            f[np.isnan(f)] = {"zero": 0.0, "one": 1.0, "2.5": 2.5}[null_policy]
        rows.append((f, y[i], keys[i]))
    uniq = sorted({k for _, _, k in rows})
    codes = np.array([uniq.index(k) for _, _, k in rows])
    F2 = np.array([f for f, _, _ in rows])
    between = [0]
    for j in range(F.shape[1]):
        if all(len({F2[i, j] for i in range(len(rows)) if codes[i] == c}) == 1 for c in range(len(uniq))):
            between.append(j + 1)
    return np.column_stack([np.ones(len(rows)), F2]), np.array([v for _, v, _ in rows]), codes, len(uniq), between


@pytest.mark.parametrize("null_policy", ["skip", "zero", "one", "2.5", "ignore"])
def test_prepare_against_naive_loop(null_policy):
    from polars_ds_extension_b200.linear_models import _group_column, _mixed_inputs

    rng = np.random.default_rng(5)
    n = 300
    keys = np.array([f"k{v}" for v in rng.integers(0, 25, n)], dtype=object)
    keys[rng.random(n) < 0.05] = None                              # null groups are dropped
    gl = np.array([int(k[1:]) % 7 if k is not None else 0 for k in keys], dtype=np.float64)   # constant within groups
    F = np.column_stack([rng.normal(size=n), gl, rng.normal(size=n)])
    y = rng.normal(size=n)
    if null_policy != "ignore":
        F[rng.random(n) < 0.05, 0] = np.nan
        y[rng.random(n) < 0.03] = np.nan
    vals, null = _group_column({"g": keys}, "g")
    X, yy, codes, G, between = _mixed_inputs(np.column_stack([F, y]), vals, null, null_policy)
    X2, y2, c2, G2, b2 = _naive_prepare(F, y, keys, null_policy)
    np.testing.assert_array_equal(X, X2)
    np.testing.assert_array_equal(yy, y2)
    np.testing.assert_array_equal(codes, c2)
    assert G == G2 and between == b2
    assert 2 in between and 1 not in between


def test_prepare_raise_and_integer_keys():
    from polars_ds_extension_b200.linear_models import _mixed_inputs

    Z = np.array([[1.0, 2.0], [np.nan, 3.0], [2.0, 4.0]])
    keys = np.array([10, 3, 10])
    with pytest.raises(ValueError, match="Nulls found in Dataframe."):
        _mixed_inputs(Z, keys, np.zeros(3, dtype=bool), "raise")
    X, y, codes, G, between = _mixed_inputs(Z, keys, np.zeros(3, dtype=bool), "skip")
    assert codes.tolist() == [0, 0] and G == 1 and between == [0]
    X, y, codes, G, between = _mixed_inputs(Z, keys, np.array([False, True, False]), "raise")   # the null row's group is null
    assert codes.tolist() == [0, 0] and between == [0]


def test_arrow_key_columns():
    """Arrow string and integer keys (the package's Frame) give the codes of the plain object / numpy path."""
    import pyarrow as pa

    from polars_ds_extension_b200.frame import Frame
    from polars_ds_extension_b200.linear_models import _group_column, _mixed_inputs

    rng = np.random.default_rng(6)
    n = 500
    words = [f"w{v}" if v % 11 else None for v in rng.integers(0, 60, n)]
    ints = [int(v) if v % 13 else None for v in rng.integers(-40, 40, n)]
    Z = rng.normal(size=(n, 2))
    frame = Frame({"s": pa.array(words), "i": pa.array(ints, type=pa.int64())})
    for name, plain in (("s", np.array(words, dtype=object)), ("i", np.array(ints, dtype=object))):
        k1, n1 = _group_column(frame, name)
        k2, n2 = _group_column({name: plain}, name)
        np.testing.assert_array_equal(n1, n2)
        keep = ~n2
        _, ref = np.unique(plain[keep].astype(str if name == "s" else np.int64), return_inverse=True)
        a = _mixed_inputs(Z, k1, n1, "skip")
        np.testing.assert_array_equal(a[2], ref.ravel())
        assert a[3] == ref.max() + 1


def test_unfitted_model():
    from polars_ds_extension_b200.linear_models import MixedModel

    m = MixedModel()
    assert not m.is_fit() and repr(m) == "MixedModel (not fitted yet)"
    assert m.coeffs_.size == 0 and m.std_errors_.size == 0 and m.dfs_.size == 0
    assert m.gamma_ == 0.0 and m.resid_variance_ == 0.0
    with pytest.raises(ValueError, match="Model is not fit yet."):
        m.report()


def test_two_sided_p_values():
    from polars_ds_extension_b200.linear_models import _two_sided_p

    t = np.array([0.0, 0.5, -1.7, 2.5, 8.0, -40.0])
    df = np.array([1.0, 3.0, 10.0, 39.0, 958.0, 5.0])
    np.testing.assert_allclose(_two_sided_p(t, df), np.clip(2.0 * st.t.sf(np.abs(t), df), 0, 1), rtol=1e-10, atol=1e-300)
