"""MixedModel on the GPU against the REML oracle (tests/mixed_oracle.py).

The lifted case is the data of the reference's test_mixed_model_recovers_fixed_effect (RandomState(42), 40 groups x 25
rows), checked with that test's own thresholds.  Parity with the oracle is 1e-6 relative on gamma, beta, the standard
errors and the residual variance: near the optimum the golden section's comparisons turn on last-bit differences of a
flat deviance, so the device may stop at a slightly different gamma; its deviance is checked to be as good.  Data with
large column offsets are compared with the oracle on the unshifted data (see test_parity_large_offsets)."""
import ctypes as C

import numpy as np
import pytest

from tests.mixed_oracle import deviance, fit_reml, lifted_case

pytestmark = pytest.mark.gpu


def _rel(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return float(np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-300))


def _prepare(d, features, null_policy="skip"):
    from polars_ds_extension_b200.linear_models import _columns_of, _group_column, _mixed_inputs

    keys, key_null = _group_column(d, "group")
    return _mixed_inputs(_columns_of(d, list(features) + ["y"]), keys, key_null, null_policy)


def _col(frame, name):
    """A column of report() as a list, for a polars DataFrame or this package's Frame."""
    c = frame[name]
    return c.to_list() if hasattr(c, "to_list") else c.to_pylist()


def _check_parity(d, features, ranks="dense"):
    from polars_ds_extension_b200.linear_models import _mixed_fit

    X, y, codes, G, between = _prepare(d, features)
    ref = fit_reml(X, y, codes, G, between, ranks=ranks)
    coeffs, se, dfs, gamma, rv, _ = _mixed_fit(X, y, codes, G, between, 200, 1e-10)
    assert abs(gamma - ref["gamma"]) <= 1e-6 * max(abs(ref["gamma"]), 1e-6)
    assert _rel(coeffs, ref["coeffs"]) < 1e-6
    assert _rel(se, ref["std_errors"]) < 1e-6
    assert abs(rv - ref["resid_variance"]) < 1e-6 * ref["resid_variance"]
    assert np.array_equal(dfs, ref["dfs"])
    d_dev, d_ref = deviance(X, y, codes, G, gamma), deviance(X, y, codes, G, ref["gamma"])
    assert d_dev <= d_ref + 1e-12 * abs(d_ref)
    return X, y, codes, G, between


def _case(kind, seed=0):
    rng = np.random.default_rng(seed)
    if kind == "balanced":
        G, m = 30, 12
        g = np.repeat(np.arange(G), m)
    else:
        G = 50
        g = np.repeat(np.arange(G), rng.integers(1, 30, G))
    n = g.size
    u = rng.normal(0.0, {"none": 0.0, "strong": 5.0}.get(kind, 1.0), G)[g]
    x1, x2 = rng.normal(size=n), rng.normal(size=n)
    w = rng.normal(size=G)[g]                                   # a group-level (between) covariate
    y = 0.5 + 1.5 * x1 - 0.7 * x2 + 0.3 * w + u + rng.normal(size=n)
    return {"y": y, "x1": x1, "x2": x2, "w": w, "group": g}


def test_lifted_reference_case():
    from polars_ds_extension_b200.frame import Frame
    from polars_ds_extension_b200.linear_models import MixedModel

    d = lifted_case()
    mm = MixedModel().fit_df(Frame(d), features=["x", "noise"], target="y", group="group")
    assert mm.is_fit()
    rep = mm.report()
    assert _col(rep, "effect") == ["Intercept", "x", "noise"]
    b0, b1, _ = _col(rep, "estimate")
    assert abs(b0 - 1.5) < 0.5 and abs(b1 - 2.0) < 0.2
    p = _col(rep, "p_value")
    assert p[1] < 1e-6 and p[2] > 0.05
    assert mm.gamma_ > 0.0 and np.all(mm.dfs_ > 0)
    assert repr(mm).startswith("MixedModel(Random Intercept, REML)\nGroup: group\n")
    _check_parity(d, ["x", "noise"])


@pytest.mark.parametrize("kind", ["balanced", "unbalanced", "none", "strong"])
def test_parity(kind):
    _check_parity(_case(kind), ["x1", "x2", "w"])


@pytest.mark.parametrize("seed", [7, 8, 9])
@pytest.mark.parametrize("offset", ["y", "x1", "both"])
def test_parity_large_offsets(offset, seed):
    """A target and/or a within-varying feature shifted by 1e4 is the same model (the intercept absorbs the shift), so
    the device fit on the shifted data must match the oracle on the unshifted data at the parity tolerance.  The oracle
    is not run on the shifted data: the reference's own arithmetic (y - X beta after x'(x - gamma/(1+gamma n) s))
    moves gamma by up to ~3e-5 there, while the device centres every column before the search."""
    from polars_ds_extension_b200.linear_models import _mixed_fit

    X, y, codes, G, between = _prepare(_case("unbalanced", seed), ["x1", "x2", "w"])
    ref = fit_reml(X, y, codes, G, between)
    Xs, ys = X.copy(), y.copy()
    if offset in ("y", "both"):
        ys += 1e4
    if offset in ("x1", "both"):
        Xs[:, 1] += 1e4
    coeffs, se, dfs, gamma, rv, _ = _mixed_fit(Xs, ys, codes, G, between, 200, 1e-10)
    b0 = ref["coeffs"][0] + (1e4 if offset != "x1" else 0.0) - (1e4 * ref["coeffs"][1] if offset != "y" else 0.0)
    assert abs(gamma - ref["gamma"]) <= 1e-6 * ref["gamma"]
    assert abs(rv - ref["resid_variance"]) <= 1e-6 * ref["resid_variance"]
    assert _rel(coeffs[1:], ref["coeffs"][1:]) < 1e-6 and _rel(se[1:], ref["std_errors"][1:]) < 1e-6
    assert abs(coeffs[0] - b0) <= 1e-6 * abs(b0)
    assert np.array_equal(dfs, ref["dfs"])
    d_dev, d_ref = deviance(X, y, codes, G, gamma), deviance(X, y, codes, G, ref["gamma"])
    assert d_dev <= d_ref + 1e-12 * abs(d_ref)


def test_shuffled_rows_and_string_keys():
    d = _case("unbalanced", 3)
    perm = np.random.default_rng(1).permutation(d["y"].size)
    s = {k: v[perm] for k, v in d.items()}
    s["group"] = np.array([f"g{v:03d}" for v in s["group"]], dtype=object)
    _check_parity(s, ["x1", "x2", "w"])


def test_bit_reproducible_and_row_order():
    from polars_ds_extension_b200.linear_models import _mixed_fit

    X, y, codes, G, between = _prepare(_case("unbalanced", 5), ["x1", "x2", "w"])
    a = _mixed_fit(X, y, codes, G, between, 200, 1e-10)
    b = _mixed_fit(X, y, codes, G, between, 200, 1e-10)
    for u, v in zip(a, b):
        assert np.array_equal(u, v)
    perm = np.random.default_rng(2).permutation(y.size)
    c = _mixed_fit(X[perm], y[perm], codes[perm], G, between, 200, 1e-10)
    for u, v in zip(a[:5], c[:5]):
        assert _rel(u, v) <= 1e-6


@pytest.mark.parametrize("column", ["x1", "y"])
def test_shifted_column(column):
    """Shifting a within-varying feature, or the target, by 1e4 is a reparametrisation: gamma, sigma^2, the slopes
    and their standard errors stay put (the intercept absorbs the shift)."""
    from polars_ds_extension_b200.linear_models import _mixed_fit

    X, y, codes, G, between = _prepare(_case("unbalanced", 7), ["x1", "x2", "w"])
    a = _mixed_fit(X, y, codes, G, between, 200, 1e-10)
    Xs, ys = X.copy(), y.copy()
    if column == "x1":
        Xs[:, 1] += 1e4
    else:
        ys += 1e4
    b = _mixed_fit(Xs, ys, codes, G, between, 200, 1e-10)
    assert np.array_equal(a[2], b[2])
    assert abs(a[3] - b[3]) <= 1e-6 * a[3] and abs(a[4] - b[4]) <= 1e-6 * a[4]
    assert _rel(a[0][1:], b[0][1:]) <= 1e-6 and _rel(a[1][1:], b[1][1:]) <= 1e-6


def test_launches_do_not_depend_on_max_iter():
    from polars_ds_extension_b200._lib import lib
    from polars_ds_extension_b200.linear_models import _mixed_fit

    X, y, codes, G, between = _prepare(_case("balanced"), ["x1", "x2"])
    counts = []
    for it in (5, 200):
        c0 = lib().pdsb_kernel_launch_count()
        _, _, _, _, _, evals = _mixed_fit(X, y, codes, G, between, it, 1e-10)
        counts.append(lib().pdsb_kernel_launch_count() - c0)
        if it == 5:
            assert evals == 8          # two to start, one per step, one at the optimum
    assert counts[0] == counts[1]


def test_errors():
    from polars_ds_extension_b200._lib import Matrix, lib
    from polars_ds_extension_b200.linear_models import _mixed_fit, _view

    X, y, codes, G, between = _prepare(_case("balanced"), ["x1", "x2"])
    with pytest.raises(ValueError, match="same number of rows"):
        _mixed_fit(X, y[:-1], codes, G, between, 200, 1e-10)
    # the C entry point itself checks the shapes
    Xc, yc = np.ascontiguousarray(X), np.ascontiguousarray(y[:-1].reshape(-1, 1))
    out = [np.empty(3) for _ in range(3)]
    g, rv = C.c_double(), C.c_double()
    b = np.asarray(between, dtype=np.int64)
    rc = lib().pdsb_mixed_fit(C.byref(_view(Xc)), C.byref(_view(yc)), codes.ctypes.data, G, b.ctypes.data, b.size, 200,
                              1e-10, out[0].ctypes.data, out[1].ctypes.data, out[2].ctypes.data, C.addressof(g),
                              C.addressof(rv), None)
    assert rc != 0 and b"same number of rows" in lib().pdsb_last_error()
    with pytest.raises(ValueError, match="Not enough rows to fit a mixed model"):
        _mixed_fit(X[:3], y[:3], codes[:3], G, [0], 200, 1e-10)
    Xz = X.copy()
    Xz[:, 2] = 0.0
    with pytest.raises(ValueError, match=r"X'HiX is not positive definite; design may be rank-deficient\."):
        _mixed_fit(Xz, y, codes, G, between, 200, 1e-10)
    bad = codes.copy()
    bad[3] = G
    with pytest.raises(ValueError, match=r"Group codes must lie in \[0, n_groups\)"):
        _mixed_fit(X, y, bad, G, between, 200, 1e-10)
    Xw = np.random.default_rng(0).normal(size=(400, 65))
    with pytest.raises(ValueError, match="1 to 64 fixed effects"):
        _mixed_fit(Xw, Xw[:, 0], np.arange(400) % 7, 7, [0], 200, 1e-10)


def test_large_unsorted_structure_ranks():
    from polars_ds_extension_b200.linear_models import _mixed_fit

    rng = np.random.default_rng(11)
    G = 10_000
    g = np.repeat(np.arange(G), rng.integers(50, 151, G))
    n = g.size
    perm = rng.permutation(n)
    g = g[perm]
    feats = rng.normal(size=(n, 16))
    feats[:, 0] = rng.normal(size=G)[g]                         # the between feature
    y = feats @ np.linspace(-1.0, 1.0, 16) + rng.normal(size=G)[g] + rng.normal(size=n)
    d = {f"x{j}": feats[:, j] for j in range(16)} | {"y": y, "group": g}
    X, y, codes, G2, between = _prepare(d, [f"x{j}" for j in range(16)])
    assert G2 == G and between == [0, 1]
    _check_parity(d, [f"x{j}" for j in range(16)], ranks="structure")
    dfs = _mixed_fit(X, y, codes, G, between, 200, 1e-10)[2]
    assert np.array_equal(dfs, np.array([G - 2, G - 2] + [n - G - 15] * 15, dtype=np.float64))
