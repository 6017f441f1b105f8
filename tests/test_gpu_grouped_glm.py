"""GLM.fit_by / fit_df_by and pdsb_dev_grouped_glm_f64 on the GPU: every group against the loop of GLM.fit over the
groups and against the IRLS oracle (tests/glm_oracle.py), on data generated here.

The grouped fit sums its moments per warp and solves with K5's group_solve, the single fit sums them on the tensor cores
and solves with K3, so the two agree to rounding: 1e-9 relative in the max-norm, the tolerance test_gpu_glm.py holds the
single fit to.  Iteration counts are equal.  tol is 1e-8: IRLS converges quadratically, so a group's last two steps lie
decades either side of it on this data."""
import numpy as np
import pytest

from tests.glm_oracle import faer_irls

pytestmark = pytest.mark.gpu

FAMILIES = ("gaussian", "poisson", "binomial", "gamma")
FAMILY_IDS = {"gaussian": 0, "poisson": 1, "binomial": 2, "gamma": 3}
TOL = 1e-8
RTOL = 1e-9


def _rel(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return float(np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-300))


def _with_ones(X, add_bias):
    return np.column_stack([X, np.ones(len(X))]) if add_bias else X


def _target(family, X, rng):
    """A well-conditioned response of `family` for the rows X (each group gets its own coefficients)."""
    p = X.shape[1]
    beta = rng.uniform(-0.4, 0.4, p)
    eta = X @ beta
    if family == "gaussian":
        return eta + 0.5 + 0.1 * rng.standard_normal(len(X))
    if family == "poisson":
        return rng.poisson(np.exp(np.clip(eta + 0.7, -2.0, 2.0))).astype(np.float64)
    if family == "binomial":
        return (rng.uniform(size=len(X)) < 1.0 / (1.0 + np.exp(-eta))).astype(np.float64)
    return rng.gamma(shape=2.0, scale=np.exp(np.clip(0.3 * eta, -1.0, 1.0)) / 2.0)


def _data(family, sizes, p, seed):
    """X, y and the group key of every row (keys 100, 101, ... in that order, rows shuffled across groups)."""
    rng = np.random.default_rng(seed)
    Xs, ys, ks = [], [], []
    for g, m in enumerate(sizes):
        X = 0.5 * rng.standard_normal((m, p))
        if family == "gamma":          # the inverse link needs eta = X beta > 0, with or without a bias
            X += 1.0
        Xs.append(X)
        ys.append(_target(family, X, rng))
        ks.append(np.full(m, 100 + g))
    X, y, k = np.vstack(Xs), np.concatenate(ys), np.concatenate(ks)
    perm = rng.permutation(len(y))
    # keep the first row of each group first so the first-seen order is the key order
    first = np.array([np.flatnonzero(k[perm] == 100 + g)[0] for g in range(len(sizes))])
    perm = np.concatenate([perm[first], np.delete(perm, first)])
    return X[perm], y[perm], k[perm]


def _loop(family, X, y, key, keys, add_bias, max_iter=100):
    from polars_ds_extension_b200.linear_models import GLM, _glm_fit

    m = GLM(add_bias=add_bias, family=family, max_iter=max_iter, tol=TOL)
    return [_glm_fit(m._family, X[key == k], y[key == k].reshape(-1, 1), add_bias, max_iter, TOL) for k in keys]


@pytest.mark.parametrize("add_bias", [True, False])
@pytest.mark.parametrize("family", FAMILIES)
def test_agrees_with_loop_and_oracle(family, add_bias):
    from polars_ds_extension_b200.linear_models import GLM

    X, y, key = _data(family, [400, 37, 1500, 90, 250], 4, seed=FAMILY_IDS[family] + 10 * add_bias)
    res = GLM(add_bias=add_bias, family=family, tol=TOL).fit_by(X, y, key)
    assert list(res["group"]) == [100, 101, 102, 103, 104]
    assert res["coeffs"].shape == (5, 4 + add_bias) and res["coeffs"].dtype == np.float64
    assert res["n_iter"].dtype == np.int64
    for g, (c, it) in enumerate(_loop(family, X, y, key, res["group"], add_bias)):
        sel = key == res["group"][g]
        ref, ref_it = faer_irls(_with_ones(X[sel], add_bias), y[sel], family, TOL, 100)
        assert _rel(res["coeffs"][g], c) < RTOL and _rel(res["coeffs"][g], ref) < RTOL, g
        assert res["n_iter"][g] == it == ref_it, g


@pytest.mark.parametrize("family", ["poisson", "gamma"])
def test_group_sizes_around_the_item_boundary(family):
    from polars_ds_extension_b200.linear_models import GLM

    sizes = [8191, 8192, 8193, 3 * 8192 + 5, 16385, 300]
    X, y, key = _data(family, sizes, 3, seed=3)
    res = GLM(add_bias=True, family=family, tol=TOL).fit_by(X, y, key)
    for g, (c, it) in enumerate(_loop(family, X, y, key, res["group"], True)):
        assert _rel(res["coeffs"][g], c) < RTOL and res["n_iter"][g] == it, g


def test_tiny_groups():
    """1 row (one feature, no bias), exactly q rows, and fewer rows than coefficients.  The last is rank-deficient: the
    split of the coefficients along the null direction is set by rounding in both paths (DESIGN.md §5), so there the
    fitted values are compared, which are unique (the fit interpolates the group's rows)."""
    from polars_ds_extension_b200.linear_models import GLM

    rng = np.random.default_rng(5)
    X1 = rng.standard_normal((7, 1))
    y1 = 1.0 + rng.standard_normal(7)
    k1 = np.array([0, 1, 1, 2, 2, 2, 2])
    res = GLM(add_bias=False, family="gaussian", tol=TOL).fit_by(X1, y1, k1)
    for g, (c, it) in enumerate(_loop("gaussian", X1, y1, k1, res["group"], False)):
        assert _rel(res["coeffs"][g], c) < RTOL and res["n_iter"][g] == it, g
    assert res["coeffs"][0, 0] == pytest.approx(y1[0] / X1[0, 0], rel=1e-12)

    X, y, key = _data("gaussian", [3, 2, 40], 2, seed=6)          # q = 3: exactly q rows, then fewer
    res = GLM(add_bias=True, family="gaussian", tol=TOL).fit_by(X, y, key)
    loop = _loop("gaussian", X, y, key, res["group"], True)
    for g in (0, 2):
        assert _rel(res["coeffs"][g], loop[g][0]) < 1e-8 and res["n_iter"][g] == loop[g][1], g
    sel = key == 101
    eta = _with_ones(X[sel], True) @ res["coeffs"][1]
    assert np.all(np.isfinite(res["coeffs"][1]))
    assert _rel(eta, y[sel]) < 1e-8 and _rel(eta, _with_ones(X[sel], True) @ loop[1][0]) < 1e-8


@pytest.mark.parametrize("family", FAMILIES)
def test_failures_stay_in_their_group(family):
    """A group whose moments go non-finite (y outside the family's domain, or not finite) gets NaN coefficients and FAILED; a group
    with a zero feature next to the bias (rank-deficient) gets 0 for it, as the loop does; a group that runs out of
    iterations gets MAX_ITER.  The other groups are untouched, bit for bit."""
    import torch

    from polars_ds_extension_b200 import device as dev
    from polars_ds_extension_b200._lib import GLM_CONVERGED, GLM_FAILED, GLM_MAX_ITER

    X, y, key = _data(family, [300, 300, 300, 300], 3, seed=7)
    order = np.argsort(key, kind="stable")
    X, y, key = X[order].copy(), y[order].copy(), key[order]
    off = np.array([0, 300, 600, 900, 1200])
    # outside the domain: mu_0 < 0 under the log link, mu_0 > 1 under the logit; an inf or NaN response otherwise
    bad = {"gaussian": np.inf, "poisson": -100.0, "binomial": 2.0, "gamma": np.nan}[family]
    y[300:600] = np.where(np.arange(300) % 7 == 0, bad, y[300:600])
    X[600:900, 1] = 0.0

    def run(X, y, off, max_iter=100):
        Xd = torch.tensor(X.T.copy(), device="cuda")
        b, st, it = dev.grouped_glm(Xd, torch.tensor(y, device="cuda"), torch.tensor(off, device="cuda"),
                                    FAMILY_IDS[family], add_bias=True, tol=TOL, max_iter=max_iter)
        return b.cpu().numpy(), st.cpu().numpy(), it.cpu().numpy()

    b, st, it = run(X, y, off)
    loop = [faer_irls(_with_ones(X[off[g]:off[g + 1]], True), y[off[g]:off[g + 1]], family, TOL, 100)
            for g in (0, 1)]
    # the oracle's triangular solve refuses the exact zero pivot: it fits group 2 without the zero feature
    reduced, red_it = faer_irls(_with_ones(np.delete(X[600:900], 1, axis=1), True), y[600:900], family, TOL, 100)
    loop.append((np.insert(reduced, 1, 0.0), red_it))
    loop.append(faer_irls(_with_ones(X[900:], True), y[900:], family, TOL, 100))
    # non-finite moments: NaN coefficients, which end the group's fit as they end the loop's
    assert st[1] == GLM_FAILED and np.isnan(b[1]).all() and np.isnan(loop[1][0]).all() and it[1] == loop[1][1]
    for g in (0, 3):
        assert st[g] == GLM_CONVERGED and _rel(b[g], loop[g][0]) < RTOL and it[g] == loop[g][1]
    assert st[2] == GLM_CONVERGED and b[2, 1] == 0.0 and _rel(b[2], loop[2][0]) < RTOL and it[2] == loop[2][1]
    from polars_ds_extension_b200.linear_models import _glm_fit

    single, single_it = _glm_fit(FAMILY_IDS[family], X[600:900], y[600:900].reshape(-1, 1), True, 100, TOL)
    assert single[1] == 0.0 and _rel(b[2], single) < RTOL and it[2] == single_it

    b1, st1, it1 = run(X, y, off, max_iter=1)          # one iteration moves every healthy group by more than tol
    for g in (0, 3):
        ref, ref_it = faer_irls(_with_ones(X[off[g]:off[g + 1]], True), y[off[g]:off[g + 1]], family, TOL, 1)
        assert st1[g] == GLM_MAX_ITER and it1[g] == ref_it == 1 and _rel(b1[g], ref) < RTOL
    assert st1[2] == GLM_MAX_ITER and it1[2] == 1

    # the healthy groups alone, bit for bit
    bh, sth, ith = run(np.vstack([X[:300], X[900:]]), np.concatenate([y[:300], y[900:]]), np.array([0, 300, 600]))
    assert np.array_equal(bh, b[[0, 3]]) and np.array_equal(ith, it[[0, 3]]) and np.array_equal(sth, st[[0, 3]])


@pytest.mark.parametrize("family", ["poisson", "binomial"])
def test_independent_of_other_groups_and_repeatable(family):
    from polars_ds_extension_b200.linear_models import GLM

    X, y, key = _data(family, [500, 9000, 120, 20000, 64], 5, seed=11)
    m = GLM(add_bias=True, family=family, tol=TOL)
    res = m.fit_by(X, y, key)
    again = m.fit_by(X, y, key)
    assert np.array_equal(res["coeffs"], again["coeffs"]) and np.array_equal(res["n_iter"], again["n_iter"])
    for g, k in enumerate(res["group"]):                      # each group alone
        sel = key == k
        one = m.fit_by(X[sel], y[sel], key[sel])
        assert np.array_equal(one["coeffs"][0], res["coeffs"][g]) and one["n_iter"][0] == res["n_iter"][g]
    # groups reordered: the rows of group 103 first
    perm = np.concatenate([np.flatnonzero(key == 103), np.flatnonzero(key != 103)])
    swapped = m.fit_by(X[perm], y[perm], key[perm])
    for g, k in enumerate(swapped["group"]):
        assert np.array_equal(swapped["coeffs"][g], res["coeffs"][list(res["group"]).index(k)])


def test_device_entry_with_mask_matches_host_entry():
    import torch

    from polars_ds_extension_b200 import device as dev
    from polars_ds_extension_b200._lib import GLM_EMPTY
    from polars_ds_extension_b200.linear_models import GLM

    X, y, key = _data("poisson", [700, 9000, 50, 300], 3, seed=13)
    order = np.argsort(key, kind="stable")
    X, y, key = X[order], y[order], key[order]
    off = np.array([0, 700, 9700, 9750, 10050])
    mask = (np.random.default_rng(1).uniform(size=len(y)) < 0.8).astype(np.float64)
    mask[9700:9750] = 0.0                                        # group 2 keeps no row
    b, st, it = dev.grouped_glm(torch.tensor(X.T.copy(), device="cuda"), torch.tensor(y, device="cuda"),
                                torch.tensor(off, device="cuda"), FAMILY_IDS["poisson"], add_bias=True, tol=TOL,
                                mask=torch.tensor(mask, device="cuda"))
    b, st, it = b.cpu().numpy(), st.cpu().numpy(), it.cpu().numpy()
    assert st[2] == GLM_EMPTY and np.isnan(b[2]).all() and it[2] == 0
    kept = mask != 0.0
    host = GLM(add_bias=True, family="poisson", tol=TOL).fit_by(X[kept], y[kept], key[kept])
    assert list(host["group"]) == [100, 101, 103]
    for g, h in zip((0, 1, 3), range(3)):
        assert _rel(b[g], host["coeffs"][h]) < RTOL and it[g] == host["n_iter"][h]


def test_fit_df_by_with_nulls():
    import pyarrow as pa

    import polars_ds_extension_b200 as pds
    from polars_ds_extension_b200.linear_models import GLM

    X, y, key = _data("gamma", [400, 600, 250], 2, seed=17)
    x0 = X[:, 0].tolist()
    x0[5] = None
    yl = y.tolist()
    yl[9] = None
    df = pds.Frame({"a": pa.array(x0, pa.float64()), "b": pa.array(X[:, 1]), "y": pa.array(yl, pa.float64()),
                    "k": pa.array(key)})
    m = GLM(add_bias=True, family="gamma", tol=TOL)
    res = m.fit_df_by(df, ["a", "b"], "y", by="k")
    assert list(res["k"]) == [100, 101, 102] and not m.is_fit()
    keep = np.ones(len(y), dtype=bool)
    keep[[5, 9]] = False
    for g, k in enumerate(res["k"]):
        sel = (key == k) & keep
        single = GLM(add_bias=True, family="gamma", tol=TOL).fit(X[sel], y[sel])
        assert _rel(res["coeffs"][g], np.append(single.coeffs(), single.bias())) < RTOL


def test_million_groups():
    """1e6 groups x 100 rows: the call completes and a sample of groups equals the oracle."""
    import torch

    from polars_ds_extension_b200 import device as dev

    ng, m, p = 1_000_000, 100, 3
    g = torch.Generator(device="cuda").manual_seed(0)
    X = 0.5 * torch.randn((p, ng * m), dtype=torch.float64, device="cuda", generator=g)
    beta = torch.tensor([0.3, -0.2, 0.1], dtype=torch.float64, device="cuda")
    lam = torch.exp(torch.clamp(beta @ X + 0.5, -2.0, 2.0))
    y = torch.poisson(lam, generator=g)
    off = torch.arange(0, ng * m + 1, m, dtype=torch.int64, device="cuda")
    b, st, it = dev.grouped_glm(X, y, off, FAMILY_IDS["poisson"], add_bias=True, tol=TOL)
    torch.cuda.synchronize()
    st = st.cpu().numpy()
    assert (st == 0).all()
    Xh, yh, bh, ith = X.cpu().numpy(), y.cpu().numpy(), b.cpu().numpy(), it.cpu().numpy()
    for gi in np.random.default_rng(0).choice(ng, 200, replace=False):
        rows = slice(gi * m, (gi + 1) * m)
        ref, ref_it = faer_irls(_with_ones(Xh[:, rows].T, True), yh[rows], "poisson", TOL, 100)
        assert _rel(bh[gi], ref) < RTOL and ith[gi] == ref_it, gi
