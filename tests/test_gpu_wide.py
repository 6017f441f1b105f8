"""Wide designs: lin_reg and its family from 65 up to 258 features (the moments hold at most 260 columns, [X | Y | 1]),
against float64 references.

Above 64 features every stage of a fit takes a route that narrower fits never reach, and each route changes again at
its own width:
  * moments: the DMMA and wgmma kernels decline and the tile kernel (gram_simt_kernel) takes every call.  Its register
    blocks per thread are chosen by q1 = p + t + 1 (1 up to 88, 2 for 89-124, 4 for 125-176, 9 for 177-260), and its tile
    rows shrink (f32: 64 from q1 = 125; f64: 32 from 125, 16 from 253).  Several targets take it below 64 features too
    (p + t + 1 > 64 with p <= 64);
  * solve: A and B live in shared memory up to q = 112 (one target), in the global workspace from 113;
  * predict on a resident frame: one ring slot and one consumer warpgroup for p + t > 200;
  * report: HC2 / HC3 read G^-1 from shared memory while q^2 elements fit (q <= 170 in f64, 241 in f32), from global
    memory above;
  * rolling / recursive: the generic pass C, up to 129 coefficients.
Every boundary has a case on each side.  The columns are x_j = mu_j + sigma_j z with distinct means and scales, so a
swapped, dropped or transposed entry shows, and the row counts are not multiples of any tile.
"""
import math

import numpy as np
import pyarrow as pa
import pytest

import polars_ds_extension_b200 as pds
import polars_ds_extension_b200.config as cfg
from oracle import lin_reg_oracle as orc
from oracle.lin_reg_oracle import window_ols
from polars_ds_extension_b200 import Frame
from polars_ds_extension_b200._lib import (METHOD_CD, METHOD_INV, METHOD_LSTSQ, METHOD_NNLS, METHOD_RCOND,
                                           SOLVER_CHOLESKEY, SOLVER_QR, SOLVER_SVD, PdsbError)
from tests.backends import OracleBackend, PluginBackend
from tests.parity_rule import accept_f32, accept_f64

pytestmark = pytest.mark.gpu

GPU = PluginBackend()
ORC = OracleBackend()
U32 = 2.0 ** -24           # unit roundoff of float32
PDSB_GATED = 1


def _col_stats(rng, ncols, span):
    """Distinct means in [-span, span] and distinct scales in [0.5, 4], in shuffled order."""
    mu = rng.permutation(np.linspace(-span, span, ncols))
    sig = rng.permutation(np.geomspace(0.5, 4.0, ncols))
    return mu, sig


# ---------------------------------------------------------------------------------------------------------------------
# 1. moments at the device layer
# ---------------------------------------------------------------------------------------------------------------------
def _device_columns(torch, n, ncols, dtype, seed, span=3.0):
    """(ncols, ld) device matrix with column j = mu_j + sigma_j z, rounded to `dtype`; rows past n are zero."""
    rng = np.random.default_rng(seed)
    mu, sig = _col_stats(rng, ncols, span)
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    ld = (n + 31) // 32 * 32
    z = torch.randn((ncols, n), generator=g, device="cuda", dtype=torch.float64)
    Z = torch.zeros((ncols, ld), dtype=dtype, device="cuda")
    Z[:, :n] = (z * torch.from_numpy(sig).cuda()[:, None] + torch.from_numpy(mu).cuda()[:, None]).to(dtype)
    return Z, ld


def _moments_ref(Zh, W):
    """numpy float64 [X | Y | 1]^T diag(w) [X | Y | 1] of the host rows Zh (q1, n; the last row is the ones or the mask
    column), and the same with absolute values (the scale of the float32 rounding bound)."""
    ref = (Zh * W) @ Zh.T
    A = (np.abs(Zh) * np.abs(W)) @ np.abs(Zh).T
    return ref, A


def _assert_moments(M, ref, A, f32, what):
    d = np.diag(ref)
    scale = np.sqrt(np.outer(d, d))
    err = np.abs(M - ref)
    if f32:
        # the tile kernel sums at most 128 rows of float32 products per tile in a float32 FMA chain (one more rounding
        # with a weight), then adds the tile in float64
        bound = 130 * U32 * A + 1e-12 * scale
    else:
        bound = 1e-12 * scale
    assert np.isfinite(M).all(), what
    bad = np.argwhere(~(err <= bound))
    assert bad.size == 0, (f"{what}: {len(bad)} entries off, first {bad[:4].tolist()}: "
                           f"worst err/bound {float(np.max(err / bound)):.3g}")


MOMENT_SHAPES = [(86, 1), (87, 1), (122, 1), (123, 1), (174, 1), (175, 1), (250, 1), (251, 1), (258, 1),
                 (62, 4), (60, 6), (200, 5)]


@pytest.mark.parametrize("variant", ["plain", "weighted", "masked"])
@pytest.mark.parametrize("dtype", ["f64", "f32"])
@pytest.mark.parametrize("n,p,t", [(200_003, p, t) for p, t in MOMENT_SHAPES] + [(15, 200, 1)])
def test_wide_moments_vs_numpy(n, p, t, dtype, variant):
    """The tile kernel at every width boundary (MAXT 86/87, 122/123, 174/175; f64 tile rows 250/251), at the widest
    shape, with several targets below 64 features, and on fewer rows than one tile; bit-reproducible and symmetric."""
    import torch

    from polars_ds_extension_b200 import device as dev
    from polars_ds_extension_b200._lib import lib

    f32 = dtype == "f32"
    td = torch.float32 if f32 else torch.float64
    Z, ld = _device_columns(torch, n, p + t, td, seed=1000 + 10 * p + t)
    w = mask = None
    if variant == "weighted":
        w = (torch.rand(ld, device="cuda", dtype=torch.float64) * 1.5 + 0.5).to(td)
    elif variant == "masked":
        mask = (torch.rand(ld, device="cuda") > 0.25).to(td)
        Z *= mask[None, :]                         # masked rows are zero in X and Y (packer contract)
    X, Y = Z[:p], Z[p:]
    Zh = np.concatenate([Z[:, :n].double().cpu().numpy(),
                         (mask[:n].double().cpu().numpy() if mask is not None else np.ones(n))[None, :]])
    W = np.ones(n) if w is None else w[:n].double().cpu().numpy()
    # float32 below 65 features: skip the wgmma kernel, which takes up to 4 targets, so the tile kernel runs here too
    L = lib()
    L.pdsb_set_moments_path(1 if f32 and p <= 64 else 0)
    try:
        M1 = dev.moments(X, Y, n=n, w=w, mask=mask).cpu().numpy()
        path = L.pdsb_last_moments_path()
        M2 = dev.moments(X, Y, n=n, w=w, mask=mask).cpu().numpy()
    finally:
        L.pdsb_set_moments_path(0)
    if f32:
        assert path == 0, f"moments path {path}: the register or wgmma kernel took a wide call"
    ref, A = _moments_ref(Zh, W)
    _assert_moments(M1, ref, A, f32, f"{dtype} {variant} n={n} p={p} t={t}")
    assert np.array_equal(M1, M2)
    assert np.array_equal(M1, M1.T)


@pytest.mark.parametrize("p", [100, 199, 200, 258])
def test_wide_frame_moments_and_predict(p):
    """Resident frame at p + t = 101, 200 (ring of at least two slots), 201 and 259 (one slot, one warpgroup): moments
    against numpy, predict on the frame == predict on the column-major matrix bit for bit, and both == X beta within
    float32 rounding of the row's dot product."""
    import torch

    from polars_ds_extension_b200 import device as dev
    from polars_ds_extension_b200._lib import lib

    n, t = 200_003, 1
    Z, ld = _device_columns(torch, n, p + t, torch.float32, seed=2000 + p)
    bt = torch.from_numpy(((np.arange(p) % 7) - 3) / 4.0).cuda()
    noise = torch.randn(n, device="cuda", dtype=torch.float64, generator=torch.Generator(device="cuda").manual_seed(p))
    Z[p, :n] = (bt @ Z[:p, :n].double() + 0.5 + noise).float()       # a target that depends on every feature
    X, Y = Z[:p], Z[p:]
    frame = dev.to_frame(Z, n=n)
    Zh = np.concatenate([Z[:, :n].double().cpu().numpy(), np.ones((1, n))])
    Mf = dev.moments_frame(frame, n, p + t, 0, p, p, t).cpu().numpy()
    assert lib().pdsb_last_moments_path() == 0
    ref, A = _moments_ref(Zh, np.ones(n))
    _assert_moments(Mf, ref, A, True, f"frame p={p}")
    beta, status = dev.solve(torch.from_numpy(Mf).cuda(), p, t, add_bias=True)
    pc, rc = dev.predict(X, Y, beta, status, add_bias=True, n=n)
    pf = torch.empty((t, ld), dtype=torch.float32, device="cuda")
    rf = torch.empty((t, ld), dtype=torch.float32, device="cuda")
    dev.predict_frame(frame, n, p + t, 0, p, p, t, beta, status, True, pf, rf)
    assert int(status[0]) == 0
    assert torch.equal(pf[:, :n], pc[:, :n]) and torch.equal(rf[:, :n], rc[:, :n])
    b = beta.cpu().numpy()[0]
    xb = b[:p] @ Zh[:p] + b[p]
    # beta rounded to float32 (one rounding per term) and a float32 FMA chain over p + 1 terms
    tol = (p + 3) * U32 * (np.abs(b[:p]) @ np.abs(Zh[:p]) + abs(b[p]))
    pred = pc[0, :n].double().cpu().numpy()
    resid = rc[0, :n].double().cpu().numpy()
    y = Zh[p]
    assert np.all(np.abs(pred - xb) <= tol), float(np.max(np.abs(pred - xb) / tol))
    assert np.all(np.abs(resid - (y - xb)) <= tol + 2 * U32 * (np.abs(y) + np.abs(xb)))


# ---------------------------------------------------------------------------------------------------------------------
# 2. the solve at the device layer, on numpy-built float64 moments
# ---------------------------------------------------------------------------------------------------------------------
def _design(seed, n, p, span=3.0, noise=0.1):
    """X (n, p) with distinct column means / scales, y = X beta + 0.5 + noise."""
    rng = np.random.default_rng(seed)
    mu, sig = _col_stats(rng, p, span)
    X = mu + sig * rng.standard_normal((n, p))
    beta = ((np.arange(p) % 7) - 3) / 4.0
    y = X @ beta + 0.5 + noise * rng.standard_normal(n)
    return X, y


def _gram_problem(q, seed, n=20_011):
    """q coefficients = q - 1 features and a bias: (X with the ones column last, y, device moments M)."""
    import torch

    X, y = _design(seed, n, q - 1)
    Zh = np.column_stack([X, y, np.ones(n)])
    M = Zh.T @ Zh
    Xb = np.column_stack([X, np.ones(n)])
    return Xb, y, torch.from_numpy(M).cuda()


def _gram_of(M, p):
    idx = list(range(p)) + [p + 1]
    return M.cpu().numpy()[np.ix_(idx, idx)]


@pytest.mark.parametrize("q", [112, 113, 200, 259])
def test_wide_solve_lstsq_and_inverse(q):
    """LSTSQ (pivoted QR, Jacobi SVD, Cholesky; with and without ridge) and the explicit inverse on both sides of the
    shared / global workspace switch (q = 112 / 113) and up to the widest fit, against the oracle on the same data."""
    from polars_ds_extension_b200 import device as dev

    Xb, y, M = _gram_problem(q, seed=3000 + q)
    p = q - 1
    for solver, how in [(SOLVER_QR, "qr"), (SOLVER_SVD, "svd"), (SOLVER_CHOLESKEY, "choleskey")]:
        for l2 in (0.0, 0.5):
            beta, status = dev.solve(M, p, 1, add_bias=True, method=METHOD_LSTSQ, solver=solver, l2_reg=l2)
            assert int(status[0]) == 0
            ref = orc.faer_solve_lr(Xb, y[:, None], l2, True, how)[:, 0]
            accept_f64(beta.cpu().numpy()[0], ref, f"q={q} {how} l2={l2}")
    beta, status, aux = dev.solve(M, p, 1, add_bias=True, method=METHOD_INV, want_aux=True)
    G = _gram_of(M, p)
    inv = aux.cpu().numpy()[: q * q].reshape(q, q)
    accept_f64(inv, np.linalg.inv(G), f"q={q} inverse")
    accept_f64(beta.cpu().numpy()[0], np.linalg.solve(G, Xb.T @ y), f"q={q} inv beta")


@pytest.mark.parametrize("q", [113, 200, 259])
def test_wide_solve_rcond(q):
    """RCOND: the Jacobi eigen-solve, the descending order of the singular values in aux, and the cut.  The threshold
    sits in the widest gap of the lower half of the spectrum, above at least the three smallest eigenvalues, so that
    it drops several directions and rounding cannot move one across it."""
    from polars_ds_extension_b200 import device as dev

    Xb, y, M = _gram_problem(q, seed=3100 + q)
    p = q - 1
    S = np.sort(np.linalg.eigvalsh(_gram_of(M, p)))[::-1]
    lo = q // 2
    i = lo + int(np.argmax(S[lo:q - 3] / S[lo + 1:q - 2]))
    rcond = math.sqrt(S[i] * S[i + 1]) / math.sqrt(S[0])
    assert S[i] / S[i + 1] > 1.01
    beta, status, aux = dev.solve(M, p, 1, add_bias=True, method=METHOD_RCOND, tol=rcond, want_aux=True)
    ref, sv = orc.faer_solve_lr_rcond(Xb, y[:, None], 0.0, True, rcond)
    accept_f64(aux.cpu().numpy()[:q], sv, f"q={q} singular values")
    accept_f64(beta.cpu().numpy()[0], ref[:, 0], f"q={q} rcond beta")


@pytest.mark.parametrize("q", [113, 259])
@pytest.mark.parametrize("kind", ["lasso", "enet", "nnls"])
def test_wide_solve_iterative(q, kind):
    """Coordinate descent (lasso, elastic net) and projected NNLS on a wide Gram for a fixed number of sweeps (tol = 0:
    no early stop, so both sides run the same sweeps) against the oracle's restatements on the same data."""
    from polars_ds_extension_b200 import device as dev

    Xb, y, M = _gram_problem(q, seed=3200 + q)
    p = q - 1
    it = 25
    if kind == "nnls":
        beta, _ = dev.solve(M, p, 1, add_bias=True, method=METHOD_NNLS, tol=0.0, max_iter=it)
        ref = orc.faer_nn_lr(Xb, y[:, None], True, 0.0, it)[:, 0]
    else:
        l1, l2 = (0.01, 0.0) if kind == "lasso" else (0.01, 0.02)
        beta, _ = dev.solve(M, p, 1, add_bias=True, method=METHOD_CD, l1_reg=l1, l2_reg=l2, tol=0.0, max_iter=it)
        ref = orc.faer_coordinate_descent(Xb, y[:, None], l1, l2, True, 0.0, it, False)[:, 0]
    got = beta.cpu().numpy()[0]
    assert np.isfinite(got).all()
    accept_f64(got, ref, f"q={q} {kind}")


def test_wide_solve_rank_deficient():
    """Two equal columns at q = 150: gated, the status says so; ungated, a finite beta that satisfies the normal
    equations (documented deviation 1: a basic solution, not the reference's bit pattern).  The gate's tolerance sits
    well below the same design's ratio with the copied column replaced by a fresh one, so only the rank fires it."""
    import torch

    from polars_ds_extension_b200 import device as dev

    q = 150
    p = q - 1
    Xb, y, M = _gram_problem(q, seed=3300)
    Mh = M.cpu().numpy()
    G_full = _gram_of(M, p)
    ln_ratio = np.linalg.slogdet(G_full)[1] - np.sum(np.log(np.diag(G_full)))
    tol = math.exp(ln_ratio - 10.0)
    beta, status = dev.solve(M, p, 1, add_bias=True, singular_x_tol=tol)
    assert int(status[0]) == 0
    a, b = 17, 120                                            # column b := column a, exactly
    Mh[b, :] = Mh[a, :]
    Mh[:, b] = Mh[:, a]
    Md = torch.from_numpy(Mh).cuda()
    for solver in (SOLVER_QR, SOLVER_SVD, SOLVER_CHOLESKEY):
        _, status = dev.solve(Md, p, 1, add_bias=True, solver=solver, singular_x_tol=tol)
        assert int(status[0]) == PDSB_GATED, solver
    beta, status = dev.solve(Md, p, 1, add_bias=True, solver=SOLVER_QR)
    assert int(status[0]) == 0
    bh = beta.cpu().numpy()[0]
    assert np.isfinite(bh).all()
    G = _gram_of(Md, p)
    rhs = Mh[np.ix_(list(range(p)) + [p + 1], [p])][:, 0]
    resid = np.abs(G @ bh - rhs)
    assert np.all(resid <= 1e-9 * (np.abs(G) @ np.abs(bh) + np.abs(rhs))), float(np.max(resid))


# ---------------------------------------------------------------------------------------------------------------------
# 3. end to end through the plugin ABI
# ---------------------------------------------------------------------------------------------------------------------
def _wide_frame(seed, n, p, f64, span=0.5, noise=0.1, nulls=0.0, weights=False):
    """Frame of x0..x{p-1}, y (and w) in the expression's dtype.  A narrower mean span than the device tests: the f32
    restatement solves in float32, and the acceptance rule needs it to be meaningful."""
    X, y = _design(seed, n, p, span, noise)
    rng = np.random.default_rng(seed + 1)
    dt = np.float64 if f64 else np.float32
    d = {}
    for i in range(p):
        m = (rng.random(n) < nulls) if nulls else None
        d[f"x{i}"] = X[:, i].astype(dt) if m is None else pa.array(X[:, i].astype(dt), mask=m)
    d["y"] = y.astype(dt)
    if weights:
        d["w"] = rng.uniform(0.5, 2.0, n).astype(dt)
    return Frame(d), [f"x{i}" for i in range(p)]


def _three(monkeypatch, f64, df, make):
    """(gpu, oracle in the same precision, f64 oracle on the same inputs) of the expression `make()` builds."""
    monkeypatch.setattr(cfg, "LIN_REG_EXPR_F64", f64)
    e = make()
    g, o = GPU.eval(df, e), ORC.eval(df, e)
    if f64:
        return g, o, o
    monkeypatch.setattr(cfg, "LIN_REG_EXPR_F64", True)
    truth = ORC.eval(df, make())
    monkeypatch.setattr(cfg, "LIN_REG_EXPR_F64", False)
    return g, o, truth


def _accept(f64, g, o, truth, what):
    assert g is not None and o is not None, what
    if f64:
        accept_f64(g, o, what)
    else:
        accept_f32(g, o, truth, what)


def _accept_pred(f64, g, o, truth, what):
    """pred by the parity rule; resid on the predictions' scale (differences of O(1) numbers)"""
    (gp, gv), (op, ov), (tp, tv) = g["pred"], o["pred"], truth["pred"]
    assert np.array_equal(gv, ov) and np.array_equal(gv, tv), what
    v = tv
    _accept(f64, gp[v], op[v], tp[v], f"{what} pred")
    scale = np.abs(tp[v]).max()
    er_g = np.max(np.abs(g["resid"][0][v] - truth["resid"][0][v])) / scale
    er_o = np.max(np.abs(o["resid"][0][v] - truth["resid"][0][v])) / scale
    assert er_g <= (1e-6 if f64 else max(er_o, 2e-6)), (what, er_g, er_o)


# no rank gate: a wide design whose columns share a mean direction has a small det(G) / prod diag(G) and would trip the
# reference's determinant-ratio gate; the gate itself is tested at the device layer above
NO_GATE = dict(singular_x_tol=0.0)


@pytest.mark.parametrize("f64", [True, False])
@pytest.mark.parametrize("p,bias", [(65, True), (65, False), (87, True), (111, True), (112, True), (175, False),
                                    (258, True), (258, False)])
def test_wide_lin_reg_vs_oracle(monkeypatch, f64, p, bias):
    df, xs = _wide_frame(4000 + p, 20_011, p, f64)
    g, o, truth = _three(monkeypatch, f64, df, lambda: pds.lin_reg(*xs, target="y", add_bias=bias, **NO_GATE))
    _accept(f64, g, o, truth, f"p={p} bias={bias} coeffs")
    g, o, truth = _three(monkeypatch, f64, df,
                         lambda: pds.lin_reg(*xs, target="y", add_bias=bias, return_pred=True, **NO_GATE))
    _accept_pred(f64, g, o, truth, f"p={p} bias={bias}")


@pytest.mark.parametrize("f64", [True, False])
def test_wide_lin_reg_nulls_and_weights(monkeypatch, f64):
    """null_policy="skip" with nulls spread over 175 features (masked rows through the tile kernel), and a weighted fit
    at 150 features."""
    df, xs = _wide_frame(4100, 20_011, 175, f64, nulls=0.0002)
    g, o, truth = _three(monkeypatch, f64, df,
                         lambda: pds.lin_reg(*xs, target="y", add_bias=True, null_policy="skip", **NO_GATE))
    _accept(f64, g, o, truth, "skip coeffs")
    g, o, truth = _three(monkeypatch, f64, df, lambda: pds.lin_reg(*xs, target="y", add_bias=True, null_policy="skip",
                                                                   return_pred=True, **NO_GATE))
    assert not g["pred"][1].all()                           # some rows were dropped
    _accept_pred(f64, g, o, truth, "skip")
    df, xs = _wide_frame(4101, 20_011, 150, f64, weights=True)
    g, o, truth = _three(monkeypatch, f64, df,
                         lambda: pds.lin_reg(*xs, target="y", add_bias=True, weights="w", **NO_GATE))
    _accept(f64, g, o, truth, "weighted coeffs")


@pytest.mark.parametrize("f64", [True, False])
def test_wide_rcond_multi_target_and_ar(monkeypatch, f64):
    """lin_reg_w_rcond at 150 features; six targets on 120 features (coefficients and pred / resid); query_ar_coeffs
    with 120 lags, against numpy's least squares on the lagged matrix too."""
    df, xs = _wide_frame(4200, 20_011, 150, f64)
    g, o, truth = _three(monkeypatch, f64, df, lambda: pds.lin_reg_w_rcond(*xs, target="y", add_bias=True, rcond=1e-9))
    for k in ("coeffs", "singular_values"):
        _accept(f64, g[k], o[k], truth[k], f"rcond {k}")

    p, t = 120, 6
    rng = np.random.default_rng(4201)
    X, _ = _design(4202, 20_011, p, span=0.5)
    B = rng.standard_normal((p, t))
    Y = X @ B + 0.1 * rng.standard_normal((20_011, t))
    dt = np.float64 if f64 else np.float32
    dm = Frame({f"x{i}": X[:, i].astype(dt) for i in range(p)} | {f"y{k}": Y[:, k].astype(dt) for k in range(t)})
    xs = [f"x{i}" for i in range(p)]
    ys = [f"y{k}" for k in range(t)]
    g, o, truth = _three(monkeypatch, f64, dm, lambda: pds.lin_reg(*xs, target=ys, add_bias=True, **NO_GATE))
    assert sorted(g) == sorted(o)
    for k in o:
        _accept(f64, g[k], o[k], truth[k], f"multi {k}")
    g, o, truth = _three(monkeypatch, f64, dm,
                         lambda: pds.lin_reg(*xs, target=ys, add_bias=True, return_pred=True, **NO_GATE))
    assert sorted(g) == sorted(o) and len(o) == 2 * t
    for k in range(t):
        pair = [{"pred": v[f"target_{k}_pred"], "resid": v[f"target_{k}_resid"]} for v in (g, o, truth)]
        _accept_pred(f64, *pair, f"multi target {k}")

    # a weakly correlated AR(1): 120 strongly correlated lags would make det(G) / prod diag(G) trip the default rank gate
    lag, n = 120, 20_011
    e = rng.standard_normal(n + 500)
    x = np.zeros(n + 500)
    for i in range(1, n + 500):
        x[i] = 0.2 * x[i - 1] + e[i]
    x = x[500:]
    da = Frame({"x": x.astype(dt)})
    g, o, truth = _three(monkeypatch, f64, da, lambda: pds.query_ar_coeffs("x", lag=lag))
    _accept(f64, g, o, truth, "ar")
    xa = x.astype(dt).astype(np.float64)
    A = np.column_stack([xa[lag - i:n - i] for i in range(1, lag + 1)] + [np.ones(n - lag)])
    lst = np.linalg.lstsq(A, xa[lag:], rcond=None)[0]
    accept_f64(truth, lst, "ar oracle vs lstsq")
    if f64:
        accept_f64(g, lst, "ar vs lstsq")
    else:
        accept_f32(g, o, lst, "ar vs lstsq")


@pytest.mark.parametrize("f64", [True, False])
def test_wide_lin_reg_above_the_moments_bound(monkeypatch, f64):
    """259 features and one target need 261 moment columns: a clean error naming the bound, and no result left
    behind."""
    from polars_ds_extension_b200._lib import lib

    monkeypatch.setattr(cfg, "LIN_REG_EXPR_F64", f64)
    df, xs = _wide_frame(4300, 2_000, 259, f64)
    live = lib().pdsb_plugin_live_results()
    for rp in (False, True):
        with pytest.raises(PdsbError, match=r"p\+t\+1=261 out of range \(max 260\)"):
            df.evaluate(pds.lin_reg(*xs, target="y", add_bias=True, return_pred=rp))
    assert lib().pdsb_plugin_live_results() == live


def test_fast_group_paths_stop_at_64_features(monkeypatch):
    """group_by(...).agg(..., fast=True) and over(key, fast=True) take at most 64 features and say so; fast=False, one
    call per group, fits 65 features and matches the oracle."""
    monkeypatch.setattr(cfg, "LIN_REG_EXPR_F64", True)
    p = 65
    df, xs = _wide_frame(4400, 6_000, p, True)
    gid = np.repeat(np.arange(3), 2_000)
    df = df.with_columns(g=gid)
    e = pds.lin_reg(*xs, target="y", add_bias=True, **NO_GATE)
    with pytest.raises(PdsbError, match=r"p=65 not supported \(1\.\.64\)"):
        df.group_by("g").agg(e, fast=True)
    ep = pds.lin_reg(*xs, target="y", add_bias=True, return_pred=True, **NO_GATE)
    with pytest.raises(PdsbError, match=r"p=65 not supported \(1\.\.64\)"):
        df.select(ep.over("g", fast=True))
    slow = GPU.group_eval(df, "g", e, fast=False)
    ref = ORC.group_eval(df, "g", e)
    assert len(slow) == len(ref) == 3
    for k in range(3):
        accept_f64(slow[k], ref[k], f"group {k}")


# ---------------------------------------------------------------------------------------------------------------------
# 4. lin_reg_report / wls report at wide q
# ---------------------------------------------------------------------------------------------------------------------
def _high_leverage(df, xs, p, target_h=0.9):
    """Move row 0 along a fixed direction until its leverage in [X | 1] is target_h (float64 frames)."""
    X = np.column_stack([df[c].to_numpy() for c in xs])
    n = X.shape[0]
    u = np.random.default_rng(7).standard_normal(p)
    rest = np.column_stack([X[1:], np.ones(n - 1)])
    Gi = np.linalg.inv(rest.T @ rest)
    # x(s) = [s u, 1]: a(s) = x^T G_rest^-1 x = s^2 uAu + 2 s uAb + c, and h = a / (1 + a)
    uAu, uAb, c = u @ Gi[:p, :p] @ u, u @ Gi[:p, p], Gi[p, p]
    a = target_h / (1.0 - target_h)
    s = (-uAb + math.sqrt(uAb ** 2 - uAu * (c - a))) / uAu
    X[0] = s * u
    cols = {c: X[:, i] for i, c in enumerate(xs)}
    return Frame({**{k: v for k, v in df.columns.items() if k not in cols}, **cols})


def _assert_report(f64, g, o, truth, what):
    assert g["features"] == o["features"], what
    for k in o:
        if k == "features":
            continue
        if k == "p>|t|":
            # p-values span many decades: element-wise relative comparison on ln p
            lg, lo, lt = (np.log(np.maximum(np.asarray(v[k], np.float64), 1e-300)) for v in (g, o, truth))
            eg, eo = np.max(np.abs(lg - lt) / np.abs(lt)), np.max(np.abs(lo - lt) / np.abs(lt))
            assert eg <= (1e-6 if f64 else max(eo, 2e-6)), (what, k, eg, eo)
        else:
            _accept(f64, g[k], o[k], truth[k], f"{what}:{k}")


REPORT_CASES = [(True, q) for q in (113, 170, 171, 200, 259)] + [(False, q) for q in (241, 242, 259)]


@pytest.mark.parametrize("f64,q", REPORT_CASES)
@pytest.mark.parametrize("se", ["se", "hc0", "hc1", "hc2", "hc3"])
def test_wide_report_vs_oracle(monkeypatch, f64, q, se):
    """Every field of the report against the oracle on both sides of the shared-memory bound of G^-1 in the HC weights
    kernel (q^2 elements: 170 / 171 in f64, 241 / 242 in f32) and at the widest fit; the f64 frames carry one row of
    leverage 0.9 so that 1 - h is exercised."""
    p = q - 1
    df, xs = _wide_frame(5000 + q, 20_011, p, f64, noise=1.0)
    if f64:
        df = _high_leverage(df, xs, p)
    g, o, truth = _three(monkeypatch, f64, df, lambda: pds.lin_reg_report(*xs, target="y", add_bias=True, std_err=se))
    _assert_report(f64, g, o, truth, f"{'f64' if f64 else 'f32'} q={q} {se}")


@pytest.mark.parametrize("f64", [True, False])
def test_wide_weighted_report_vs_oracle(monkeypatch, f64):
    df, xs = _wide_frame(5300, 20_011, 199, f64, noise=1.0, weights=True)
    g, o, truth = _three(monkeypatch, f64, df, lambda: pds.lin_reg_report(*xs, target="y", weights="w", add_bias=True))
    _assert_report(f64, g, o, truth, "wls q=200")


# ---------------------------------------------------------------------------------------------------------------------
# 5. rolling / recursive at wide D (the generic pass C)
# ---------------------------------------------------------------------------------------------------------------------
def _online(X, y, window, min_rows, bias):
    import torch

    from polars_ds_extension_b200 import device as dev
    from polars_ds_extension_b200._lib import lib

    Xt = torch.from_numpy(np.ascontiguousarray(X.T)).cuda()
    yt = torch.from_numpy(y).cuda()
    co, pr, va = dev.online_lin_reg(Xt, yt, window=window, min_rows=min_rows, add_bias=bias)
    return co.cpu().numpy(), pr.cpu().numpy(), va.cpu().numpy().astype(bool), int(lib().pdsb_last_online_path())


@pytest.mark.parametrize("D,bias,window", [(64, True, 300), (100, False, 301), (129, True, 299), (100, True, 0)])
def test_wide_rolling_and_recursive_vs_definition(D, bias, window):
    """Rolling windows of about 300 rows at 64, 100 and 129 coefficients (the generic kernel's widest), and a recursive
    fit at 100: every checked row == OLS on its window (f64), pred == x . beta."""
    n = 2_500
    p = D - int(bias)
    X, y = _design(6000 + D + window, n, p, span=1.0)
    start = window if window else 2 * D
    co, pr, va, route = _online(X, y, window, start, bias)
    assert route == 3
    Z = np.column_stack([X] + ([np.ones(n)] if bias else []))
    assert not va[: start - 1].any() and va[start - 1:].all()
    rng = np.random.default_rng(D)
    rows = sorted(set(rng.integers(start - 1, n, 40).tolist()) | {start - 1, start, n - 1, 1023, 1024, 2047, 2048})
    for j in rows:
        lo = j - window + 1 if window else 0
        truth = window_ols(Z, y, lo, j + 1)
        accept_f64(co[j], truth, f"D={D} window={window} row {j}")
        assert abs(pr[j] - Z[j] @ co[j]) <= 1e-12 * (np.abs(Z[j]) @ np.abs(co[j]))


@pytest.mark.parametrize("window", [300, 0])
def test_wide_rolling_above_the_generic_bound(window):
    """130 coefficients do not fit the generic kernel's shared memory: a clean error that names the bound, 129."""
    n, p = 1_000, 129
    X, y = _design(6100, n, p, span=1.0)
    with pytest.raises(PdsbError, match=r"130 coefficients exceed the device limit of 129"):
        _online(X, y, window, window or 400, True)
