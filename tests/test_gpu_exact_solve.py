"""The dense solves against exact rational solutions: K3 (solve_kernel, one CTA per problem) on exact moments uploaded
from numpy, and K5's group_solve (one thread per group: K5, the multi-target fit, AR and the grouped report) through
pdsb_dev_grouped_*, on integer designs whose moments every route forms exactly (tests/test_gpu_exact_moments.py).

Every β is held to tests/exact_oracle.accept: rel(got, exact) <= max(10 err_lapack, q u64 kappa_2(G), 8 u64).  The f32 grouped
entries see the same exact f64 moments on integer data (f32 products of integers below 2^12, f32 chains below 2^24:
documented deviation 5), so they are held to the same rule.  Which side of group_solve's shared / global workspace
switch a case is on is restated by exact_oracle.k5_solve_in_shared; the sweeps below cover both sides.
"""
import math

import numpy as np
import pytest

from tests.exact_oracle import (K5_FULL_Q, PMAX, U64, Design, accept, conditioning_design, exact_det, exact_gate_ratio,
                                exact_moments, exact_report, exact_solve, gram, int_design, k3_cases, k3_moments,
                                k5_case, k5_cases, k5_solve_in_shared, k5_switch_q, kappa, sizes_full, sizes_sweep)
from tests.parity_rule import rel

pytestmark = pytest.mark.gpu

QR, SVD, CHOL = 0, 1, 2
LSTSQ, CD, NNLS, INV = 0, 1, 2, 4
METHOD_NAME = {QR: "qr", SVD: "svd", CHOL: "chol"}
GATED = 1
RIDGE = 3          # an integer ridge keeps G + l2 I exact


def _torch():
    import torch
    return torch


def _dev():
    from polars_ds_extension_b200 import device as dev
    return dev


# ---------------------------------------------------------------------------------------------------------------------
# K3 on exact moments
# ---------------------------------------------------------------------------------------------------------------------
def _k3(M, p, t, bias, **kw):
    torch = _torch()
    beta, status, *aux = _dev().solve(torch.from_numpy(M.astype(np.float64)).cuda(), p, t, add_bias=bias, **kw)
    return beta.cpu().numpy(), int(status[0]), (aux[0].cpu().numpy() if aux else None)


@pytest.mark.parametrize("q,bias", k3_cases())
def test_k3_lstsq_exact(q, bias):
    """QR, Cholesky and svd, with and without ridge, at every q from 1 to 65."""
    p = q - int(bias)
    M = k3_moments(p, 1)
    for ridge in (0, RIDGE):
        G, b = gram(M, p, 1, bias)
        G[np.arange(p), np.arange(p)] += ridge
        ex = exact_solve(G, b)
        for solver in (QR, CHOL, SVD):
            beta, status, _ = _k3(M, p, 1, bias, solver=solver, l2_reg=float(ridge))
            assert status == 0
            accept(beta[0], ex, G, b, METHOD_NAME[solver], f"K3 q={q} bias={bias} ridge={ridge} {METHOD_NAME[solver]}")


@pytest.mark.parametrize("q", list(range(2, PMAX + 1, 3)) + [PMAX])
def test_k3_multi_target_exact(q):
    """t = 2..4 targets: one factorisation, each target's β against its exact solution."""
    p = q - 1
    for t in (2, 3, 4):
        M = k3_moments(p, t)
        beta, status, _ = _k3(M, p, t, True)
        assert status == 0
        for c in range(t):
            G, b = gram(M, p, t, True, target=c)
            accept(beta[c], exact_solve(G, b), G, b, "qr", f"K3 q={q} t={t} target {c}")


@pytest.mark.parametrize("q", [1, 2, 3, 5, 8, 13, 21, 22, 33, 40, 64, 65])
def test_k3_inverse_exact(q):
    """METHOD_INV: β and the aux G^-1 (row-major) against the exact inverse, column by column under the rule."""
    p = q - 1 if q > 1 else 1
    bias = q > 1
    M = k3_moments(p, 1)
    G, b = gram(M, p, 1, bias)
    beta, status, aux = _k3(M, p, 1, bias, method=INV, want_aux=True)
    assert status == 0
    accept(beta[0], exact_solve(G, b), G, b, "qr", f"K3 INV q={q} beta")
    Gi = aux[:q * q].reshape(q, q)
    E = exact_solve(G, np.eye(q, dtype=np.int64))
    for c in range(q):
        e = np.zeros(q, np.int64)
        e[c] = 1
        accept(Gi[:, c], E[:, c], G, e, "qr", f"K3 INV q={q} column {c}")


# ---------------------------------------------------------------------------------------------------------------------
# K5 group_solve through the grouped entries
# ---------------------------------------------------------------------------------------------------------------------
def _upload_groups(X, Y, keep, dtype, multi=False):
    """X (p, ld) and y (ld,) (or Z = [Y | X] for the multi-target entry) on the device, NaN on the dropped rows."""
    torch = _torch()
    n = X.shape[0]
    ld = max((n + 31) // 32 * 32, 32)
    cols = np.concatenate([Y.T, X.T]) if multi else np.concatenate([X.T, Y[:, :1].T])
    Zh = np.zeros((cols.shape[0], ld))
    Zh[:, :n] = cols
    Zh[:, :n][:, ~keep] = np.nan
    Z = torch.from_numpy(Zh).to(dtype).cuda()
    return Z


def _group_truth(X, Y, keep, span, p, bias, t=1, c=0):
    s, e = span
    M = exact_moments(Design(X[s:e], Y[s:e], None, keep[s:e]))
    G, b = gram(M, p, t, bias, target=c)
    return M, G, b, int(keep[s:e].sum())


def _check_groups(beta, status, X, Y, keep, offsets, spans, p, bias, what, t=1, method="qr"):
    q = p + int(bias)
    for g, span in enumerate(spans):
        nk = int(keep[span[0]:span[1]].sum())
        if nk < q:
            assert status[g] == GATED, f"{what}: group {g} ({nk} kept rows < q = {q}) not gated"
            assert np.isnan(beta[g]).all(), f"{what}: gated group {g} has a β"
            continue
        assert status[g] == 0, f"{what}: group {g} ({nk} rows) status {status[g]}"
        for c in range(t):
            _, G, b, _ = _group_truth(X, Y, keep, span, p, bias, t, c)
            ex = exact_solve(G, b)
            got = beta[g][c] if t > 1 else beta[g]
            accept(got, ex, G, b, method, f"{what}: group {g} ({nk} rows) target {c}")


def _grouped(X, Y, keep, offsets, p, bias, dtype, **kw):
    torch = _torch()
    Z = _upload_groups(X, Y, keep, dtype)
    offs = torch.from_numpy(offsets).cuda()
    beta, status = _dev().grouped_lin_reg(Z[:p], Z[p], offs, add_bias=bias, **kw)
    return beta.cpu().numpy(), status.cpu().numpy()


@pytest.mark.parametrize("q,bias", k5_cases())
def test_k5_lin_reg_exact(q, bias):
    """Every q from 1 to 65 (with the bias on even q, without on odd q, both at the boundaries), f64 and f32, on both
    sides of the shared / global workspace switch; the full size list at the boundaries."""
    p = q - int(bias)
    sizes = sizes_full(q) if q in K5_FULL_Q else sizes_sweep(q)
    X, Y, keep, offsets, spans = k5_case(7000 + q, p, bias, sizes)
    side = "shared" if k5_solve_in_shared(p, q) else "global"
    torch = _torch()
    for dtype in (torch.float64, torch.float32):
        beta, status = _grouped(X, Y, keep, offsets, p, bias, dtype)
        _check_groups(beta, status, X, Y, keep, offsets, spans, p, bias, f"K5 {dtype} q={q} bias={bias} ({side})")
        beta2, status2 = _grouped(X, Y, keep, offsets, p, bias, dtype)
        assert np.array_equal(status, status2) and np.array_equal(beta, beta2, equal_nan=True)


@pytest.mark.parametrize("q", sorted({2, 3, 8, k5_switch_q(True, INV), k5_switch_q(True, INV) + 1, 21, 22, 40, 65}))
def test_k5_report_beta_exact(q):
    """The grouped report's METHOD_INV solve (nrhs = q + 1: its workspace switch comes earlier), β under the rule; the
    classic se, t, p and interval of the largest and smallest solvable groups against mpmath."""
    torch = _torch()
    p = q - 1
    X, Y, keep, offsets, spans = k5_case(8000 + q, p, True, sizes_sweep(q))
    for dtype in (torch.float64, torch.float32):
        Z = _upload_groups(X, Y, keep, dtype)
        out, status = _dev().grouped_report(Z[:p], Z[p], torch.from_numpy(offsets).cuda(), add_bias=True)
        out, status = out.cpu().numpy(), status.cpu().numpy()
        side = "shared" if k5_solve_in_shared(p, q, INV) else "global"
        _check_groups(out[:, 0, :], status, X, Y, keep, offsets, spans, p, True, f"K17 {dtype} q={q} ({side})")
        if dtype == torch.float64 and q <= 40:
            for g in (len(spans) - 3, spans.index(max(spans, key=lambda s: s[1] - s[0]))):
                if keep[spans[g][0]:spans[g][1]].sum() <= q:
                    continue
                M, G, b, _ = _group_truth(X, Y, keep, spans[g], p, True)
                _check_report(out[g, :6], exact_report(M, p, True), G, f"K17 q={q} group {g}")


def _check_report(got, ex, G, what):
    """β to lim = max(q u64 kappa_2, 64 u64), se and t (through diag G^-1 and a square root) to 10 lim, ln p to 1e-9
    plus that bound times t^2, the interval to max(10 lim, 1e-10)."""
    q = G.shape[0]
    lim = max(q * U64 * kappa(G), 64 * U64)
    for r, name in ((0, "beta"), (1, "se"), (2, "t")):
        assert rel(got[r], ex[r]) <= max(lim, 10 * lim if r else lim), f"{what} {name}: {rel(got[r], ex[r]):.3e} > {lim:.3e}"
    lp_g, lp_e = np.log(np.maximum(got[3], 1e-300)), np.log(np.maximum(ex[3], 1e-300))
    tol = 1e-9 * np.maximum(1.0, np.abs(lp_e)) + 4.0 * ex[2] ** 2 * lim
    keep = ex[3] > 1e-280
    assert np.all(np.abs(lp_g - lp_e)[keep] <= tol[keep]), f"{what} ln p: {np.abs(lp_g - lp_e)} vs {tol}"
    assert rel(got[4:6], ex[4:6]) <= max(10 * lim, 1e-10), f"{what} interval: {rel(got[4:6], ex[4:6]):.3e}"


@pytest.mark.parametrize("q", [2, 5, 20, 21, 22, 23, 40, 63])
def test_k5_multi_target_exact(q):
    """t = 3 targets through the multi-target entry (up to 65 features and targets together): the fz / fy column
    mapping of every target under the rule, on both sides of its workspace switch (20 / 21 coefficients)."""
    torch = _torch()
    p, t = q - 1, 3
    X, Y, keep, offsets, spans = k5_case(9000 + q, p, True, sizes_sweep(q), t=t)
    Z = _upload_groups(X, Y, keep, torch.float64, multi=True)
    beta, status = _dev().grouped_lin_reg_multi(Z, torch.from_numpy(offsets).cuda(), t, add_bias=True)
    side = "shared" if k5_solve_in_shared(p, q, t=t) else "global"
    _check_groups(beta.cpu().numpy(), status.cpu().numpy(), X, Y, keep, offsets, spans, p, True,
                  f"K5 multi q={q} ({side})", t=t)


@pytest.mark.parametrize("lag", [1, 2, 5, 16, 20, 21, 33, 64])
def test_k5_ar_exact(lag):
    """The AR entry's lagged design, formed on the device (f64, and f32 through the AR register kernel), against the
    exact fit of the same lagged design."""
    torch = _torch()
    rng = np.random.default_rng(lag)
    sizes = [lag, lag + 1, 2 * lag + 3, 129, 8193 + lag, 3 * 8192 + 1]
    xs = [rng.integers(-8, 9, size=m).astype(np.int64) for m in sizes]
    offsets = np.array([0] + list(np.cumsum(sizes)), np.int64)
    for dtype in (torch.float64, torch.float32):
        xh = torch.from_numpy(np.concatenate(xs)).to(dtype).cuda()
        beta, status = _dev().grouped_ar_coeffs(xh, torch.from_numpy(offsets).cuda(), lag, add_bias=True,
                                                singular_x_tol=0.0)
        _check_ar(beta.cpu().numpy(), status.cpu().numpy(), xs, lag, f"AR {dtype} lag={lag}")


def _check_ar(beta, status, xs, lag, what):
    for g, x in enumerate(xs):
        m = len(x)
        rows = m - lag
        if rows < lag + 1:
            assert status[g] == GATED, (g, status[g])
            continue
        Xl = np.stack([x[lag - 1 - k:m - 1 - k] for k in range(lag)], axis=1)
        yl = x[lag:]
        M = exact_moments(Design(Xl, yl[:, None]))
        G, b = gram(M, lag, 1, True)
        if exact_det(G) == 0:
            continue
        assert status[g] == 0, (g, status[g])
        accept(beta[g], exact_solve(G, b), G, b, "qr", f"{what} group {g} ({rows} rows)")


# ---------------------------------------------------------------------------------------------------------------------
# the rank gate
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("q", [3, 8, 21, 22, 40, 65])
@pytest.mark.parametrize("solver", [QR, CHOL, SVD])
def test_gate_follows_the_exact_ratio(q, solver):
    """Gated iff ln det G - sum ln G_ii <= ln tol: at tol = R * 1.01 the gate fires, at R / 1.01 it does not, on K3 and
    on K5 (the group is the same rows)."""
    torch = _torch()
    p = q - 1
    d = int_design(11, 3000, p, near=(0, 1, 40))
    M = exact_moments(d)
    G, b = gram(M, p, 1, True)
    lnR = exact_gate_ratio(G)
    offs = torch.tensor([0, 3000], dtype=torch.int64).cuda()
    Z = _upload_groups(d.X, d.Y, np.ones(3000, bool), torch.float64)
    for f, gated in ((1.01, True), (1 / 1.01, False)):
        tol = math.exp(lnR) * f
        _, st, _ = _k3(M, p, 1, True, solver=solver, singular_x_tol=tol)
        assert (st == GATED) == gated, f"K3 solver {solver} q={q} tol=R*{f:.3f}: status {st}"
        beta, status = _dev().grouped_lin_reg(Z[:p], Z[p], offs, add_bias=True, singular_x_tol=tol, solver=solver)
        st5 = int(status[0])
        assert (st5 == GATED) == gated, f"K5 solver {solver} q={q} tol=R*{f:.3f}: status {st5}"
        if gated:
            assert torch.isnan(beta).all()
        else:
            accept(beta[0].cpu().numpy(), exact_solve(G, b), G, b, "qr", f"K5 gate-side q={q}")


SINGULAR = {"sum": ("sum", 0, 1, 2), "dup": ("dup", 0, 3), "zero": ("zero", 2)}


@pytest.mark.parametrize("kind", list(SINGULAR) + ["const_in_group"])
@pytest.mark.parametrize("q", [5, 22, 65])
def test_singular_designs_gate_and_solve(kind, q):
    """Exactly singular designs gate at every tol >= 1e-10 (K3, K5); ungated they give a finite β that satisfies the
    normal equations (documented deviation 1: a basic solution)."""
    torch = _torch()
    p = q - 1
    n = 3000
    if kind == "const_in_group":
        d = int_design(13, n, p)
        d.X[:, 1] = 5                        # constant within the group, next to the bias
    else:
        d = int_design(13, n, p, dep=SINGULAR[kind])
    M = exact_moments(d)
    G, b = gram(M, p, 1, True)
    assert exact_det(G) == 0
    offs = torch.tensor([0, n], dtype=torch.int64).cuda()
    Z = _upload_groups(d.X, d.Y, np.ones(n, bool), torch.float64)
    for tol in (1e-10, 1e-6, 0.5):
        for solver in (QR, CHOL, SVD):
            _, st, _ = _k3(M, p, 1, True, solver=solver, singular_x_tol=tol)
            assert st == GATED, (kind, q, tol, solver)
            _, status = _dev().grouped_lin_reg(Z[:p], Z[p], offs, add_bias=True, singular_x_tol=tol, solver=solver)
            assert int(status[0]) == GATED, (kind, q, tol, solver, "K5")
    Gf, bf = G.astype(np.float64), b.astype(np.float64)
    beta3, st, _ = _k3(M, p, 1, True)
    beta5, status = _dev().grouped_lin_reg(Z[:p], Z[p], offs, add_bias=True)
    for name, bh in (("K3", beta3[0]), ("K5", beta5[0].cpu().numpy())):
        assert np.isfinite(bh).all(), (name, kind, q)
        resid = np.abs(Gf @ bh - bf)
        assert np.all(resid <= 1e-9 * (np.abs(Gf) @ np.abs(bh) + np.abs(bf))), (name, kind, q, float(resid.max()))


# ---------------------------------------------------------------------------------------------------------------------
# coordinate descent and NNLS
# ---------------------------------------------------------------------------------------------------------------------
def cd_sweeps(G, b, n, ysum, bias, l1, l2, positive, sweeps):
    """K3 / K5's coordinate descent (faer_coordinate_descent), restated: fixed sweeps."""
    G, b = G.astype(np.float64), b.astype(np.float64)
    q = G.shape[0]
    p = q - int(bias)
    beta = np.zeros(q)
    for _ in range(sweeps):
        for j in range(p):
            part = sum(G[i, j] * beta[i] for i in range(q) if i != j)
            mu = b[j] - part
            if positive and mu < 0:
                beta[j] = 0.0
            else:
                beta[j] = np.sign(mu) * max(abs(mu) - n * l1, 0.0) / (G[j, j] + n * l2)
        if bias:
            beta[p] = (ysum - sum(beta[j] * G[j, p] for j in range(p))) / n
    return beta


def nnls_sweeps(G, b, bias, sweeps):
    G, b = G.astype(np.float64), b.astype(np.float64)
    q = G.shape[0]
    beta, mu = np.zeros(q), -b.copy()
    for _ in range(sweeps):
        for k in range(q):
            upd = beta[k] - mu[k] / G[k, k]
            if not bias or k < q - 1:
                upd = max(upd, 0.0)
            mu += (upd - beta[k]) * G[:, k]
            beta[k] = upd
    return beta


ITER = [(q, kind) for q in (3, 9, 21, 22, 40) for kind in ("lasso", "enet", "positive", "nnls")]


def _iter_kw(kind):
    return {"lasso": dict(method=CD, l1_reg=0.05), "enet": dict(method=CD, l1_reg=0.02, l2_reg=0.3),
            "positive": dict(method=CD, l1_reg=0.01, positive=True), "nnls": dict(method=NNLS)}[kind]


@pytest.mark.parametrize("q,kind", ITER)
def test_iterative_methods(q, kind):
    """Fixed sweeps (tol = 0): K3 and K5 agree to 1e-12 on the same exact M and with the restatement.  Converged: the
    KKT conditions hold on the exact G to 1e-9 relative."""
    torch = _torch()
    p, n = q - 1, 3000
    d = int_design(17 + q, n, p)
    M = exact_moments(d)
    G, b = gram(M, p, 1, True)
    kw = _iter_kw(kind)
    offs = torch.tensor([0, n], dtype=torch.int64).cuda()
    Z = _upload_groups(d.X, d.Y, np.ones(n, bool), torch.float64)
    sweeps = 3
    b3, _, _ = _k3(M, p, 1, True, tol=0.0, max_iter=sweeps, **kw)
    b5, _ = _dev().grouped_lin_reg(Z[:p], Z[p], offs, add_bias=True, tol=0.0, max_iter=sweeps, **kw)
    b5 = b5[0].cpu().numpy()
    if kind == "nnls":
        ref = nnls_sweeps(G, b, True, sweeps)
    else:
        ref = cd_sweeps(G, b, n, float(M[p, -1]), True, kw.get("l1_reg", 0.0), kw.get("l2_reg", 0.0),
                        kw.get("positive", False), sweeps)
    assert rel(b3[0], b5) <= 1e-12 and rel(b5, ref) <= 1e-12, (rel(b3[0], b5), rel(b5, ref))
    b3, _, _ = _k3(M, p, 1, True, tol=1e-15, max_iter=20000, **kw)
    b5, _ = _dev().grouped_lin_reg(Z[:p], Z[p], offs, add_bias=True, tol=1e-15, max_iter=20000, **kw)
    Gf, bf = G.astype(np.float64), b.astype(np.float64)
    for name, beta in (("K3", b3[0]), ("K5", b5[0].cpu().numpy())):
        scale = np.abs(Gf) @ np.abs(beta) + np.abs(bf)
        if kind == "nnls":
            mu = Gf @ beta - bf
            assert np.all(mu[:p] >= -1e-9 * scale[:p]), (name, mu)
            assert np.all(np.abs(beta[:p] * mu[:p]) <= 1e-9 * np.abs(beta[:p]) * scale[:p]), name
            assert abs(mu[p]) <= 1e-9 * scale[p], name
            continue
        l1, l2 = n * kw.get("l1_reg", 0.0), n * kw.get("l2_reg", 0.0)
        g = Gf @ beta - bf
        g[:p] += l2 * beta[:p]
        assert abs(g[p]) <= 1e-9 * scale[p], (name, "bias row")
        for j in range(p):
            s = 1e-9 * (scale[j] + l1)
            if beta[j] == 0.0:
                hi = math.inf if kw.get("positive") else l1 + s        # beta_j >= 0: only g_j >= -l1 binds
                assert -l1 - s <= g[j] <= hi, (name, kind, j, g[j], l1)
            else:
                assert beta[j] > 0 or not kw.get("positive"), (name, j)
                assert abs(g[j] + math.copysign(l1, beta[j])) <= s, (name, kind, j, g[j], l1)


# ---------------------------------------------------------------------------------------------------------------------
# the single report (K9) and the HC types
# ---------------------------------------------------------------------------------------------------------------------
def _report_single(X, y, p, se_type):
    import ctypes as C

    from polars_ds_extension_b200._lib import check, lib
    torch = _torch()
    n = X.shape[0]
    ld = (n + 31) // 32 * 32
    Zh = np.zeros((p + 1, ld))
    Zh[:p, :n] = X.T
    Zh[p, :n] = y
    Z = torch.from_numpy(Zh).cuda()
    q = p + 1
    out = torch.empty(8 * q, dtype=torch.float64, device="cuda")
    check(lib().pdsb_dev_report_f64(C.c_void_p(Z.data_ptr()), ld, C.c_void_p(Z[p].data_ptr()), None, None, n, p, 1,
                                    se_type, 1.0, C.c_void_p(out.data_ptr()),
                                    C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    return out.cpu().numpy().reshape(8, q)


@pytest.mark.parametrize("p,n", [(1, 40), (3, 200), (8, 500), (20, 3000)])
def test_single_report_exact(p, n):
    d = int_design(23 + p, n, p)
    M = exact_moments(d)
    G, _ = gram(M, p, 1, True)
    _check_report(_report_single(d.X, d.Y[:, 0], p, 0)[:6], exact_report(M, p, True), G, f"K9 p={p}")


@pytest.mark.parametrize("se_type", [1, 2, 3, 4])
@pytest.mark.parametrize("p,n", [(2, 30), (4, 300), (6, 500)])
def test_hc_reports_exact(se_type, p, n):
    """hc0..hc3 on K9 and on K17 (f64) against the exact sandwich on the group's exact residuals."""
    torch = _torch()
    d = int_design(29 + p, n, p)
    M = exact_moments(d)
    G, _ = gram(M, p, 1, True)
    ex = exact_report(M, p, True, rows=(d.X, d.Y[:, 0]), se_type=se_type)
    _check_report(_report_single(d.X, d.Y[:, 0], p, se_type)[:6], ex, G, f"K9 hc{se_type - 1} p={p}")
    Z = _upload_groups(d.X, d.Y, np.ones(n, bool), torch.float64)
    out, status = _dev().grouped_report(Z[:p], Z[p], torch.tensor([0, n], dtype=torch.int64).cuda(), add_bias=True,
                                        se_type=se_type)
    assert int(status[0]) == 0
    _check_report(out[0, :6].cpu().numpy(), ex, G, f"K17 hc{se_type - 1} p={p}")


# ---------------------------------------------------------------------------------------------------------------------
# conditioning sweep
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("decade", list(range(2, 13)))
def test_conditioning_sweep(decade):
    """kappa_2(G) from 1e2 to 1e12, one design per decade, on K3 (QR, Cholesky) and K5 (f64): the error stays within
    q u kappa_2 (or 10 LAPACK) at every decade, with no jump at a route or size boundary."""
    torch = _torch()
    d, p = conditioning_design(decade)
    n = d.n
    M = exact_moments(d)
    G, b = gram(M, p, 1, True)
    ex = exact_solve(G, b)
    for solver in (QR, CHOL):
        beta, st, _ = _k3(M, p, 1, True, solver=solver)
        assert st == 0
        accept(beta[0], ex, G, b, METHOD_NAME[solver], f"K3 kappa 1e{decade}")
    Z = _upload_groups(d.X, d.Y, np.ones(n, bool), torch.float64)
    beta, status = _dev().grouped_lin_reg(Z[:p], Z[p], torch.tensor([0, n], dtype=torch.int64).cuda(), add_bias=True)
    assert int(status[0]) == 0
    accept(beta[0].cpu().numpy(), ex, G, b, "qr", f"K5 kappa 1e{decade}")
