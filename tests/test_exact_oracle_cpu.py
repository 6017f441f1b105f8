"""The exact references of tests/exact_oracle.py on the CPU: they agree with LAPACK where LAPACK is accurate, the
moments are the float64 Z' W Z, and the acceptance rule sees one row.  For every case that tests/test_gpu_exact_solve.py
runs, the rule rejects the exact answer of the same problem with one row dropped or duplicated, with two coefficients
swapped, or with a ridge on the bias diagonal; so a device solve that passes it used every row, once."""
import math

import numpy as np
import pytest

from tests.exact_oracle import (METHOD_INV, U64, Design, accepted, conditioning_design, exact_gate_ratio, exact_gated,
                                exact_inverse, exact_moments, exact_report, exact_solve, gram, int_design, k3_cases,
                                k3_design, k3_moments, k5_case, k5_cases, k5_solve_in_shared, k5_switch_q, kappa,
                                K5_FULL_Q, sizes_full, sizes_sweep, student_t_ppf975, student_t_sf2)


@pytest.mark.parametrize("q", [1, 2, 5, 12, 30])
def test_exact_solve_matches_numpy_when_well_conditioned(q):
    d = int_design(q, 500, q, tag=False)
    G, b = gram(exact_moments(d), q, 1, False)
    assert kappa(G) < 1e3
    ex = exact_solve(G, b)
    ref = np.linalg.solve(G.astype(np.float64), b.astype(np.float64))
    assert np.max(np.abs(ex - ref)) <= 1e-14 * np.max(np.abs(ref))
    Gi = exact_inverse(G)
    assert np.max(np.abs(Gi @ G.astype(np.float64) - np.eye(q))) < 1e-13


@pytest.mark.parametrize("n,p,t,weights,drop", [(7, 3, 1, False, 0.0), (300, 5, 2, True, 0.2), (1000, 12, 4, True, 0.5)])
def test_exact_moments_are_the_float64_gram(n, p, t, weights, drop):
    d = int_design(n, n, p, t, weights=weights, drop_frac=drop)
    M = exact_moments(d)
    Z = np.concatenate([d.X, d.Y, np.ones((n, 1), np.int64)], axis=1)
    W = (np.ones(n, np.int64) if d.w is None else d.w) * d.kept()
    Mi = (Z * W[:, None]).T @ Z                                 # int64 end to end
    assert np.array_equal(M, Mi)
    Zf = Z.astype(np.float64)
    assert np.array_equal(M.astype(np.float64), (Zf * W[:, None]).T @ Zf)
    assert M[-1, -1] == W.sum()


def test_exact_statistics():
    """The t distribution of mpmath against scipy, and the exact report against a float64 restatement."""
    from scipy import stats
    for dof in (1, 5, 37, 2000):
        assert abs(float(student_t_ppf975(dof)) - stats.t.ppf(0.975, dof)) < 1e-12 * stats.t.ppf(0.975, dof)
        for tv in (0.3, 2.0, 7.5):
            assert abs(float(student_t_sf2(tv, dof)) - 2 * stats.t.sf(tv, dof)) < 1e-10 * 2 * stats.t.sf(tv, dof)
    d = int_design(3, 200, 3)
    M = exact_moments(d)
    Xb = np.concatenate([d.X, np.ones((200, 1))], axis=1)
    y = d.Y[:, 0].astype(np.float64)
    beta = np.linalg.lstsq(Xb, y, rcond=None)[0]
    e = y - Xb @ beta
    Ginv = np.linalg.inv(Xb.T @ Xb)
    for se_type, se in ((0, np.sqrt(e @ e / 196 * np.diag(Ginv))),
                        (1, np.sqrt(np.diag(Ginv @ (Xb.T * e ** 2) @ Xb @ Ginv)))):
        rows = None if se_type == 0 else (d.X, d.Y[:, 0])
        rep = exact_report(M, 3, True, rows=rows, se_type=se_type)
        assert np.allclose(rep[0], beta, rtol=1e-12, atol=0)
        assert np.allclose(rep[1], se, rtol=1e-10, atol=0)
        assert np.allclose(rep[3], 2 * stats.t.sf(np.abs(beta / se), 196), rtol=1e-8)


def _rejections(Z, p, t, bias, target=0, method="qr"):
    """The rule on the problem of the rows Z = [X | Y | 1] rejects: one row dropped, one row duplicated, the two
    coefficients farthest apart swapped, 1 added to the bias diagonal.  Returns q u kappa_2(G)."""
    Zf = Z.astype(np.float64)
    M = (Zf.T @ Zf).astype(np.int64)
    G, b = gram(M, p, t, bias, target)
    ex = exact_solve(G, b)
    assert ex is not None
    r = Z.shape[0] // 2
    z = Z[r].astype(np.int64)
    for sign, what in ((-1, "dropped"), (1, "duplicated")):
        Gp, bp = gram(M + sign * np.outer(z, z), p, t, bias, target)
        xp = exact_solve(Gp, bp)
        assert xp is None or not accepted(xp, ex, G, b, method), f"one row {what} passes the rule"
    if ex.size > 1:
        i, j = int(np.argmax(ex)), int(np.argmin(ex))
        sw = ex.copy()
        sw[[i, j]] = sw[[j, i]]
        assert not accepted(sw, ex, G, b, method), "two coefficients swapped pass the rule"
    if bias:
        Gp = G.copy()
        Gp[-1, -1] += 1
        assert not accepted(exact_solve(Gp, b), ex, G, b, method), "a ridge on the bias diagonal passes the rule"
    return G.shape[0] * U64 * kappa(G)


@pytest.mark.parametrize("q,bias", k3_cases())
def test_rule_sees_one_row_k3(q, bias):
    p = q - int(bias)
    d = k3_design()
    Z = np.concatenate([d.X[:, :p], d.Y[:, :1], np.ones((d.n, 1), np.int64)], axis=1)
    assert np.array_equal((Z.astype(np.float64).T @ Z).astype(np.int64), k3_moments(p, 1))
    for method in ("qr", "chol", "svd"):
        assert _rejections(Z, p, 1, bias, method=method) <= 1e-8


@pytest.mark.parametrize("q,bias", k5_cases())
def test_rule_sees_one_row_k5(q, bias):
    """The largest group of every grouped case (the hardest to see one row in)."""
    p = q - int(bias)
    sizes = sizes_full(q) if q in K5_FULL_Q else sizes_sweep(q)
    X, Y, keep, offsets, spans = k5_case(7000 + q, p, bias, sizes)
    s, e = max(spans, key=lambda sp: sp[1] - sp[0])
    Z = np.concatenate([X[s:e], Y[s:e], np.ones((e - s, 1), np.int64)], axis=1)[keep[s:e]]
    assert _rejections(Z, p, 1, bias) <= 1e-8
    # every group the GPU test solves has an exact answer; the ones that gate for their row count have < q kept rows
    assert offsets[-1] == X.shape[0]
    for g, (s, e) in enumerate(spans):
        if keep[s:e].sum() >= q:
            G, b = gram(exact_moments(Design(X[s:e], Y[s:e], None, keep[s:e])), p, 1, bias)
            assert exact_solve(G, b) is not None, g


@pytest.mark.parametrize("q", [3, 8, 21, 22, 40, 65])
def test_gate_cases_sit_on_both_sides(q):
    """The gate tests' tolerances R * 1.01 and R / 1.01 fall on opposite sides of the exact decision, and an exactly
    singular design gates at any tolerance."""
    d = int_design(11, 3000, q - 1, near=(0, 1, 40))
    G, _ = gram(exact_moments(d), q - 1, 1, True)
    lnR = exact_gate_ratio(G)
    assert math.isfinite(lnR)
    assert exact_gated(G, math.exp(lnR) * 1.01) and not exact_gated(G, math.exp(lnR) / 1.01)
    assert q * U64 * kappa(G) < 1e-2 * math.log(1.01)     # the device's ln det is far more accurate than the margin
    S = gram(exact_moments(int_design(13, 3000, q - 1, dep=("dup", 0, 3 if q > 4 else 1))), q - 1, 1, True)[0]
    assert exact_gated(S, 1e-300)


def test_k5_workspace_switch_restated():
    """group_solve_launch (k5_solve.h:80): lin_reg's workspace leaves shared memory after 21 coefficients, the report's
    (nrhs = q + 1) earlier, the multi-target fit's (three targets) at 20; the GPU sweeps cover both sides of each."""
    assert k5_switch_q(True) == 21 and k5_switch_q(False) == 21
    assert k5_switch_q(True, METHOD_INV) == 17
    assert k5_switch_q(True, 0, 3) == 20
    qs = [q for q, _ in k5_cases()]
    assert set(range(1, 66)) <= set(qs)
    assert k5_solve_in_shared(20, 21) and not k5_solve_in_shared(21, 22)


def test_conditioning_sweep_covers_every_decade():
    for dec in range(2, 13):
        d, p = conditioning_design(dec)
        G, _ = gram(exact_moments(d), p, 1, True)
        assert dec <= math.log10(kappa(G)) < dec + 1
