"""NumPy restatements of pl_smooth_spline (the reference's src/num_ext/splines.rs).

* ``dense_smooth_spline``: the reference's dense algorithm (faer_smooth_spline) with its error strings: dense Q
  (n x n-2), R^-1 Q' by a Cholesky of R, M = I + lambda Q R^-1 Q', solved by Cholesky with the column-pivoted QR fallback.
  O(n^2) memory, O(n^3) time: for n up to a few thousand.
* ``reinsch_ld``: the Reinsch band system (R + lambda Q'Q) gamma = Q'y, g = y - lambda Q gamma, solved by a pentadiagonal
  LDL' in long double (80-bit on x86-64).  The truth for the accuracy rule.
* ``reinsch_f64``: the same band system by ``scipy.linalg.solveh_banded`` in f64: the sequential f64 baseline.
"""
from __future__ import annotations

import numpy as np
import scipy.linalg as sla

NOT_INCREASING = "Input is not increasing."


class SplineError(ValueError):
    pass


def check_inputs(x, y):
    """The symbol's checks in the reference's order (nulls, lengths, n >= 3, strictly increasing x)."""
    if any(v is None for v in x) or any(v is None for v in y):
        raise SplineError("Input x or y has nulls.")
    x = np.asarray(x, dtype=np.float64)
    y = np.asarray(y, dtype=np.float64)
    if len(x) != len(y):
        raise SplineError("Input lengths are not the same.")
    if len(x) < 3:
        raise SplineError("Must have >= 3 points.")
    with np.errstate(invalid="ignore"):
        if np.any(np.diff(x) <= 0.0):          # a NaN gap compares False: not caught, as in the reference
            raise SplineError(NOT_INCREASING)
    return x, y


def dense_smooth_spline(x, y, lam: float) -> np.ndarray:
    x, y = check_inputs(x, y)
    if lam == 0.0:                             # M = I: the reference solves I g = y
        return y.copy()
    n = len(x)
    m = n - 2
    with np.errstate(all="ignore"):
        h = np.diff(x)
        Q = np.zeros((n, m))
        j = np.arange(m)
        Q[j, j] = 1.0 / h[:-1]
        Q[j + 1, j] = -(1.0 / h[:-1] + 1.0 / h[1:])
        Q[j + 2, j] = 1.0 / h[1:]
        R = np.zeros((m, m))
        R[j, j] = (h[:-1] + h[1:]) / 3.0
        R[j[:-1], j[:-1] + 1] = h[1:-1] / 6.0
        R[j[:-1] + 1, j[:-1]] = h[1:-1] / 6.0
        try:
            xx = sla.cho_solve(sla.cho_factor(R, lower=True, check_finite=False), Q.T, check_finite=False)
        except np.linalg.LinAlgError:
            return np.full(n, np.nan)          # the reference's sp_cholesky error path (not reached for increasing x)
        M = np.eye(n) + lam * (Q @ xx)
        try:
            return sla.cho_solve(sla.cho_factor(M, lower=True, check_finite=False), y, check_finite=False)
        except np.linalg.LinAlgError:
            Qf, Rf, piv = sla.qr(M, pivoting=True, check_finite=False)
            z = sla.solve_triangular(Rf, Qf.T @ y, check_finite=False)
            g = np.empty(n)
            g[piv] = z
            return g


def bands(x, y, lam: float, dtype=np.float64):
    """Bands of A = R + lambda Q'Q (diagonal d, first e, second f; length m each, the last one / two unused) and
    rhs = Q'y; also (a, b, c), the three nonzeros of every column of Q."""
    x = np.asarray(x, dtype=dtype)
    y = np.asarray(y, dtype=dtype)
    lam = dtype(lam)
    h = np.diff(x)
    r = dtype(1) / h
    a, c = r[:-1], r[1:]
    b = -(a + c)
    m = len(x) - 2
    d = (h[:-1] + h[1:]) / dtype(3) + lam * (a * a + b * b + c * c)
    e = np.zeros(m, dtype=dtype)
    f = np.zeros(m, dtype=dtype)
    e[:-1] = h[1:-1] / dtype(6) + lam * (b[:-1] * a[1:] + c[:-1] * b[1:])
    f[:-2] = lam * c[:-2] * a[2:]
    rhs = a * y[:-2] + b * y[1:-1] + c * y[2:]
    return d, e, f, rhs, (a, b, c)


def _g_from_gamma(y, gam, lam, abc):
    a, b, c = abc
    qg = np.zeros(len(y), dtype=gam.dtype)
    qg[:-2] += a * gam
    qg[1:-1] += b * gam
    qg[2:] += c * gam
    return y - lam * qg


def reinsch_ld(x, y, lam: float) -> np.ndarray:
    """g by a long-double pentadiagonal LDL' of the band system (returned as f64)."""
    x, y = check_inputs(x, y)
    ld = np.longdouble
    if lam == 0.0:
        return y.copy()
    d, e, f, rhs, abc = bands(x, y, lam, ld)
    m = len(d)
    dd = [ld(0)] * m
    l1 = [ld(0)] * (m + 1)       # l1[j] = L[j, j-1]
    l2 = [ld(0)] * (m + 2)       # l2[j] = L[j, j-2]
    dl, el, fl = d.tolist(), e.tolist(), f.tolist()
    for j in range(m):
        v = dl[j]
        if j >= 1:
            v -= l1[j] * l1[j] * dd[j - 1]
        if j >= 2:
            v -= l2[j] * l2[j] * dd[j - 2]
        dd[j] = v
        if j + 1 < m:
            t = el[j]
            if j >= 1:
                t -= l1[j] * l2[j + 1] * dd[j - 1]
            l1[j + 1] = t / v
        if j + 2 < m:
            l2[j + 2] = fl[j] / v
    z = rhs.tolist()
    for j in range(m):
        if j >= 1:
            z[j] -= l1[j] * z[j - 1]
        if j >= 2:
            z[j] -= l2[j] * z[j - 2]
    gam = [ld(0)] * m
    for j in range(m - 1, -1, -1):
        v = z[j] / dd[j]
        if j + 1 < m:
            v -= l1[j + 1] * gam[j + 1]
        if j + 2 < m:
            v -= l2[j + 2] * gam[j + 2]
        gam[j] = v
    g = _g_from_gamma(np.asarray(y, dtype=ld), np.array(gam, dtype=ld), ld(lam), abc)
    return g.astype(np.float64)


def reinsch_f64(x, y, lam: float) -> np.ndarray:
    """g by scipy.linalg.solveh_banded on the f64 band system (sequential banded Cholesky)."""
    x, y = check_inputs(x, y)
    if lam == 0.0:
        return y.copy()
    d, e, f, rhs, abc = bands(x, y, lam)
    m = len(d)
    ab = np.zeros((3, m))
    ab[0, 2:] = f[:-2]
    ab[1, 1:] = e[:-1]
    ab[2, :] = d
    gam = sla.solveh_banded(ab, rhs, lower=False, check_finite=False)
    return _g_from_gamma(y, gam, lam, abc)


def rel_err(g, ref, y) -> float:
    """max |g - ref| / max |y|"""
    return float(np.max(np.abs(np.asarray(g) - np.asarray(ref))) / np.max(np.abs(y)))
