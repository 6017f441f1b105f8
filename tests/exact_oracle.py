"""Exact references for the moments pass and the dense solves, on integer data (CPU only).

On designs whose values are small integers every moments route is exact: an f32 product of two integers below 2^12 is
exact, and an f32 chain of such products stays exact while its partial sums stay below 2^24.  The device moments must
then equal the int64 moments bit for bit.  With exact moments the solution of the normal equations is a rational number,
computed here by fraction-free elimination over the integers (sympy's DomainMatrix over ZZ), so any error left in a
device solve is the solver's own.  It is held to one rule (`accept`):

    err = rel(got, exact)   (vector-relative, as parity_rule.rel)
    accept iff err <= max(10 * err_lapack, q * u64 * kappa_2(G), 8 * u64)

where err_lapack is the error of the same method in LAPACK float64 on the same G (pivoted QR, Cholesky, or an
eigen-decomposition for svd).  The floor of 8 ulps is for the best-conditioned problems (q = 1, kappa = 1), where
LAPACK's answer can happen to be the correctly rounded one and a Householder step on a 1 x 1 system still rounds a few
times.  On the designs below one dropped or duplicated row moves the exact answer by orders of
magnitude more than that bound (tests/test_exact_oracle_cpu.py proves it for every case the GPU tests run).
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from fractions import Fraction
from functools import lru_cache
from typing import Optional

import mpmath
import numpy as np
import scipy.linalg as sla
from sympy import ZZ
from sympy.polys.matrices import DomainMatrix
from sympy.polys.matrices.exceptions import DMNonInvertibleMatrixError

from tests.parity_rule import rel

U64 = 2.0 ** -53
FLOOR_ULPS = 8 * U64
TAG_MOD, TAG_OFF = 251, 125          # row-tag column (row % 251) - 125: no row of a design is all zero


# ---------------------------------------------------------------------------------------------------------------------
# designs
# ---------------------------------------------------------------------------------------------------------------------
@dataclass
class Design:
    X: np.ndarray                      # (n, p) int64
    Y: np.ndarray                      # (n, t) int64
    w: Optional[np.ndarray] = None     # (n,) int64 weights 1..4, or None
    keep: Optional[np.ndarray] = None  # (n,) bool: False = a masked / NaN (null) row, None = every row kept

    @property
    def n(self):
        return self.X.shape[0]

    def kept(self):
        return np.ones(self.n, bool) if self.keep is None else self.keep


def int_design(seed, n, p, t=1, tag=True, lo=-8, hi=8, weights=False, drop_frac=0.0, row0=0, near=None, dep=None,
               scale=None) -> Design:
    """An int64 design of n rows, p features, t targets.

    Features are uniform in [lo, hi]; with ``tag`` the last feature is the row tag (row0 + r) % 251 - 125.  Targets are
    small integer combinations of up to four non-tag features plus integer noise, so |y| <= 72.  weights: 1..4 per row.
    drop_frac: that share of rows is not kept (a mask of 0, or NaN rows for the null-dropping entries).
    Conditioning knobs:
      near  = (a, b, k): x_b = x_a + e with e = +-1 on k rows and 0 elsewhere (near-collinear, kappa ~ n / k);
      dep   = ("sum", a, b, c): x_c = x_a + x_b;  ("dup", a, b): x_b = x_a;  ("zero", a): x_a = 0 (exactly singular);
      scale = {j: s}: column j times 2^s (exact in floating point).
    """
    rng = np.random.default_rng(seed)
    X = rng.integers(lo, hi + 1, size=(n, p), dtype=np.int64)
    if tag and p >= 1:
        X[:, p - 1] = (np.arange(row0, row0 + n, dtype=np.int64) % TAG_MOD) - TAG_OFF
    if near is not None:
        a, b, k = near
        e = np.zeros(n, np.int64)
        rows = rng.choice(n, size=min(k, n), replace=False)
        e[rows] = rng.choice(np.array([-1, 1]), size=rows.size)
        X[:, b] = X[:, a] + e
    if dep is not None:
        if dep[0] == "sum":
            X[:, dep[3]] = X[:, dep[1]] + X[:, dep[2]]
        elif dep[0] == "dup":
            X[:, dep[2]] = X[:, dep[1]]
        elif dep[0] == "zero":
            X[:, dep[1]] = 0
        else:
            raise ValueError(dep)
    if scale:
        for j, s in scale.items():
            X[:, j] <<= s
    free = [j for j in range(p) if not (tag and j == p - 1)][:4]
    Y = rng.integers(-8, 9, size=(n, t), dtype=np.int64)
    for c in range(t):
        for j in free:
            Y[:, c] += int(rng.integers(-2, 3)) * np.clip(X[:, j], -8, 8)
    w = rng.integers(1, 5, size=n, dtype=np.int64) if weights else None
    keep = (rng.random(n) >= drop_frac) if drop_frac > 0 else None
    return Design(X, Y, w, keep)


def f32_chain_ok(d: Design, chain: int) -> bool:
    """Every f32 chain of `chain` rows of w z_i z_j sums integers below 2^24 (then it is exact in any order)."""
    zmax = max(int(np.abs(d.X).max(initial=1)), int(np.abs(d.Y).max(initial=1)), 1)
    wmax = 1 if d.w is None else int(d.w.max())
    return chain * wmax * zmax * zmax < 2 ** 24


def exact_moments(d: Design) -> np.ndarray:
    """M = [X | Y | 1]' diag(w keep) [X | Y | 1] in int64 ((p + t + 1)^2), asserting no entry reaches 2^53 (so the
    float64 matrix product below, whose every partial sum is an integer of at most that size, is exact)."""
    n = d.n
    Z = np.concatenate([d.X, d.Y, np.ones((n, 1), np.int64)], axis=1)
    wk = np.ones(n, np.int64) if d.w is None else d.w.astype(np.int64)
    wk = wk * d.kept()
    A = np.abs(Z).max(axis=0).astype(np.float64)
    bound = np.outer(A, A) * float(wk.sum())
    assert bound.max() < 2.0 ** 53, "exact moments would overflow 2^53"
    Zf = Z.astype(np.float64)
    M = (Zf * wk[:, None].astype(np.float64)).T @ Zf
    Mi = M.astype(np.int64)
    assert np.array_equal(Mi.astype(np.float64), M)
    return Mi


def gram(M, p, t=1, bias=True, target=0):
    """(G, b) of a fit of target `target` on p features (and the bias) from the moments of [X | Y | 1]."""
    idx = list(range(p)) + ([p + t] if bias else [])
    G = M[np.ix_(idx, idx)].copy()
    b = M[idx, p + target].copy()
    return G, b


# ---------------------------------------------------------------------------------------------------------------------
# exact linear algebra (cached by the bytes of the integer inputs)
# ---------------------------------------------------------------------------------------------------------------------
def _dm(A):
    A = np.asarray(A)
    assert A.dtype.kind in "iu", "exact routines take integer matrices"
    rows = [[ZZ(int(v)) for v in r] for r in A.reshape(A.shape[0], -1)]
    return DomainMatrix(rows, (A.shape[0], A.reshape(A.shape[0], -1).shape[1]), ZZ)


_SOLVE_CACHE: dict = {}


def exact_solve_frac(G, B):
    """G^-1 B as a list of columns of Fractions, or None when G is singular."""
    G = np.ascontiguousarray(G, np.int64)
    B = np.ascontiguousarray(np.asarray(B).reshape(G.shape[0], -1), np.int64)
    key = (G.shape, G.tobytes(), B.shape, B.tobytes())
    if key not in _SOLVE_CACHE:
        try:
            num, den = _dm(G).solve_den(_dm(B))
        except DMNonInvertibleMatrixError:
            _SOLVE_CACHE[key] = None
        else:
            den = int(den)
            rows = num.to_list()
            _SOLVE_CACHE[key] = [[Fraction(int(rows[i][c]), den) for i in range(G.shape[0])] for c in range(B.shape[1])]
    return _SOLVE_CACHE[key]


def exact_solve(G, B):
    """G^-1 B correctly rounded to float64, shape of B ((q,) or (q, k)); None when G is singular."""
    x = exact_solve_frac(G, B)
    if x is None:
        return None
    out = np.array([[float(v) for v in col] for col in x]).T
    return out[:, 0] if np.asarray(B).ndim == 1 else out


@lru_cache(maxsize=None)
def _det_cached(shape, data):
    G = np.frombuffer(data, np.int64).reshape(shape)
    return int(_dm(G).det())


def exact_det(G) -> int:
    G = np.ascontiguousarray(G, np.int64)
    return _det_cached(G.shape, G.tobytes())


def exact_gate_ratio(G) -> float:
    """ln det G - sum ln G_ii from the exact determinant (the rank gate's statistic); -inf when det G <= 0 or a
    diagonal entry is <= 0."""
    G = np.asarray(G, np.int64)
    d = exact_det(G)
    diag = [int(v) for v in np.diag(G)]
    if d <= 0 or min(diag, default=1) <= 0:
        return -math.inf
    with mpmath.workdps(50):
        r = mpmath.log(d) - mpmath.fsum(mpmath.log(v) for v in diag)
        return float(r)


def exact_gated(G, tol) -> bool:
    """The rank gate's exact decision: gated iff some G_ii <= 0 or ln det G - sum ln G_ii <= ln tol."""
    return exact_gate_ratio(G) <= math.log(tol)


def exact_inverse(G):
    q = np.asarray(G).shape[0]
    return exact_solve(G, np.eye(q, dtype=np.int64))


def kappa(G) -> float:
    """kappa_2(G) of a symmetric positive definite G: the extreme eigenpairs from LAPACK, each eigenvalue refined as the
    Rayleigh quotient of its vector evaluated in mpmath (the error of a Rayleigh quotient is quadratic in the vector's)."""
    Gf = np.asarray(G, np.float64)
    lam, V = np.linalg.eigh(Gf)
    out = []
    with mpmath.workdps(40):
        Gm = [[mpmath.mpf(int(v)) for v in r] for r in np.asarray(G, np.int64)] if np.asarray(G).dtype.kind in "iu" \
            else [[mpmath.mpf(float(v)) for v in r] for r in Gf]
        for k in (0, -1):
            v = [mpmath.mpf(float(x)) for x in V[:, k]]
            Gv = [mpmath.fsum(a * b for a, b in zip(row, v)) for row in Gm]
            out.append(mpmath.fsum(a * b for a, b in zip(v, Gv)) / mpmath.fsum(a * a for a in v))
    lo, hi = out
    return math.inf if lo <= 0 else float(hi / lo)


# ---------------------------------------------------------------------------------------------------------------------
# the acceptance rule
# ---------------------------------------------------------------------------------------------------------------------
def lapack_solve(G, B, method="qr"):
    """The same method in LAPACK float64 on the same G: pivoted QR, Cholesky, or eigh for svd."""
    Gf = np.asarray(G, np.float64)
    Bf = np.asarray(B, np.float64)
    if method == "qr":
        Q, R, P = sla.qr(Gf, pivoting=True)
        z = sla.solve_triangular(R, Q.T @ Bf)
        x = np.empty_like(z)
        x[P] = z
        return x
    if method == "chol":
        return sla.cho_solve(sla.cho_factor(Gf), Bf)
    if method == "svd":
        lam, V = np.linalg.eigh(Gf)
        return V @ ((V.T @ Bf) / (lam if Bf.ndim == 1 else lam[:, None]))
    raise ValueError(method)


def bound(G, B, exact, method="qr"):
    """max(10 err_lapack, q u64 kappa_2(G), 8 u64): the largest error the rule accepts for this problem."""
    q = np.asarray(G).shape[0]
    return max(10.0 * rel(lapack_solve(G, B, method), exact), q * U64 * kappa(G), FLOOR_ULPS)


def accepted(got, exact, G, B, method="qr") -> bool:
    return bool(np.all(np.isfinite(got))) and rel(got, exact) <= bound(G, B, exact, method)


def accept(got, exact, G, B, method="qr", what=""):
    err, lim = rel(got, exact), bound(G, B, exact, method)
    assert np.all(np.isfinite(got)) and err <= lim, f"{what}: error {err:.3e} > bound {lim:.3e} (method {method})"
    return err


# ---------------------------------------------------------------------------------------------------------------------
# exact report: beta, classic / HC standard errors, t, p and the 95 % interval
# ---------------------------------------------------------------------------------------------------------------------
def student_t_sf2(tval, dof):
    """2 P(T > |t|) for T ~ t(dof): the regularised incomplete beta I_{dof / (dof + t^2)}(dof / 2, 1 / 2), 50 digits."""
    with mpmath.workdps(50):
        t2 = mpmath.mpf(tval) ** 2
        return mpmath.betainc(mpmath.mpf(dof) / 2, mpmath.mpf(1) / 2, 0, mpmath.mpf(dof) / (dof + t2), regularized=True)


def student_t_ppf975(dof):
    """The 0.975 quantile of t(dof) in mpmath: the root of 2 P(T > x) = 0.05, from scipy's float64 value."""
    from scipy import stats
    x0 = float(stats.t.ppf(0.975, dof))
    with mpmath.workdps(50):
        f = lambda x: student_t_sf2(x, dof) - mpmath.mpf("0.05")
        return mpmath.findroot(f, (mpmath.mpf(x0), mpmath.mpf(x0) * (1 + mpmath.mpf(2) ** -30)), solver="secant")


def exact_report(M, p, bias, rows=None, se_type=0):
    """The report block (beta, se, t, p, ci_lo, ci_hi) of the fit of y on p features from exact moments M (t = 1), as
    float64 (6, q), or None when G is singular.  rows: (Xk (m, p) int, yk (m,) int) of the kept rows, needed for the
    HC types (se_type 1..4 = hc0..hc3); classic se reads the moments only."""
    G, b = gram(M, p, 1, bias)
    q = G.shape[0]
    n = int(M[-1, -1])
    beta = exact_solve_frac(G, b)
    if beta is None:
        return None
    beta = beta[0]
    Ginv = exact_solve_frac(G, np.eye(q, dtype=np.int64))     # Ginv[c][i] = (G^-1)[i][c]
    dof = n - q
    if se_type == 0:
        yy = Fraction(int(M[p, p]))
        rss = yy - sum(Fraction(int(b[i])) * beta[i] for i in range(q))
        var = [rss / dof * Ginv[i][i] for i in range(q)]
    else:
        Xk, yk = rows
        Zk = np.concatenate([Xk, np.ones((Xk.shape[0], 1), np.int64)], axis=1) if bias else Xk
        meat = [[Fraction(0)] * q for _ in range(q)]
        for r in range(Zk.shape[0]):
            z = [int(v) for v in Zk[r]]
            e = Fraction(int(yk[r])) - sum(z[i] * beta[i] for i in range(q))
            wgt = e * e
            if se_type >= 3:
                h = sum(z[a] * sum(Ginv[c][a] * z[c] for c in range(q)) for a in range(q))
                wgt = wgt / (1 - h) if se_type == 3 else wgt / ((1 - h) * (1 - h))
            for a in range(q):
                for c in range(q):
                    meat[a][c] += wgt * z[a] * z[c]
        var = []
        for i in range(q):
            v = sum(Ginv[r][i] * sum(meat[r][c] * Ginv[i][c] for c in range(q)) for r in range(q))
            if se_type == 2:
                v = v * Fraction(n, dof)
            var.append(v)
    ta = student_t_ppf975(dof)
    out = np.empty((6, q))
    with mpmath.workdps(50):
        for i in range(q):
            bm = mpmath.mpf(beta[i].numerator) / beta[i].denominator
            se = mpmath.sqrt(mpmath.mpf(var[i].numerator) / var[i].denominator)
            tv = bm / se
            out[:, i] = [float(bm), float(se), float(tv), float(student_t_sf2(tv, dof)), float(bm - ta * se),
                         float(bm + ta * se)]
    return out


# ---------------------------------------------------------------------------------------------------------------------
# K5's workspace switch, restated
# ---------------------------------------------------------------------------------------------------------------------
METHOD_INV = 4


def k5_solve_in_shared(p, q, method=0, t=1):
    """Whether group_solve runs on the shared-memory workspace of a 32-thread CTA (True) or on the global one.
    Restates group_solve_launch and group_solve_nrhs (polars_ds_extension_b200/csrc/kernels/k5_solve.h:69-85); the two
    change together."""
    nrhs = q + 1 if method == METHOD_INV else t
    per_thread = (q * q + q * nrhs + q + (p + t + 1) * (p + t + 2) // 2) * 8
    return per_thread * 32 <= 200 * 1024


def k5_switch_q(bias=True, method=0, t=1):
    """The last q whose solve stays in shared memory."""
    last = 0
    for q in range(1, 66):
        p = q - int(bias)
        if p >= 0 and k5_solve_in_shared(p, q, method, t):
            last = q
    return last


# ---------------------------------------------------------------------------------------------------------------------
# the cases of tests/test_gpu_exact_solve.py (tests/test_exact_oracle_cpu.py proves the rule sees one row in each)
# ---------------------------------------------------------------------------------------------------------------------
PMAX, TMAX = 65, 4


@lru_cache(maxsize=None)
def k3_design():
    """K3's design: 4000 rows, 65 features, 4 targets (no row tag: every feature is uniform in [-8, 8])."""
    return int_design(31337, 4000, PMAX, TMAX, tag=False)


@lru_cache(maxsize=None)
def _k3_full_moments():
    return exact_moments(k3_design())


def k3_moments(p, t):
    """Exact moments of [X[:, :p] | Y[:, :t] | 1] of k3_design()."""
    idx = list(range(p)) + [PMAX + c for c in range(t)] + [PMAX + TMAX]
    return _k3_full_moments()[np.ix_(idx, idx)]


def k3_cases():
    return [(q, bias) for q in range(1, PMAX + 1) for bias in (False, True) if q - int(bias) >= 1]


# ---------------------------------------------------------------------------------------------------------------------
# the grouped cases of tests/test_gpu_exact_solve.py (tests/test_exact_oracle_cpu.py proves the rule sees one row in each)
# ---------------------------------------------------------------------------------------------------------------------
def sizes_full(q):
    """Group sizes at the boundaries: empty, one row, q - 1 / q / q + 1 rows, one 128-row trip of the register kernel and
    either side of it, one 8192-row item and either side, two items, and 3 * 8192 + 1 rows (three items of 8320 rows
    and a short fourth: item_range's 128-row rounding)."""
    return [0, 1, q - 1, q, q + 1, 127, 128, 129, 8191, 8192, 8193, 16385, 3 * 8192 + 1]


def sizes_sweep(q):
    return [q - 1, q, q + 1, 129, 8193, 3 * 8192 + 1]


def k5_case(seed, p, bias, sizes, t=1, nulls=True):
    """Groups of the given sizes, back to back, as one design; with `nulls` two more groups of q + 1 rows of which one
    (-> q kept rows) and two (-> q - 1 kept rows, gated) are NaN.  Every group with at least q kept rows is nonsingular
    (rows redrawn otherwise).  Returns (X, Y, keep, offsets, [(start, end)])."""
    q = p + int(bias)
    sizes = [max(m, 0) for m in sizes] + ([q + 1, q + 1] if nulls else [])
    Xs, Ys, ks, spans, r0 = [], [], [], [], 0
    for g, m in enumerate(sizes):
        for attempt in range(50):
            d = int_design(seed + 1000 * g + attempt, m, p, t, row0=r0)
            keep = np.ones(m, bool)
            if nulls and g >= len(sizes) - 2:
                keep[1:1 + (1 if g == len(sizes) - 2 else 2)] = False
            if keep.sum() < q:
                break
            G, _ = gram(exact_moments(Design(d.X, d.Y, None, keep)), p, t, bias)
            if exact_det(G) != 0:
                break
        Xs.append(d.X)
        Ys.append(d.Y)
        ks.append(keep)
        spans.append((r0, r0 + m))
        r0 += m
    offsets = np.array([0] + [e for _, e in spans], np.int64)
    return np.concatenate(Xs), np.concatenate(Ys), np.concatenate(ks), offsets, spans


K5_FULL_Q = sorted({1, 2, 3, k5_switch_q(True), k5_switch_q(True) + 1, k5_switch_q(False), k5_switch_q(False) + 1,
                    40, 64, 65})


def k5_cases():
    out = []
    for q in range(1, 66):
        for bias in (True, False):
            p = q - int(bias)
            if p < 1 or p > 64 or (bias and q % 2 == 1 and q not in K5_FULL_Q) or (not bias and q % 2 == 0 and q not in K5_FULL_Q):
                continue
            out.append((q, bias))
    return out




@lru_cache(maxsize=None)
def _conditioning_designs():
    """decade -> (kappa_2, knobs) of the first bias design of 6 features on 4000 rows (without, then with the row tag),
    with x_1 = x_0 + e (e = +-1 on k rows) and x_2 scaled by 2^s, whose kappa_2(G) falls in [10^decade, 10^(decade + 1))."""
    found = {}
    for tag in (False, True):
        for s in range(0, 13):
            for k in (4000, 1000, 300, 100, 30, 10, 3, 1):
                d = int_design(41, 4000, 6, tag=tag, near=(0, 1, k), scale={2: s} if s else None)
                G, _ = gram(exact_moments(d), 6, 1, True)
                kp = kappa(G)
                dec = int(math.floor(math.log10(kp)))
                if dec not in found:
                    found[dec] = (kp, tag, k, s)
    return found


def conditioning_design(decade):
    """(design, p) of the conditioning sweep: kappa_2(G) in [10^decade, 10^(decade + 1))."""
    _, tag, k, s = _conditioning_designs()[decade]
    return int_design(41, 4000, 6, tag=tag, near=(0, 1, k), scale={2: s} if s else None), 6
