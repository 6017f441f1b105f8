"""CPU oracle for `MixedModel.fit_df`: a NumPy restatement of the reference's REML fit.

Test infrastructure only, like ``tests/glm_oracle.py``: the package never imports it.  It follows fit_reml and profile
(/root/reference/src/linear/mixed/mod.rs:121-272) line by line: the Woodbury apply of H^-1 = (I + gamma Z Z')^-1
over group sums, the Cholesky of X'HiX, the golden-section search over gamma in [0, 1e6] and the containment degrees of
freedom from column-pivoted QR ranks of X[:, between] and the dense [X | Z].  `ranks="structure"` takes those ranks
from the design's structure instead (rank [X | Z] = non-empty groups + rank of X's within-group part), for sizes where
the dense [X | Z] cannot be formed.
"""
from __future__ import annotations

import numpy as np
import scipy.linalg as sla


class MixedFitError(ValueError):
    pass


def _apply_hi(v, codes, counts, gamma):
    gs = np.bincount(codes, weights=v, minlength=counts.size)
    scaled = gamma * gs / (1.0 + gamma * counts)
    return v - scaled[codes]


def profile(X, y, codes, counts, gamma):
    """(beta, resid_var, deviance) at gamma, or raises with the reference's message."""
    n, p = X.shape
    hix = np.column_stack([_apply_hi(X[:, j], codes, counts, gamma) for j in range(p)])
    hiy = _apply_hi(y, codes, counts, gamma)
    a = X.T @ hix
    b = X.T @ hiy
    try:
        L = np.linalg.cholesky(a)
    except np.linalg.LinAlgError:
        raise MixedFitError("X'HiX is not positive definite; design may be rank-deficient.")
    beta = sla.cho_solve((L, True), b)
    r = y - X @ beta
    resid_var = float(r @ _apply_hi(r, codes, counts, gamma)) / (n - p)
    if not resid_var > 0.0:
        raise MixedFitError("Residual variance estimate is non-positive.")
    slogdet = 2.0 * float(np.sum(np.log(np.abs(np.diag(L)))))
    deviance = (n - p) * np.log(resid_var) + float(np.sum(np.log(1.0 + gamma * counts))) + slogdet
    return beta, resid_var, deviance


def deviance(X, y, codes, n_groups, gamma):
    counts = np.bincount(codes, minlength=n_groups).astype(np.float64)
    return profile(X, y, codes, counts, gamma)[2]


def matrix_rank(A, tol=1e-9):
    """Leading |R_ii| > tol |R_00| of a column-pivoted QR (mod.rs matrix_rank)."""
    if A.shape[0] == 0 or A.shape[1] == 0:
        return 0
    R = sla.qr(A, mode="r", pivoting=True)[0]
    d = np.abs(np.diag(R))
    if d[0] == 0.0:
        return 0
    k = 0
    while k < d.size and d[k] > tol * d[0]:
        k += 1
    return k


def fit_reml(X, y, codes, n_groups, between_idx, max_iter=200, tol=1e-10, ranks="dense"):
    """dict(coeffs, std_errors, dfs, gamma, resid_variance, evals) as the reference's fit_reml."""
    X = np.asarray(X, dtype=np.float64)
    y = np.asarray(y, dtype=np.float64).ravel()
    codes = np.asarray(codes, dtype=np.int64).ravel()
    n, p = X.shape
    if n != y.size or n != codes.size:
        raise MixedFitError("X, y, and group must have the same number of rows.")
    if n <= p:
        raise MixedFitError("Not enough rows to fit a mixed model with this many fixed effects.")
    counts = np.bincount(codes, minlength=n_groups).astype(np.float64)
    evals = 0

    def dev(g):
        nonlocal evals
        evals += 1
        return profile(X, y, codes, counts, g)[2]

    phi = (np.sqrt(5.0) - 1.0) / 2.0
    lo, hi = 0.0, 1e6
    c = hi - phi * (hi - lo)
    e = lo + phi * (hi - lo)
    fc, fe = dev(c), dev(e)
    for _ in range(max_iter):
        if hi - lo < tol:
            break
        if fc < fe:
            hi, e, fe = e, c, fc
            c = hi - phi * (hi - lo)
            fc = dev(c)
        else:
            lo, c, fc = c, e, fe
            e = lo + phi * (hi - lo)
            fe = dev(e)
    gamma = (lo + hi) / 2.0
    beta, resid_var, _ = profile(X, y, codes, counts, gamma)
    evals += 1
    hix = np.column_stack([_apply_hi(X[:, j], codes, counts, gamma) for j in range(p)])
    L = np.linalg.cholesky(X.T @ hix)
    cov = sla.cho_solve((L, True), np.eye(p))
    std_errors = np.sqrt(resid_var * np.diag(cov))

    between = sorted(set(int(j) for j in between_idx))
    if ranks == "dense":
        rank_between = matrix_rank(X[:, between])
        Zd = np.zeros((n, n_groups))
        Zd[np.arange(n), codes] = 1.0
        rank_combined = matrix_rank(np.column_stack([X, Zd]))
    else:
        rank_between = matrix_rank(X[:, between])
        means = np.column_stack([np.bincount(codes, weights=X[:, j], minlength=n_groups) for j in range(p)])
        nz = counts > 0
        means[nz] /= counts[nz, None]
        within = X - means[codes]
        rank_combined = int(nz.sum()) + matrix_rank(within)
    dfs = np.array([n_groups - rank_between if j in between else n - rank_combined for j in range(p)], dtype=np.float64)
    return {"coeffs": beta, "std_errors": std_errors, "dfs": dfs, "gamma": gamma, "resid_variance": resid_var,
            "evals": evals}


def lifted_case():
    """The data of the reference's test_mixed_model_recovers_fixed_effect (tests/test_linear_models.py:274-311)."""
    rng = np.random.RandomState(42)
    n_groups, per_group = 40, 25
    n = n_groups * per_group
    group = np.repeat(np.arange(n_groups), per_group)
    u = rng.normal(0.0, 1.0, n_groups)[group]
    x = rng.normal(0.0, 1.0, n)
    noise_col = rng.normal(0.0, 1.0, n)
    e = rng.normal(0.0, 0.5, n)
    y = 1.5 + 2.0 * x + u + e
    return {"y": y, "x": x, "noise": noise_col, "group": group}
