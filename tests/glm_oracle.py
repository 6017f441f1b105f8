"""CPU oracle for `GLM.fit`: a NumPy restatement of the reference's IRLS loop.

Test infrastructure only, like ``oracle/lin_reg_oracle.py`` (whose weighted least-squares solve it reuses): the package
never imports it.  It follows faer_irls (/root/reference/src/linear/glm/glm_solvers.rs:249-359) line by line, with
the link and variance functions of src/linear/glm/link_functions.rs:1-79 and the family table of
glm_solvers.rs:17-63.  ``GLM::fit_unchecked`` (glm_solvers.rs:196-216) appends the ones column before calling it, so
the caller passes X with the ones column already last when the model has a bias.

One deliberate deviation, shared with the device path: the logit inverse is the overflow-free sigmoid of
logistic_solver.rs:10-18 (the reference's exp(eta) / (1 + exp(eta)) is NaN above eta ~ 709).
"""
from __future__ import annotations

import numpy as np

from oracle.lin_reg_oracle import faer_weighted_lr


def _sigmoid(x):
    r = 1.0 / (1.0 + np.exp(-np.abs(x)))
    return np.where(x >= 0.0, r, 1.0 - r)


# family -> (g, g^-1, g', V)                                             link_functions.rs:13-79
_IDENTITY = (lambda m: m, lambda e: e, lambda m: np.ones_like(m))
_LOG = (np.log, np.exp, lambda m: 1.0 / m)
_LOGIT = (lambda m: np.log(m / (1.0 - m)), _sigmoid, lambda m: 1.0 / (m * (1.0 - m)))
_INVERSE = (lambda m: 1.0 / m, lambda e: 1.0 / e, lambda m: -((1.0 / m) * (1.0 / m)))
FAMILIES = {
    "gaussian": (*_IDENTITY, lambda m: np.ones_like(m)),
    "normal": (*_IDENTITY, lambda m: np.ones_like(m)),
    "poisson": (*_LOG, lambda m: m),
    "binomial": (*_LOGIT, lambda m: m * (1.0 - m)),
    "logistic": (*_LOGIT, lambda m: m * (1.0 - m)),
    "gamma": (*_INVERSE, lambda m: m * m),
}


def link_inverse(family: str, eta):
    """g^-1 (GeneralizedLinearModel::glm_predict, glm_solvers.rs:219-225)."""
    return FAMILIES[family][1](np.asarray(eta, dtype=np.float64))


def faer_irls(X, y, family: str, tol: float, max_iter: int):
    """(beta, n_iter).  beta has X.shape[1] entries (bias last when X carries the ones column)."""
    link, inv, deriv, variance = FAMILIES[family]
    X = np.asarray(X, dtype=np.float64)
    y = np.asarray(y, dtype=np.float64).reshape(-1)
    n = X.shape[0]
    beta = np.zeros(X.shape[1])                                          # :261
    with np.errstate(all="ignore"):
        if family in ("binomial", "logistic"):                           # :266-287
            mu = (y + 0.5) * 0.5
        else:
            mu = (y + y.sum() / n) * 0.5
        eta = link(mu)                                                   # :289
        n_iter = 0
        for _ in range(max_iter):                                        # :291
            n_iter += 1
            d = deriv(mu)                                                # :293-298
            w = 1.0 / (d * d * variance(mu))
            z = eta + d * (y - mu)                                       # :300-307
            xtw = X.T * w[None, :]
            # faer's col_piv_qr propagates a NaN or inf of X'WX / X'Wz into the solution; LAPACK is not asked to
            # factor a non-finite matrix here
            if np.isfinite(xtw @ X).all() and np.isfinite(xtw @ z).all():
                beta_new = faer_weighted_lr(X, z.reshape(-1, 1), w, "qr").reshape(-1)   # :310-315, lr_solvers.rs:386-409
            else:
                beta_new = np.full(X.shape[1], np.nan)
            eta = X @ beta_new                                           # :317-330
            mu = inv(eta)                                                # :332-335
            max_diff = 0.0                                               # :337-341: f64::max ignores NaN
            for b, bn in zip(beta, beta_new):
                v = abs(b - bn)
                if not np.isnan(v):
                    max_diff = max(max_diff, v)
            beta = beta_new
            if max_diff < tol:                                           # :344-349
                break
    return beta, n_iter


# The data of the reference's test_glm_family (tests/test_linear_models.py:191-253): RandomState(42), 500 x 4.
_LIFTED_Y = {
    "gaussian": lambda X, rng: X @ np.array([1.0, -0.5, 0.3, 0.8]) + rng.randn(X.shape[0]) * 0.1,
    "binomial": lambda X, rng: rng.binomial(1, 1.0 / (1.0 + np.exp(-(X @ np.array([1.0, -0.5, 0.3, 0.8]))))).astype(float),
    "poisson": lambda X, rng: rng.poisson(np.exp(np.clip(X @ np.array([0.5, -0.25, 0.15, 0.4]), -2.0, 2.0))).astype(float),
    "gamma": lambda X, rng: rng.gamma(shape=2.0,
                                      scale=np.exp(np.clip(X @ np.array([0.3, -0.15, 0.09, 0.24]), -2.0, 2.0)) / 2.0),
}
LIFTED_FAMILIES = tuple(_LIFTED_Y)
# iterations faer_irls takes on that data with a bias at tol 1e-8
LIFTED_ITERS = {"gaussian": 2, "binomial": 5, "poisson": 5, "gamma": 10}


def lifted_case(family: str):
    rng = np.random.RandomState(42)
    X = rng.randn(500, 4)
    return X, _LIFTED_Y[family](X, rng)
