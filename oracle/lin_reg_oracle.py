"""CPU oracle for the polars_ds linear-regression expression family.

TEST INFRASTRUCTURE ONLY.  Nothing under ``polars_ds_extension_b200/`` may import this
module; only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s CPU-baseline /
``--impl reference`` legs use it, and only as the checker / the timed CPU arm.

What it is: a NumPy/SciPy restatement ("port") of the reference's algorithm for the
``lin_reg`` hot path, function by function, each citing the reference file:line it follows
(paths relative to /root/reference).  The reference is Rust on top of the un-vendored crate
``faer 0.23.2 @ git 8377404e78`` (Cargo.lock:701-703); it cannot be compiled in this image
(no cargo/rustc, no polars wheel), so the dense primitives faer provides are restated with
their LAPACK equivalents:

    faer matmul            -> numpy ``@``           (lr_solvers.rs:191,269)
    faer col_piv_qr        -> scipy.linalg.qr(pivoting=True)   (lr_solvers.rs:292,353)
    faer thin_svd          -> numpy.linalg.svd      (lr_solvers.rs:225,284,362)
    faer llt               -> numpy.linalg.cholesky (lr_solvers.rs:288,369)
    student_t_sf / _ppf    -> scipy.stats.t.sf / .ppf  (stats_utils/beta.rs:24-37,365-377)

Parity pin: the reference ships no golden files for this path; its own tests pin it against
scikit-learn / numpy.linalg.lstsq / closed-form identities on seeded or literal data
(tests/test_linear_exprs.py, tests/test_many.py:1636-1726).  ``tests/test_oracle_golden.py``
re-runs every reproducible one of those known-answer tests against THIS module with the same
seeds, literals and tolerances, so the oracle is pinned at exactly the boundary the reference's
test-suite pins the reference.  It is not bit-pinned against the Rust binary (which cannot be
built here); DESIGN.md says so.

dtype: every function takes ``dt`` (np.float64 or np.float32) and computes in that dtype, as the
reference's generic ``T: RealField + Float`` code does for the ``_f32`` symbols.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from fractions import Fraction
from typing import List, Optional, Sequence, Tuple

import numpy as np
import scipy.linalg as sla
from scipy import stats as _st

PARALLEL_MATMUL_THRESHOLD = 4096  # src/utils/parallelism.rs:36-42 (no numeric effect)


# --------------------------------------------------------------------------------------
# Input model: a nullable, named column (what a polars Series carries over the plugin ABI)
# --------------------------------------------------------------------------------------
@dataclass
class Col:
    name: str
    values: np.ndarray                    # any numeric dtype
    valid: Optional[np.ndarray] = None    # bool mask, True = not null; None = no nulls

    def has_nulls(self) -> bool:
        return self.valid is not None and not bool(self.valid.all())

    def __len__(self) -> int:
        return len(self.values)


def col(name, values, valid=None) -> Col:
    """Build a Col; a python list containing None becomes a nullable column."""
    if isinstance(values, (list, tuple)) and any(v is None for v in values):
        valid = np.array([v is not None for v in values], dtype=bool)
        values = np.array([0.0 if v is None else v for v in values], dtype=np.float64)
    return Col(name, np.asarray(values), None if valid is None else np.asarray(valid, dtype=bool))


class OracleError(Exception):
    """Mirrors PolarsError::ComputeError strings of the reference."""


# --------------------------------------------------------------------------------------
# src/linear/mod.rs:34-66  NullPolicy + parser
# --------------------------------------------------------------------------------------
# The fill literal is kept exact (a Fraction; a float only for inf / nan): the reference parses it as NullPolicy<f64> for
# the f64 symbols and NullPolicy<f32> for the _f32 twins (`str::parse::<T>`, correctly rounded once to T), so it is
# rounded to the compute dtype only where the frame is built (fill_value).
def parse_null_policy(value: str) -> Tuple[str, Optional[object]]:
    v = value.lower()
    if v == "raise":
        return ("raise", None)
    if v == "skip":
        return ("skip", None)
    if v == "zero":
        return ("fill", Fraction(0))
    if v == "one":
        return ("fill", Fraction(1))
    if v == "ignore":
        return ("ignore", None)
    if v == "skip_window":
        return ("skip_window", None)
    try:
        x = float(value)
    except ValueError:
        raise OracleError("Invalid NullPolicy.")
    try:
        return ("fill", Fraction(value))
    except ValueError:
        return ("fill", x)                 # inf / nan


def round_to_binary(x: Fraction, mant_bits: int, emin: int, emax: int) -> float:
    """x rounded once, to nearest with ties to even, to the binary format with `mant_bits` significand bits (implicit
    bit included) and normal exponents emin..emax; overflow gives +-inf.  Exact rational arithmetic throughout."""
    if x == 0:
        return 0.0
    sign, a = (-1 if x < 0 else 1), abs(x)
    e = a.numerator.bit_length() - a.denominator.bit_length()      # 2^(e-1) < a < 2^(e+1)
    if a >= Fraction(2) ** (e + 1):
        e += 1
    elif a < Fraction(2) ** e:
        e -= 1
    q = Fraction(2) ** (max(e, emin) - (mant_bits - 1))              # the spacing of the format around a
    m = round(a / q)                                                 # Fraction.__round__: half to even
    r = m * q
    if r >= Fraction(2) ** (emax + 1):
        return sign * math.inf
    return sign * float(r)                                           # exact: r has <= mant_bits significant bits


def fill_value(fill, dt):
    """The parsed fill literal as the reference's NullPolicy<T> holds it: rounded once to dt."""
    if not isinstance(fill, Fraction):
        return dt(fill)
    if np.dtype(dt) == np.float32:
        return np.float32(round_to_binary(fill, 24, -126, 127))
    return np.float64(round_to_binary(fill, 53, -1022, 1023))


# --------------------------------------------------------------------------------------
# src/utils/mod.rs:101-206  series_to_slice_inner: cast to T, null -> NaN
# --------------------------------------------------------------------------------------
def _to_dt(c: Col, dt) -> np.ndarray:
    v = c.values.astype(dt, copy=True)
    if c.valid is not None:
        v[~c.valid] = np.nan
    return v


# A feature under FILL / FILL_WINDOW: `cast(Float64).fill_null(lit(x))` with the f64 literal in the f64 symbols
# (linear_regression.rs:211-213, :232-234, :320-322), `cast(Float32).fill_null(lit(x))` with the f32 literal in the _f32
# twins (linear_regression_f32.rs:148-152, :169-173, :256-258).  Both cast straight to dt: every value rounds once.
def _cast_fill(c: Col, fill, dt) -> np.ndarray:
    v = c.values.astype(dt)
    if c.valid is not None:
        v[~c.valid] = fill_value(fill, dt)
    return v


# --------------------------------------------------------------------------------------
# src/num_ext/linear_regression.rs:151-267  series_to_mat_for_lr
# returns (y [n], X [n, q] with physical ones column if add_bias, mask or None)
# mask None  <=> the reference's `[true]` dummy (no rows dropped / no nulls)
# mask "has" <=> the `[false]` dummy of IGNORE / SKIP_WINDOW (nulls present, nothing dropped)
# --------------------------------------------------------------------------------------
def series_to_mat_for_lr(inputs: Sequence[Col], add_bias: bool, policy, dt):
    ncols = len(inputs) - 1
    n_features = ncols + int(add_bias)
    y_has_null = inputs[0].has_nulls()
    has_null = y_has_null or any(c.has_nulls() for c in inputs[1:])
    nrows0 = len(inputs[0])

    def finish(cols_dt: List[np.ndarray], mask):
        n = len(cols_dt[0])
        if n < n_features:
            raise OracleError("#Data < #features. No conclusive result.")
        y = cols_dt[0]
        X = np.empty((n, n_features), dtype=dt, order="F")
        for j, c in enumerate(cols_dt[1:]):
            X[:, j] = c
        if add_bias:
            X[:, -1] = dt(1.0)
        return y, X, mask

    if not has_null:  # :164-185 fast path
        if nrows0 == 0:
            raise OracleError("Empty data")
        return finish([c.values.astype(dt) for c in inputs], None)

    if nrows0 == 0:
        raise OracleError("Empty data")
    kind, fill = policy
    if kind in ("ignore", "skip_window"):      # :194-197
        return finish([_to_dt(c, dt) for c in inputs], "has")
    if kind == "raise":                        # :198
        raise OracleError("Nulls found in data")
    if kind == "skip":                         # :199-206
        mask = np.ones(nrows0, dtype=bool)
        for c in inputs:
            if c.valid is not None:
                mask &= c.valid
        return finish([c.values.astype(dt)[mask] for c in inputs], mask)
    if kind in ("fill", "fill_window"):        # :207-247
        filled = [_to_dt(inputs[0], dt)]
        for c in inputs[1:]:
            filled.append(_cast_fill(c, fill, dt))
        if y_has_null:
            if kind == "fill":
                m = inputs[0].valid.copy()
                return finish([v[m] for v in filled], m)
            return finish(filled, "has")       # FILL_WINDOW keeps y's nulls (NaN) (:240-242)
        return finish(filled, None)
    raise OracleError("Invalid NullPolicy.")


# src/num_ext/linear_regression.rs:270-349  series_to_mat_for_multi_lr
def series_to_mat_for_multi_lr(inputs: Sequence[Col], last_target_idx: int, add_bias: bool, policy, dt):
    y_has_null = any(c.has_nulls() for c in inputs[:last_target_idx])
    n_features = len(inputs) + int(add_bias) - last_target_idx
    has_null = y_has_null or any(c.has_nulls() for c in inputs[last_target_idx:])
    n = len(inputs[0])
    if n == 0:
        raise OracleError("Empty data")
    if has_null:
        kind, fill = policy
        if kind == "raise":
            raise OracleError("Nulls found in data")
        if kind != "fill":
            raise OracleError("The null policy is not supported by multi-target linear regression.")
        if y_has_null:
            raise OracleError(
                "Filling null doesn't work for multi-target lstsq when there are nulls in any of the targets."
            )
        cols = [c.values.astype(dt) for c in inputs[:last_target_idx]]
        for c in inputs[last_target_idx:]:
            cols.append(_cast_fill(c, fill, dt))
    else:
        cols = [c.values.astype(dt) for c in inputs]
    Y = np.column_stack(cols[:last_target_idx]).astype(dt)
    X = np.empty((n, n_features), dtype=dt, order="F")
    for j, c in enumerate(cols[last_target_idx:]):
        X[:, j] = c
    if add_bias:
        X[:, -1] = dt(1.0)
    return Y, X


# --------------------------------------------------------------------------------------
# src/linear/lr/lr_solvers.rs
# --------------------------------------------------------------------------------------
def get_xtx_with_lambda(X, lam, add_bias):           # :183-211
    xtx = X.T @ X
    n1 = X.shape[1] - int(add_bias)
    if lam > 0 and n1 >= 1:
        idx = np.arange(n1)
        xtx[idx, idx] += X.dtype.type(lam)
    return xtx


def build_xty(X, Y):                                  # :262-278
    return X.T @ Y


def _qr_piv(A):
    Q, R, P = sla.qr(A, pivoting=True, check_finite=False)
    return Q, R, P


def _qr_solve(qrp, B):
    Q, R, P = qrp
    z = sla.solve_triangular(R, Q.T @ B, lower=False, check_finite=False)
    out = np.empty_like(z)
    out[P] = z
    return out


def _solver_kind(s: str) -> str:                      # lr/mod.rs:18-27
    return {"qr": "qr", "svd": "svd", "choleskey": "choleskey"}.get(s, "qr")


def solve_xtx_xty(xtx, xty, how):                     # :282-294
    how = _solver_kind(how)
    if how == "svd":
        try:
            U, S, Vt = np.linalg.svd(xtx)
            return (Vt.T * (1.0 / S).astype(xtx.dtype)) @ (U.T @ xty)
        except np.linalg.LinAlgError:
            pass
    elif how == "choleskey":
        try:
            L = np.linalg.cholesky(xtx)
            return sla.cho_solve((L, True), xty, check_finite=False).astype(xtx.dtype)
        except np.linalg.LinAlgError:
            pass
    return _qr_solve(_qr_piv(xtx), xty)


def faer_solve_lr(X, Y, lam, add_bias, how):          # :299-308
    return solve_xtx_xty(get_xtx_with_lambda(X, lam, add_bias), build_xty(X, Y), how)


def faer_solve_lr_gated(X, Y, lam, add_bias, how, tol):   # :329-382
    dt = X.dtype.type
    xtx = get_xtx_with_lambda(X, lam, add_bias)
    d = np.diag(xtx)
    if np.any(~(d > 0)):
        return None
    ln_den = dt(np.sum(np.log(d), dtype=dt))
    ln_tol = dt(np.log(dt(tol)))
    how = _solver_kind(how)
    with np.errstate(divide="ignore"):
        if how == "qr":
            qrp = _qr_piv(xtx)
            ln_det = dt(np.sum(np.log(np.abs(np.diag(qrp[1]))), dtype=dt))
            if ln_det - ln_den <= ln_tol:
                return None
            return _qr_solve(qrp, build_xty(X, Y))
        if how == "svd":
            try:
                U, S, Vt = np.linalg.svd(xtx)
            except np.linalg.LinAlgError:
                return None
            ln_det = dt(np.sum(np.log(S), dtype=dt))
            if ln_det - ln_den <= ln_tol:
                return None
            return (Vt.T * (1.0 / S).astype(xtx.dtype)) @ (U.T @ build_xty(X, Y))
        try:
            L = np.linalg.cholesky(xtx)
        except np.linalg.LinAlgError:
            return None
        s = dt(np.sum(np.log(np.diag(L)), dtype=dt))
        if (s + s) - ln_den <= ln_tol:
            return None
        return sla.cho_solve((L, True), build_xty(X, Y), check_finite=False).astype(xtx.dtype)


def faer_solve_lr_rcond(X, Y, lam, add_bias, rcond):   # :216-258
    dt = X.dtype.type
    xtx = get_xtx_with_lambda(X, lam, add_bias)
    U, S, Vt = np.linalg.svd(xtx)
    singular_values = np.sqrt(S)
    threshold = dt(rcond) * singular_values[0]
    # NOTE (reference quirk, :232-240): the threshold is rcond * sqrt(S_max) but it is compared
    # against S (the eigenvalues of X'X), not against sqrt(S).
    sinv = np.where(S >= threshold, 1.0 / S, 0.0).astype(xtx.dtype)
    z = (U.T @ build_xty(X, Y)) * sinv[:, None]
    return Vt.T @ z, singular_values


def faer_weighted_lr(X, Y, w, how):                   # :386-409
    xtw = X.T * w[None, :]
    xtwx = xtw @ X
    return solve_xtx_xty(xtwx, xtw @ Y, how)


def soft_threshold_l1(z, lam):                        # :412-414
    return np.sign(z) * max(abs(z) - lam, 0.0)


def faer_coordinate_descent(X, Y, l1_reg, l2_reg, add_bias, tol, max_iter, positive):  # :426-538
    dt = X.dtype.type
    m = dt(X.shape[0])
    ncols = X.shape[1]
    n1 = ncols - int(add_bias)
    lambda_l1 = m * dt(l1_reg)
    beta = np.zeros(ncols, dtype=dt)
    xty = (X.T @ Y[:, :1])[:, 0]
    xtx = X.T @ X
    norms = np.diag(xtx) + m * dt(l2_reg)
    y_sum = dt(Y[:, 0].sum(dtype=dt))
    col_sums = X[:, :n1].sum(axis=0, dtype=dt)
    tol = dt(tol)
    for _ in range(int(max_iter)):
        max_change = dt(0)
        for j in range(n1):
            before = beta[j]
            beta[j] = 0
            dot = dt(np.dot(xtx[:, j], beta))
            main_update = xty[j] - dot
            if positive and main_update < 0:
                after = dt(0)
            else:
                after = dt(soft_threshold_l1(main_update, lambda_l1) / norms[j])
            beta[j] = after
            max_change = max(abs(after - before), max_change)
        if add_bias:
            dot_sums = dt(np.dot(beta[:n1], col_sums))
            beta[n1] = (y_sum - dot_sums) / m
        if max_change < tol:
            break
    return beta.reshape(-1, 1)


def faer_nn_lr(X, Y, add_bias, tol, max_iter):        # :542-600
    dt = X.dtype.type
    xtx = X.T @ X
    ncols = X.shape[1]
    beta = np.zeros(ncols, dtype=dt)
    mu = -(X.T @ Y[:, :1])[:, 0]
    tol = dt(tol)
    for _ in range(int(max_iter)):
        c1 = bool(np.all(mu >= -tol))
        c2 = bool(np.all(mu[beta > 0] <= tol))
        if c1 and c2:
            break
        for k in range(ncols):
            beta_k = beta[k]
            update = beta_k - mu[k] / xtx[k, k]
            if (not add_bias) or k < ncols - 1:
                update = max(update, dt(0))
            beta[k] = update
            mu = mu + (update - beta_k) * xtx[:, k]
    return beta.reshape(-1, 1)


def lr_methods(l1, l2) -> str:                        # lr/mod.rs:51-63
    if l1 > 0 and l2 <= 0:
        return "l1"
    if l1 <= 0 and l2 > 0:
        return "l2"
    if l1 > 0 and l2 > 0:
        return "elastic"
    return "normal"


# --------------------------------------------------------------------------------------
# src/linear/online_lr/lr_online_solvers.rs
# --------------------------------------------------------------------------------------
def faer_qr_lr_with_inv(X, Y, lam, add_bias):         # :120-143
    n1 = X.shape[1] - int(add_bias)
    xtx = X.T @ X
    if lam > 0 and n1 >= 1:
        idx = np.arange(n1)
        xtx[idx, idx] += X.dtype.type(lam)
    qrp = _qr_piv(xtx)
    inv = _qr_solve(qrp, np.eye(xtx.shape[0], dtype=xtx.dtype))
    w = _qr_solve(qrp, X.T @ Y)
    return inv, w


def woodbury_step(inv, w, new_x, new_y, c):           # :307-332  (in place)
    u = inv @ new_x.T                  # q x 1
    z = 1.0 / (c + (new_x @ u)[0, 0])
    inv -= z * (u @ u.T)
    y_diff = new_y - new_x @ w
    w += z * (u @ y_diff)


def _finite_row(x, y):
    return bool(np.isfinite(x).all() and np.isfinite(y).all())


def faer_recursive_lr(X, Y, n, lam):                  # :148-175
    dt = X.dtype.type
    inv, w = faer_qr_lr_with_inv(X[:n], Y[:n], dt(lam), False)
    out = [w.copy()]
    for j in range(n, X.shape[0]):
        nx, ny = X[j:j + 1], Y[j:j + 1]
        if _finite_row(nx, ny):                        # OnlineLR::update :85-89
            woodbury_step(inv, w, nx, ny, dt(1))
        out.append(w.copy())
    return out


def faer_rolling_lr(X, Y, n, lam):                    # :180-212
    dt = X.dtype.type
    inv, w = faer_qr_lr_with_inv(X[:n], Y[:n], dt(lam), False)
    out = [w.copy()]
    for j in range(n, X.shape[0]):
        rx, ry = X[j - n:j - n + 1], Y[j - n:j - n + 1]
        if _finite_row(rx, ry):
            woodbury_step(inv, w, rx, ry, dt(-1))
        nx, ny = X[j:j + 1], Y[j:j + 1]
        if _finite_row(nx, ny):
            woodbury_step(inv, w, nx, ny, dt(1))
        out.append(w.copy())
    return out


def faer_rolling_skipping_lr(X, Y, n, m, lam):        # :218-301
    dt = X.dtype.type
    xn = X.shape[0]
    out: List[Optional[np.ndarray]] = []
    is_finite = np.isfinite(X).all(axis=1) & np.isfinite(Y).all(axis=1)
    left, right = 0, n
    cnt = 0
    inv = w = None
    while right <= xn:
        sel = is_finite[left:right]
        cnt = int(sel.sum())
        if cnt >= m:
            inv, w = faer_qr_lr_with_inv(X[left:right][sel], Y[left:right][sel], dt(lam), False)
            out.append(w.copy())
            break
        left += 1
        right += 1
        out.append(None)
    if right >= xn:
        return out
    for j in range(right, xn):
        if is_finite[j - n]:
            cnt -= 1
            woodbury_step(inv, w, X[j - n:j - n + 1], Y[j - n:j - n + 1], dt(-1))
        if is_finite[j]:
            cnt += 1
            woodbury_step(inv, w, X[j:j + 1], Y[j:j + 1], dt(1))
        out.append(w.copy() if cnt >= m else None)
    return out


# --------------------------------------------------------------------------------------
# Plugin entry points.  kwargs are the dicts expr_linear.py builds (:237-248, :208-215, :467-473,
# :546-552, :599-607).  ``f32=True`` selects the `_f32` twin and its quirks.
# Outputs:  coefficients -> np.ndarray [q] or None (null list);  row outputs -> (values, valid).
# --------------------------------------------------------------------------------------
def _dt(f32):
    return np.float32 if f32 else np.float64


def _fit_single(inputs, kw, f32, y, X):
    """Dispatch of pl_lr / pl_lr_pred (linear_regression.rs:436-498, 719-780).  Returns beta [q,1] or None."""
    dt = _dt(f32)
    add_bias = kw["bias"]
    solver = kw.get("solver", "qr")
    Y = y.reshape(-1, 1)
    if kw.get("weighted", False):
        w = inputs[0].values.astype(dt)
        if len(w) != X.shape[0]:
            raise OracleError("Shape of weights is not the same as the data.")
        return faer_weighted_lr(X, Y, w, solver)
    l1, l2 = kw.get("l1_reg", 0.0), kw.get("l2_reg", 0.0)
    method = lr_methods(l1, l2)
    positive = kw.get("positive", False)
    # f32 twin hard-codes iteration counts (linear_regression_f32.rs:343,351,362,620,629,640)
    max_iter = kw.get("max_iter", 0)
    if method in ("normal", "l2") and not positive:
        tol = kw.get("singular_x_tol", 0.0)
        if tol > 0.0:
            return faer_solve_lr_gated(X, Y, dt(l2), add_bias, solver, dt(tol))
        return faer_solve_lr(X, Y, dt(l2), add_bias, solver)
    if method == "normal" and positive:
        it = kw.get("_nn_iter_f32", 200) if f32 else max_iter
        return faer_nn_lr(X, Y, add_bias, kw["tol"], it)
    it = 2000 if f32 else max_iter
    if method == "l2" and positive:
        return faer_coordinate_descent(X, Y, 0.0, l2, add_bias, kw["tol"], it, True)
    return faer_coordinate_descent(X, Y, l1, l2, add_bias, kw["tol"], it, positive)


def pl_lr(inputs: Sequence[Col], kw: dict, f32: bool = False):
    """linear_regression.rs:419-513.  -> coeffs [q] or None."""
    dt = _dt(f32)
    policy = parse_null_policy(kw["null_policy"])
    data = inputs[1:] if kw.get("weighted", False) else inputs
    y, X, _ = series_to_mat_for_lr(data, kw["bias"], policy, dt)
    beta = _fit_single(inputs, kw, f32, y, X)
    return None if beta is None else beta[:, 0].astype(dt)


def pl_lr_pred(inputs: Sequence[Col], kw: dict, f32: bool = False):
    """linear_regression.rs:704-820.  -> dict(pred=(vals, valid), resid=(vals, valid))."""
    dt = _dt(f32)
    policy = parse_null_policy(kw["null_policy"])
    data = inputs[1:] if kw.get("weighted", False) else inputs
    y, X, mask = series_to_mat_for_lr(data, kw["bias"], policy, dt)
    kw2 = dict(kw)
    kw2["_nn_iter_f32"] = 2000          # _f32.rs:620 (pred variant uses 2000, coeff variant 200)
    beta = _fit_single(inputs, kw2, f32, y, X)
    real_mask = isinstance(mask, np.ndarray) and (~mask).any()
    out_len = len(mask) if real_mask else X.shape[0]
    if beta is None:
        z = np.zeros(out_len, dtype=dt)
        v = np.zeros(out_len, dtype=bool)
        return {"pred": (z, v), "resid": (z.copy(), v.copy())}
    pred = (X @ beta)[:, 0]
    resid = y - pred
    if real_mask:
        p = np.zeros(out_len, dtype=dt)
        r = np.zeros(out_len, dtype=dt)
        p[mask] = pred
        r[mask] = resid
        return {"pred": (p, mask.copy()), "resid": (r, mask.copy())}
    ones = np.ones(out_len, dtype=bool)
    return {"pred": (pred.astype(dt), ones), "resid": (resid.astype(dt), ones.copy())}


def _fit_multi(inputs, kw, f32):
    dt = _dt(f32)
    policy = parse_null_policy(kw["null_policy"])
    lt = kw["last_target_idx"]
    Y, X = series_to_mat_for_multi_lr(inputs, lt, kw["bias"], policy, dt)
    l2 = kw.get("l2_reg", 0.0)
    tol = kw.get("singular_x_tol", 0.0)
    if tol > 0.0:
        beta = faer_solve_lr_gated(X, Y, dt(l2), kw["bias"], kw.get("solver", "qr"), dt(tol))
    else:
        beta = faer_solve_lr(X, Y, dt(l2), kw["bias"], kw.get("solver", "qr"))
    return Y, X, beta


def pl_lr_multi(inputs, kw, f32=False):
    """linear_regression.rs:517-584.  -> {target_name: coeffs or None}."""
    names = [c.name for c in inputs[: kw["last_target_idx"]]]
    _, _, beta = _fit_multi(inputs, kw, f32)
    if beta is None:
        return {nm: None for nm in names}
    return {nm: beta[:, i].astype(_dt(f32)) for i, nm in enumerate(names)}


def pl_lr_multi_pred(inputs, kw, f32=False):
    """linear_regression.rs:587-649 (f64 semantics; the f32 twin mis-slices y, _f32.rs:471-472 — not replicated)."""
    dt = _dt(f32)
    names = [c.name for c in inputs[: kw["last_target_idx"]]]
    Y, X, beta = _fit_multi(inputs, kw, f32)
    n = X.shape[0]
    out = {}
    if beta is None:
        for nm in names:
            out[f"{nm}_pred"] = (np.zeros(n, dt), np.zeros(n, bool))
            out[f"{nm}_resid"] = (np.zeros(n, dt), np.zeros(n, bool))
        return out
    pred = X @ beta
    resid = Y - pred
    for i, nm in enumerate(names):
        out[f"{nm}_pred"] = (pred[:, i].astype(dt), np.ones(n, bool))
        out[f"{nm}_resid"] = (resid[:, i].astype(dt), np.ones(n, bool))
    return out


def pl_lr_w_rcond(inputs, kw, f32=False):
    """linear_regression.rs:651-702.  -> dict(coeffs, singular_values)."""
    dt = _dt(f32)
    policy = parse_null_policy(kw["null_policy"])
    y, X, _ = series_to_mat_for_lr(inputs, kw["bias"], policy, dt)
    n, q = X.shape
    rcond = max(dt(kw["tol"]), np.finfo(dt).eps * dt(max(n, q)))
    beta, sv = faer_solve_lr_rcond(X, y.reshape(-1, 1), dt(kw.get("l2_reg", 0.0)), kw["bias"], rcond)
    return {"coeffs": beta[:, 0].astype(dt), "singular_values": sv.astype(dt)}


def _se_name(se: str) -> str:                         # linear_regression.rs:122-144
    return {"hc0": "hc0_se", "hc1": "hc1_se", "hc2": "hc2_se", "hc3": "hc3_se"}.get(se, "std_err")


def _report_tail(betas, std_err, dof, dt):
    with np.errstate(divide="ignore", invalid="ignore"):
        t_values = betas / std_err
    # p-values / t quantile are computed in f64 even for the f32 twin (_f32.rs:786-793)
    p_values = 2.0 * _st.t.sf(np.abs(t_values.astype(np.float64)), float(dof))
    t_alpha = _st.t.ppf(0.975, float(dof))
    lo = betas - dt(t_alpha) * std_err
    hi = betas + dt(t_alpha) * std_err
    return t_values.astype(dt), p_values.astype(dt), lo.astype(dt), hi.astype(dt)


def pl_lin_reg_report(inputs, kw, f32=False):
    """linear_regression.rs:822-980.  inputs[0] = var(y) (len 1), inputs[1] = y, rest features."""
    dt = _dt(f32)
    add_bias = kw["bias"]
    se_type = kw.get("std_err", "se")
    policy = parse_null_policy(kw["null_policy"])
    yv = inputs[0]
    y_var = dt(yv.values[0]) if len(yv) > 0 and (yv.valid is None or yv.valid[0]) else dt(np.nan)
    names = [c.name for c in inputs[2:]] + (["__bias__"] if add_bias else [])
    y, X, _ = series_to_mat_for_lr(inputs[1:], add_bias, policy, dt)
    n, q = X.shape
    xtx = X.T @ X
    xtx_inv = _qr_solve(_qr_piv(xtx), np.eye(q, dtype=dt))
    xtx_inv_xt = xtx_inv @ X.T
    coeffs = xtx_inv_xt @ y.reshape(-1, 1)
    betas = coeffs[:, 0]
    dof = dt(n) - dt(q)
    res = y - (X @ coeffs)[:, 0]
    ratio = dt(np.dot(res, res)) / (y_var * dt(n))     # quirk: ddof=1 variance times n (:867)
    r2 = dt(1.0) - ratio
    adj_r2 = dt(1.0) - ratio * (dt(n - 1) / (dof - dt(1.0)))
    if se_type in ("hc0", "hc1"):
        var_hc = (xtx_inv_xt * (res * res)[None, :]) @ xtx_inv_xt.T
        factor = dt(n) / dt(n - q) if se_type == "hc1" else dt(1.0)
        std_err = np.sqrt(np.diag(var_hc) * factor)
    elif se_type in ("hc2", "hc3"):
        h = np.einsum("ij,ji->i", X, xtx_inv_xt).astype(dt)
        sc = 1.0 / (1.0 - h) ** 2 if se_type == "hc3" else 1.0 / (1.0 - h)
        var_hc = (xtx_inv_xt * (res * res * sc)[None, :]) @ xtx_inv_xt.T
        std_err = np.sqrt(np.diag(var_hc))
    else:
        mse = dt(np.dot(res, res)) / dof
        std_err = np.sqrt(mse * np.diag(xtx_inv))
    std_err = std_err.astype(dt)
    t, p, lo, hi = _report_tail(betas.astype(dt), std_err, dof, dt)
    return {
        "features": names, "beta": betas.astype(dt), _se_name(se_type): std_err, "t": t, "p>|t|": p,
        "0.025": lo, "0.975": hi, "r2": dt(r2), "adj_r2": dt(adj_r2),
    }


def pl_wls_report(inputs, kw, f32=False):
    """linear_regression.rs:982-1117.  inputs = [weights, var(y), y, features...]."""
    dt = _dt(f32)
    add_bias = kw["bias"]
    policy = parse_null_policy(kw["null_policy"])
    w = inputs[0].values.astype(dt)
    yv = inputs[1]
    y_var = dt(yv.values[0]) if len(yv) > 0 and (yv.valid is None or yv.valid[0]) else dt(np.nan)
    names = [c.name for c in inputs[3:]] + (["__bias__"] if add_bias else [])
    y, X, _ = series_to_mat_for_lr(inputs[2:], add_bias, policy, dt)
    n, q = X.shape
    xtw = X.T * w[None, :]
    xtwx = xtw @ X
    xtwy = xtw @ y.reshape(-1, 1)
    qrp = _qr_piv(xtwx)
    inv = _qr_solve(qrp, np.eye(q, dtype=dt))
    coeffs = _qr_solve(qrp, xtwy)
    betas = coeffs[:, 0]
    dof = dt(n) - dt(q)
    res = y - (X @ coeffs)[:, 0]
    mse = dt(np.sum(w * res * res, dtype=dt)) / dof
    ratio = dt(np.dot(res, res)) / (y_var * dt(n))
    r2 = dt(1.0) - ratio
    adj_r2 = dt(1.0) - ratio * (dt(n - 1) / (dof - dt(1.0)))
    std_err = np.sqrt(mse * np.diag(inv)).astype(dt)
    t, p, lo, hi = _report_tail(betas.astype(dt), std_err, dof, dt)
    return {
        "features": names, "beta": betas.astype(dt), "std_err": std_err, "t": t, "p>|t|": p,
        "0.025": lo, "0.975": hi, "r2": dt(r2), "adj_r2": dt(adj_r2),
    }


def pl_recursive_lr(inputs, kw, f32=False):
    """linear_regression.rs:1121-1204.  -> dict(coeffs=list[np.ndarray|None], pred=(vals, valid)).

    For the null branch the reference pairs coeffs[i] with x row i of the FILTERED matrix
    (:1162-1171); that is an off-by-(n-1) nobody tests.  The oracle follows the no-null branch
    semantics (pred_j = x_j . beta_j) for both, and DESIGN.md flags the difference.
    """
    dt = _dt(f32)
    n = kw["n"]
    policy = parse_null_policy(kw["null_policy"])
    y, X, mask = series_to_mat_for_lr(inputs, kw["bias"], policy, dt)
    coeffs = faer_recursive_lr(X, y.reshape(-1, 1), n, dt(kw["lambda"]))
    real_mask = isinstance(mask, np.ndarray) and (~mask).any()
    nrows_out = len(mask) if real_mask else X.shape[0]
    out_c: List[Optional[np.ndarray]] = [None] * nrows_out
    pred = np.zeros(nrows_out, dt)
    valid = np.zeros(nrows_out, bool)
    if real_mask:
        kept = np.flatnonzero(mask)                     # original row index of filtered row i
        for i, c in enumerate(coeffs):
            fi = n - 1 + i                              # filtered row this coefficient belongs to
            oi = kept[fi]
            out_c[oi] = c[:, 0].astype(dt)
            pred[oi] = (X[fi:fi + 1] @ c)[0, 0]
            valid[oi] = True
    else:
        m = n - 1
        for i, c in enumerate(coeffs):
            out_c[m + i] = c[:, 0].astype(dt)
            pred[m + i] = (X[m + i:m + i + 1] @ c)[0, 0]
            valid[m + i] = True
    return {"coeffs": out_c, "pred": (pred, valid)}


def pl_rolling_lr(inputs, kw, f32=False):
    """linear_regression.rs:1206-1283."""
    dt = _dt(f32)
    n = kw["n"]
    kind, fill = parse_null_policy(kw["null_policy"])
    if kind == "skip":
        kind = "skip_window"
    elif kind == "fill":
        kind = "fill_window"
    y, X, mask = series_to_mat_for_lr(inputs, kw["bias"], (kind, fill), dt)
    has = mask is not None                              # "has" dummy or a real mask with a False
    should_skip = kind in ("skip_window", "fill_window") and has
    Y = y.reshape(-1, 1)
    if should_skip:
        coeffs = faer_rolling_skipping_lr(X, Y, n, kw["min_size"], dt(kw["lambda"]))
    else:
        coeffs = faer_rolling_lr(X, Y, n, dt(kw["lambda"]))
    nrows = X.shape[0]
    out_c: List[Optional[np.ndarray]] = [None] * nrows
    pred = np.zeros(nrows, dt)
    valid = np.zeros(nrows, bool)
    m = n - 1
    for i, c in enumerate(coeffs):
        if c is None:
            continue
        out_c[m + i] = c[:, 0].astype(dt)
        pred[m + i] = (X[m + i:m + i + 1] @ c)[0, 0]
        valid[m + i] = True
    return {"coeffs": out_c, "pred": (pred, valid)}


# --------------------------------------------------------------------------------------
# Mathematical definitions used by the property tests (what the reference's own tests assert:
# rolling == per-window OLS, recursive == prefix OLS; tests/test_linear_exprs.py:123-166,718-854)
# --------------------------------------------------------------------------------------
def window_ols(X, y, lo, hi, lam=0.0, add_bias=False):
    """OLS / ridge on rows [lo, hi) of a design X that already holds the ones column when add_bias.

    For the online (rolling / recursive) family the reference constructs OnlineLR::new(lambda, false) on that
    matrix (lr_online_solvers.rs:163-165, 195-197), so lambda is added to EVERY diagonal entry including the bias
    one — unlike pl_lr, where the bias diagonal is exempt (lr_solvers.rs:200-209).  `add_bias` is therefore
    deliberately ignored here."""
    Xw = np.asarray(X[lo:hi], dtype=np.float64)
    G = Xw.T @ Xw
    n1 = Xw.shape[1]
    G[np.arange(n1), np.arange(n1)] += lam
    return np.linalg.solve(G, Xw.T @ np.asarray(y[lo:hi], dtype=np.float64))


# ---------------------------------------------------------------------------------------------------------------------
# logistic regression: src/num_ext/logistic_regression.rs:10-99, solver src/linear/logistic/logistic_solver.rs
# ---------------------------------------------------------------------------------------------------------------------
def stable_sigmoid(x):
    """logistic_solver.rs:10-18"""
    x = np.asarray(x, dtype=np.float64)
    r = 1.0 / (1.0 + np.exp(-np.abs(x)))
    return np.where(x >= 0.0, r, 1.0 - r)


def stable_log_loss(y, z):
    """logistic_solver.rs:22-25"""
    return np.maximum(z, 0.0) - y * z + np.log1p(np.exp(-np.abs(z)))


def faer_logistic_reg(X, y, add_bias: bool, l1_reg, l2_reg, tol: float, max_iters: int):
    """logistic_solver.rs:107-146: argmin's L-BFGS (history 10, More-Thuente line search; OWL-QN when l1 > 0) on
    cost(w) = mean stable_log_loss(y, X w) + l2 / 2 |w_features|^2 (:42-74), gradient X'(sigmoid(Xw) - y) / m + l2 w
    (:80-103), from N(0, 0.01) draws of StdRng(42) (:121-124), gradient tolerance max(sqrt(eps), tol) (:127).
    argmin (Cargo.lock: argmin 0.10) is not vendored; the cost is convex, so its minimiser is restated through SciPy's
    L-BFGS-B on the same cost / gradient from a zero start, to a gradient tolerance below the reference's.  With l1 the
    non-smooth term is handled by a proximal-Newton loop (coordinate descent on the quadratic model), the optimum OWL-QN
    converges to.  X already holds the ones column when add_bias (logistic_regression.rs:27-31)."""
    from scipy.optimize import minimize

    X = np.asarray(X, dtype=np.float64)
    y = np.asarray(y, dtype=np.float64)
    m, q = X.shape
    nfeat = q - int(add_bias)
    l2 = l2_reg if (l2_reg is not None and l2_reg > 0.0) else 0.0
    l1 = max(l1_reg, np.finfo(np.float64).eps) if (l1_reg is not None and l1_reg > 0.0) else 0.0
    gtol = max(np.sqrt(np.finfo(np.float64).eps), tol)

    def cost(w):
        z = X @ w
        return stable_log_loss(y, z).sum() / m + 0.5 * l2 * float(w[:nfeat] @ w[:nfeat])

    def grad(w):
        g = X.T @ (stable_sigmoid(X @ w) - y) / m
        g[:nfeat] += l2 * w[:nfeat]
        return g

    if l1 == 0.0:
        res = minimize(cost, np.zeros(q), jac=grad, method="L-BFGS-B",
                       options={"maxiter": max(int(max_iters), 1) * 10, "gtol": min(gtol, 1e-9) * 1e-2, "ftol": 1e-16, "maxcor": 10})
        w = res.x
        for _ in range(50):                 # polish with Newton steps: the oracle is the exact minimiser
            mu = stable_sigmoid(X @ w)
            H = (X * (mu * (1.0 - mu))[:, None]).T @ X / m
            H[:nfeat, :nfeat] += l2 * np.eye(nfeat)
            g = grad(w)
            if np.linalg.norm(g) < 1e-13:
                break
            w = w - np.linalg.solve(H, g)
        return w
    # proximal Newton with coordinate descent on the l1-penalised quadratic model
    w = np.zeros(q)
    for _ in range(200):
        z = X @ w
        mu = stable_sigmoid(z)
        wt = np.maximum(mu * (1.0 - mu), 1e-12)
        zz = z + (y - mu) / wt
        A = (X * wt[:, None]).T @ X / m
        b = X.T @ (wt * zz) / m
        w_new = w.copy()
        for _cd in range(5000):
            dmax = 0.0
            for j in range(q):
                r = b[j] - A[j] @ w_new + A[j, j] * w_new[j]
                if j < nfeat:
                    v = np.sign(r) * max(abs(r) - l1, 0.0) / (A[j, j] + l2)
                else:
                    v = r / A[j, j]
                dmax = max(dmax, abs(v - w_new[j]))
                w_new[j] = v
            if dmax < 1e-14:
                break
        done = np.max(np.abs(w_new - w)) < 1e-12
        w = w_new
        if done:
            break
    return w


def pl_logistic_coeffs(inputs: Sequence[Col], kw: dict, f32: bool = False):
    """logistic_regression.rs:10-48 -> coeffs [q] (float64, bias last)."""
    policy = parse_null_policy(kw["null_policy"])
    y, X, _ = series_to_mat_for_lr(inputs, kw["bias"], policy, np.float64)
    return faer_logistic_reg(X, y, kw["bias"], kw.get("l1_reg", 0.0), kw.get("l2_reg", 0.0), kw.get("tol", 1e-5), kw.get("max_iter", 200))


def pl_logistic_pred(inputs: Sequence[Col], kw: dict, f32: bool = False):
    """logistic_regression.rs:50-99 -> (probabilities, valid): nulls re-inserted where the null policy dropped the row."""
    policy = parse_null_policy(kw["null_policy"])
    y, X, mask = series_to_mat_for_lr(inputs, kw["bias"], policy, np.float64)
    w = faer_logistic_reg(X, y, kw["bias"], kw.get("l1_reg", 0.0), kw.get("l2_reg", 0.0), kw.get("tol", 1e-5), kw.get("max_iter", 200))
    pred = stable_sigmoid(X @ w)
    if isinstance(mask, np.ndarray) and (~mask).any():
        out = np.zeros(len(mask))
        out[mask] = pred
        return out, mask.copy()
    return pred, np.ones(len(pred), dtype=bool)
