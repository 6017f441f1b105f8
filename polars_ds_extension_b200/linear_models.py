"""Model classes over the H100 engine: `LR`, `ElasticNet`, `OnlineLR`, `GLM`, `MixedModel`.

Mirror of the reference's numpy-facing classes (/root/reference/python/polars_ds/linear_models.py:134-1121), which are
thin wrappers over the PyO3 types PyLR / PyElasticNet / PyOnlineLR (src/pymodels/py_lr.rs:21-224), PyGLM
(src/pymodels/py_glm.rs:12-102) and PyMixedModel (src/pymodels/py_mixed.rs).  Same constructor arguments, method
names, null policies and error messages; the arithmetic runs in libpds_b200 (`pdsb_model_fit`, `pdsb_model_predict`,
`pdsb_online_lr_*`, `pdsb_glm_fit`, `pdsb_glm_predict`, `pdsb_mixed_fit` in include/pdsb.h): moments + solve on the
device, Woodbury updates on device-resident state, for GLM the IRLS loop of row pass + weighted moments + solve, and
for MixedModel the group pass and the REML search.  There is no CPU path: without the shared library or a CUDA device
every fit / predict raises.

Data frames: `fit_df` / `predict_df` accept this package's Arrow-backed `Frame` (and a Polars frame when polars is
installed); `GLM` has `fit_df` but, like the reference, no `predict_df`; `MixedModel` has only `fit_df`.
"""
from __future__ import annotations

import ctypes as C
from typing import Any, Dict, List, Optional, Sequence, Tuple

import numpy as np

from ._lib import (GLM_BINOMIAL, GLM_GAMMA, GLM_GAUSSIAN, GLM_POISSON, MODEL_ELASTIC_NET, MODEL_LR, MODEL_ONLINE_LR,
                   Matrix, lib)
from .frame import _group_ids, _key_order
from .typing import LRSolverMethods, NullPolicy

__all__ = ["LR", "ElasticNet", "OnlineLR", "GLM", "MixedModel"]


# ---------------------------------------------------------------------------------------------------------------
# host-side data preparation (the reference does this in Python as well: linear_models.py:45-131)
# ---------------------------------------------------------------------------------------------------------------
def _fill_value(null_policy: str) -> float:
    if null_policy == "zero":
        return 0.0
    if null_policy == "one":
        return 1.0
    try:
        v = float(null_policy)
    except Exception as e:  # same wording as linear_models.py:68-69
        raise ValueError(f"Unknown null_policy. Error: {e}")
    if not np.isfinite(v):
        raise ValueError("Unknown null_policy. Error: When null_policy is a number, it cannot be nan or infinite.")
    return v


def _nan_rows(X: np.ndarray, y: np.ndarray, null_policy: NullPolicy) -> Tuple[np.ndarray, Optional[np.ndarray]]:
    """NaN handling for numpy inputs (linear_models.py:100-131), row by row: (X with any fill applied, the rows kept or
    None for all of them).  X is N x M, y is N x 1."""
    if null_policy == "ignore":
        return X, None
    if null_policy == "raise":
        if np.isnan(X).any() or np.isnan(y).any():
            raise ValueError("Nulls found in X or y.")
        return X, None
    y_nan = np.isnan(y).any(axis=1)
    if null_policy == "skip":
        return X, ~(np.isnan(X).any(axis=1) | y_nan)
    fill = _fill_value(null_policy)
    return np.nan_to_num(X, nan=fill), ~y_nan


def _handle_nans_in_np(X: np.ndarray, y: np.ndarray, null_policy: NullPolicy) -> Tuple[np.ndarray, np.ndarray]:
    """NaN handling for numpy inputs (linear_models.py:100-131): X is N x M, y is N x 1."""
    X, keep = _nan_rows(X, y, null_policy)
    return (X, y) if keep is None else (X[keep], y[keep])


def _as_matrix(a: Any) -> np.ndarray:
    m = np.asarray(a, dtype=np.float64)       # what the reference's _sanitize_np does (linear_models.py:71-97)
    if m.ndim == 1:
        m = m.reshape((-1, 1))
    if m.ndim != 2:
        raise ValueError("Dimension mismatch.")
    n, p = m.shape
    s0, s1 = m.strides
    row_major = s1 == 8 and s0 >= 8 * p          # C order, rows possibly padded (a column slice of a wider matrix)
    col_major = s0 == 8 and s1 >= 8 * n          # F order, columns possibly padded
    if not (row_major or col_major or n <= 1 or p <= 1 and s0 > 0):
        m = np.ascontiguousarray(m)              # the C ABI takes the two dense layouts and strided vectors
    return m


def _view(m: np.ndarray) -> Matrix:
    return Matrix(m.ctypes.data, m.shape[0], m.shape[1], m.strides[0] // 8 if m.shape[0] > 1 else max(m.shape[1], 1),
                  m.strides[1] // 8 if m.shape[1] > 1 else 1)


def _call(rc: int) -> None:
    if rc != 0:   # the PyO3 classes raise ValueError(LinalgErrors::to_string) (py_lr.rs:14-18)
        raise ValueError(lib().pdsb_last_error().decode("utf-8", "replace"))


def _fit(model: int, X: np.ndarray, y: np.ndarray, add_bias: bool, solver: str = "qr", l1: float = 0.0, l2: float = 0.0,
         tol: float = 1e-5, max_iter: int = 2000, want_inv: bool = False):
    Xm, ym = _as_matrix(X), _as_matrix(y)
    q = Xm.shape[1] + int(add_bias)
    coeffs = np.empty(q, dtype=np.float64)
    inv = np.empty((q, q), dtype=np.float64) if want_inv else None
    xv, yv = _view(Xm), _view(ym)
    _call(lib().pdsb_model_fit(model, C.byref(xv), C.byref(yv), int(add_bias), solver.encode(), float(l1), float(l2),
                               float(tol), int(max_iter), coeffs.ctypes.data, inv.ctypes.data if want_inv else None))
    return coeffs, inv


def _predict(X: np.ndarray, fitted: Optional[np.ndarray], has_bias: bool) -> np.ndarray:
    if fitted is None or fitted.size == 0:
        raise ValueError("Matrix is not learned yet.")
    Xm = _as_matrix(X)
    out = np.empty((Xm.shape[0], 1), dtype=np.float64)
    xv = _view(Xm)
    _call(lib().pdsb_model_predict(C.byref(xv), fitted.ctypes.data, int(fitted.size), int(has_bias), out.ctypes.data))
    return out


def _columns_of(df: Any, names: Sequence[str]) -> np.ndarray:
    """N x len(names) float64 matrix out of a Frame / Polars frame / mapping of arrays; nulls become NaN."""
    if hasattr(df, "lazy") and hasattr(df, "collect_schema"):          # polars, when installed
        return df.lazy().select(list(names)).collect().to_numpy().astype(np.float64)
    cols = df.columns if hasattr(df, "columns") and isinstance(df.columns, dict) else df
    out = []
    for n in names:
        c = cols[n]
        if hasattr(c, "to_numpy") and not isinstance(c, np.ndarray):
            try:
                c = c.to_numpy(zero_copy_only=False)
            except TypeError:
                c = c.to_numpy()
        a = np.asarray(c)
        if a.dtype == object:
            a = np.array([np.nan if v is None else v for v in a], dtype=np.float64)
        out.append(a.astype(np.float64, copy=False))
    if not out:
        return np.empty((0, 0))
    M = np.empty((len(out[0]), len(out)))
    for r in range(0, len(M), 4096):        # column_stack in cache-sized row blocks (a plain one is ~4x slower)
        M[r:r + 4096] = np.stack([c[r:r + 4096] for c in out], axis=1)
    return M


def _df_rows(df: Any, features: List[str], target: str, null_policy: NullPolicy):
    """Null policy for data frames (linear_models.py:45-68, 296-305), row by row: (X, y, the rows kept or None for all of
    them).  Nulls, not NaNs, are what is handled."""
    Z = _columns_of(df, list(features) + [target])
    X, y = Z[:, :-1], Z[:, -1:]
    if null_policy == "ignore":
        return X, y, None
    if null_policy == "raise":
        if np.isnan(Z).any():
            raise ValueError("Nulls found in Dataframe.")
        return X, y, None
    X, keep = _nan_rows(X, y, null_policy)
    return X, y, keep


def _df_to_xy(df: Any, features: List[str], target: str, null_policy: NullPolicy) -> Tuple[np.ndarray, np.ndarray]:
    X, y, keep = _df_rows(df, features, target, null_policy)
    return (X, y) if keep is None else (X[keep], y[keep])


def _key_values(df: Any, name: str) -> np.ndarray:
    """The values of a key column of a Frame / Polars frame / mapping of arrays, as GroupBy reads them."""
    if hasattr(df, "lazy") and hasattr(df, "collect_schema"):          # polars, when installed
        return df.lazy().select(name).collect().to_series().to_numpy()
    cols = df.columns if hasattr(df, "columns") and isinstance(df.columns, dict) else df
    c = cols[name]
    if hasattr(c, "to_numpy") and not isinstance(c, np.ndarray):
        try:
            return c.to_numpy(zero_copy_only=False)
        except TypeError:
            return c.to_numpy()
    return np.asarray(c)


def _with_prediction(df: Any, names: List[str], coeffs: np.ndarray, bias: float, name: str, predict):
    if len(names) <= 0:
        raise ValueError(
            "The linear model is not fitted on a dataframe, or no feature names have been given."
            "Not enough info to predict on a dataframe. Hint: try .fit_df() or .set_input_features()."
        )
    if hasattr(df, "lazy") and hasattr(df, "collect_schema"):          # polars: stays an expression, like the reference
        import polars as pl

        pred = pl.sum_horizontal(beta * pl.col(c) for c, beta in zip(names, coeffs))
        if bias != 0.0:
            pred = pred + bias
        return df.with_columns(pred.alias(name))
    return df.with_columns(**{name: predict(_columns_of(df, names)).ravel()})


class _Base:
    feature_names_in_: List[str]
    _fitted: Optional[np.ndarray]      # coefficients, bias last when _has_bias
    _has_bias: bool

    def is_fit(self) -> bool:
        return self._fitted is not None and self._fitted.size > 0

    def set_input_features(self, features: List[str]):
        self.feature_names_in_ = list(features)
        return self

    def coeffs(self) -> np.ndarray:
        """A copy of the coefficients (bias excluded)."""
        if not self.is_fit():
            raise ValueError("Matrix is not learned yet.")
        n = self._fitted.size - int(self._has_bias)
        return self._fitted[:n].copy()

    def bias(self) -> float:
        return float(self._fitted[-1]) if (self.is_fit() and self._has_bias) else 0.0

    def _set_coeffs_and_bias(self, coeffs, bias: float) -> None:
        # set_coeffs_and_bias (lr_solvers.rs:38-51): the bias is kept only when |bias| > eps
        c = np.ascontiguousarray(coeffs, dtype=np.float64).ravel()
        self._has_bias = abs(bias) > np.finfo(np.float64).eps
        self._fitted = np.concatenate([c, [bias]]) if self._has_bias else c.copy()

    def predict(self, X: np.ndarray) -> np.ndarray:
        return _predict(X, self._fitted, self._has_bias)

    def predict_df(self, df: Any, name: str = "prediction"):
        return _with_prediction(df, self.feature_names_in_, self.coeffs(), self.bias(), name, self.predict)

    def _describe(self, title: str) -> str:
        if not self.is_fit():
            return f"{title}\nNot fitted yet."
        return f"{title}\nCoefficients: {[round(float(x), 5) for x in self.coeffs()]}\nBias/Intercept: {self.bias()}\n"


class LR(_Base):
    """Ordinary least squares / ridge (linear_models.py:134-347; PyLR, py_lr.rs:21-80)."""

    def __init__(self, has_bias: bool = False, lambda_: float = 0.0, solver: LRSolverMethods = "qr",
                 feature_names_in_: Optional[List[str]] = None):
        self._has_bias = bool(has_bias)
        self.lambda_ = float(lambda_)
        self.solver = str(solver)
        self._fitted = None
        self.feature_names_in_ = [] if feature_names_in_ is None else list(feature_names_in_)

    @classmethod
    def from_values(cls, coeffs: List[float], bias: float = 0.0, feature_names_in_: Optional[List[str]] = None):
        m = cls(has_bias=(bias != 0.0), lambda_=0.0, solver="Not Solved", feature_names_in_=feature_names_in_)
        m._set_coeffs_and_bias(coeffs, float(bias))
        return m

    def __repr__(self) -> str:
        return self._describe("Linear Regression (Ridge) Model" if self.lambda_ > 0.0 else "Linear Regression Model")

    def fit(self, X: np.ndarray, y: np.ndarray, null_policy: NullPolicy = "ignore"):
        X_, y_ = _handle_nans_in_np(_as_matrix(X), _as_matrix(y).reshape((-1, 1)), null_policy)
        self._fitted, _ = _fit(MODEL_LR, X_, y_, self._has_bias, solver=self.solver, l2=self.lambda_)
        return self

    def fit_df(self, df: Any, features: List[str], target: str, null_policy: NullPolicy = "skip",
               show_report: bool = False):
        if show_report and self.lambda_ == 0.0:
            from .exprs.expr_linear import lin_reg_report

            frame = df if hasattr(df, "select") and hasattr(df, "columns") and isinstance(df.columns, dict) else None
            if frame is not None:
                print(frame.select(lin_reg_report(*features, target=target, add_bias=self._has_bias)))
        X, y = _df_to_xy(df, list(features), target, null_policy)
        self.feature_names_in_ = list(features)
        self._fitted, _ = _fit(MODEL_LR, X, y, self._has_bias, solver=self.solver, l2=self.lambda_)
        return self


class ElasticNet(_Base):
    """Elastic net by coordinate descent (linear_models.py:350-557; PyElasticNet, py_lr.rs:82-147).  Equivalent to
    scikit-learn's with alpha = l1_reg + l2_reg and l1_ratio = l1_reg / (l1_reg + l2_reg)."""

    def __init__(self, l1_reg: float, l2_reg: float, has_bias: bool = False, tol: float = 1e-5, max_iter: int = 2000,
                 feature_names_in_: Optional[List[str]] = None):
        if l1_reg <= 0.0 and l2_reg <= 0.0:
            raise ValueError("Cannot have both l1_reg and l2_reg <= 0.")
        self.l1_reg, self.l2_reg = float(l1_reg), float(l2_reg)
        self.tol, self.max_iter = float(tol), int(max_iter)
        self._has_bias = bool(has_bias)
        self._fitted = None
        self.feature_names_in_ = [] if feature_names_in_ is None else list(feature_names_in_)

    @classmethod
    def from_values(cls, coeffs: List[float], bias: float = 0.0, feature_names_in_: Optional[List[str]] = None):
        m = cls.__new__(cls)
        m.l1_reg = m.l2_reg = float("nan")       # ElasticNet::from_values (lr_solvers.rs:99-110)
        m.tol, m.max_iter = 1e-5, 2000
        m._fitted = None
        m.feature_names_in_ = [] if feature_names_in_ is None else list(feature_names_in_)
        m._set_coeffs_and_bias(coeffs, float(bias))
        return m

    def has_bias(self) -> bool:
        return self._has_bias

    def regularizers(self) -> Tuple[float, float]:
        return self.l1_reg, self.l2_reg

    def __repr__(self) -> str:
        return self._describe("ElasticNet Model")

    def _run(self, X, y):
        self._fitted, _ = _fit(MODEL_ELASTIC_NET, X, y, self._has_bias, l1=self.l1_reg, l2=self.l2_reg, tol=self.tol,
                               max_iter=self.max_iter)
        return self

    def fit(self, X: np.ndarray, y: np.ndarray, null_policy: NullPolicy = "ignore"):
        X_, y_ = _handle_nans_in_np(_as_matrix(X), _as_matrix(y).reshape((-1, 1)), null_policy)
        return self._run(X_, y_)

    def fit_df(self, df: Any, features: List[str], target: str, null_policy: NullPolicy = "skip"):
        X, y = _df_to_xy(df, list(features), target, null_policy)
        self.feature_names_in_ = list(features)
        return self._run(X, y)


class OnlineLR:
    """Online OLS / ridge: initial fit, then rank-1 Woodbury updates (linear_models.py:560-700; PyOnlineLR,
    py_lr.rs:149-224).  The inverse of X'X and the coefficients live on the device between updates; a row with a NaN
    is ignored by `update`."""

    def __init__(self, lambda_: float = 0.0, has_bias: bool = False):
        self.lambda_ = float(lambda_)
        self._has_bias = bool(has_bias)
        self._h: Optional[int] = None
        self._q = 0

    def __del__(self):
        h, self._h = getattr(self, "_h", None), None
        if h:
            try:
                lib().pdsb_online_lr_free(h)
            except Exception:
                pass

    def _state(self, q: int, has_bias: bool) -> int:
        if self._h and self._q == q and self._has_bias == has_bias:
            return self._h
        if self._h:
            lib().pdsb_online_lr_free(self._h)
            self._h = None
        h = lib().pdsb_online_lr_new(q, int(has_bias))
        if not h:
            raise ValueError(lib().pdsb_last_error().decode("utf-8", "replace"))
        self._h, self._q, self._has_bias = h, q, has_bias
        return h

    @classmethod
    def from_coeffs_bias_inverse(cls, coeffs: List[float], bias: float, inv: np.ndarray):
        c = np.ascontiguousarray(coeffs, dtype=np.float64).ravel()
        inv = np.ascontiguousarray(inv, dtype=np.float64)
        m = cls(lambda_=0.0, has_bias=(bias > 0.0))
        has_bias = abs(bias) > np.finfo(np.float64).eps
        full = np.concatenate([c, [bias]]) if has_bias else c
        # The reference compares len(coeffs) with inv.ncols() (lr_online_solvers.rs:35-36), which rejects every model
        # WITH a bias (its inverse has one more row/column); here the inverse must match coefficients + bias.
        if inv.ndim != 2 or inv.shape != (full.size, full.size):
            raise ValueError("Dimension mismatch.")
        _call(lib().pdsb_online_lr_set(m._state(full.size, has_bias), full.ctypes.data, inv.ctypes.data))
        return m

    def is_fit(self) -> bool:
        return bool(self._h)

    def __repr__(self) -> str:
        title = "Online Linear Regression (Ridge) Model" if self.lambda_ > 0.0 else "Online Linear Regression Model"
        if not self.is_fit():
            return f"{title}\nNot fitted yet."
        return f"{title}\nCoefficients: {[round(float(x), 5) for x in self.coeffs()]}\nBias/Intercept: {self.bias()}\n"

    def _get(self, want_inv: bool = False):
        if not self._h:
            raise ValueError("Matrix is not learned yet.")
        w = np.empty(self._q, dtype=np.float64)
        inv = np.empty((self._q, self._q), dtype=np.float64) if want_inv else None
        _call(lib().pdsb_online_lr_get(self._h, w.ctypes.data, inv.ctypes.data if want_inv else None))
        return w, inv

    def coeffs(self) -> np.ndarray:
        w, _ = self._get()
        return w[: self._q - int(self._has_bias)]

    def bias(self) -> float:
        if not self._h or not self._has_bias:
            return 0.0
        return float(self._get()[0][-1])

    def inv(self) -> np.ndarray:
        return self._get(want_inv=True)[1]

    def fit(self, X: np.ndarray, y: np.ndarray):
        Xm, ym = _as_matrix(X), _as_matrix(y).reshape((-1, 1))
        if np.isnan(Xm).any() or np.isnan(ym).any():
            raise ValueError("Online regression currently must fit without null for the initial fit.")
        w, inv = _fit(MODEL_ONLINE_LR, Xm, ym, self._has_bias, l2=self.lambda_, want_inv=True)
        _call(lib().pdsb_online_lr_set(self._state(w.size, self._has_bias), w.ctypes.data, inv.ctypes.data))
        return self

    def update(self, X: np.ndarray, y: Any, c: float = 1.0):
        if not self.is_fit():
            raise ValueError("You cannot update before the initial fit of the matrix.")
        x = np.ascontiguousarray(np.asarray(X, dtype=np.float64).reshape((1, -1)))
        if x.shape[1] != self._q - int(self._has_bias):
            raise ValueError("Dimension mismatch.")
        yv = float(np.asarray(y, dtype=np.float64).reshape((1, 1))[0, 0])
        _call(lib().pdsb_online_lr_update(self._h, x.ctypes.data, yv, float(c)))
        return self

    def predict(self, X: np.ndarray) -> np.ndarray:
        w, _ = self._get()
        return _predict(X, w, self._has_bias)


# GLMFamily::from (glm_solvers.rs:49-63) for the strings the Python class accepts (linear_models.py:700, 762-763)
_GLM_FAMILIES = {"gaussian": GLM_GAUSSIAN, "normal": GLM_GAUSSIAN, "poisson": GLM_POISSON, "binomial": GLM_BINOMIAL,
                 "logistic": GLM_BINOMIAL, "gamma": GLM_GAMMA}
# the Debug names of LinkFunction / VarianceFunction (link_functions.rs) that GLM::to_string prints (glm_solvers.rs:100-104)
_GLM_NAMES = {GLM_GAUSSIAN: ("Identity", "Gaussian"), GLM_POISSON: ("Log", "Poisson"), GLM_BINOMIAL: ("Logit", "Binomial"),
              GLM_GAMMA: ("Inverse", "Gamma")}


def _glm_fit(family: int, X: np.ndarray, y: np.ndarray, add_bias: bool, max_iter: int, tol: float):
    """faer_irls on the device: (coefficients with the bias last, iterations run)."""
    Xm, ym = _as_matrix(X), _as_matrix(y)
    coeffs = np.empty(Xm.shape[1] + int(add_bias), dtype=np.float64)
    n_iter = C.c_int64(0)
    xv, yv = _view(Xm), _view(ym)
    _call(lib().pdsb_glm_fit(C.byref(xv), C.byref(yv), int(add_bias), int(family), int(max_iter), float(tol),
                             coeffs.ctypes.data, C.addressof(n_iter)))
    return coeffs, int(n_iter.value)


def _glm_fit_by(family: int, X: np.ndarray, y: np.ndarray, offsets: np.ndarray, add_bias: bool, max_iter: int,
                tol: float):
    """Every group's faer_irls on the device in one call: (coefficients [n_groups, p + bias] with the bias last,
    iterations [n_groups]).  Group g is rows [offsets[g], offsets[g+1]) of X and y."""
    Xm, ym = _as_matrix(X), _as_matrix(y)
    ng = len(offsets) - 1
    off = np.ascontiguousarray(offsets, dtype=np.int64)
    coeffs = np.empty((ng, Xm.shape[1] + int(add_bias)), dtype=np.float64)
    n_iter = np.empty(ng, dtype=np.int64)
    xv, yv = _view(Xm), _view(ym)
    _call(lib().pdsb_glm_fit_by(C.byref(xv), C.byref(yv), off.ctypes.data, ng, int(add_bias), int(family),
                                int(max_iter), float(tol), coeffs.ctypes.data, n_iter.ctypes.data, None))
    return coeffs, n_iter


class GLM:
    """Generalized linear model fitted by iteratively reweighted least squares (linear_models.py:705-950; PyGLM,
    py_glm.rs:12-102; GLM::fit -> faer_irls, glm_solvers.rs:196-216, 249-359).  Each family uses its canonical link:

        gaussian / normal    ==>   identity
        poisson              ==>   log
        binomial / logistic  ==>   logit
        gamma                ==>   inverse

    Every iteration runs on the device: weights and working response per row, the weighted moments, the QR solve.  It
    stops when no coefficient moves by `tol` or more, or after `max_iter` iterations.  Inputs outside a family's domain
    (e.g. negative counts for poisson) are not checked and give non-finite coefficients, as in the reference."""

    def __init__(self, add_bias: bool = False, solver: str = "irls", family: str = "normal", max_iter: int = 100,
                 tol: float = 1e-8, feature_names_in_: Optional[List[str]] = None):
        if solver not in ["irls"]:
            raise NotImplementedError
        if max_iter < 1:
            raise ValueError("`max_iter` must be > 1.")
        if family not in _GLM_FAMILIES:
            raise NotImplementedError
        self._add_bias = bool(add_bias)
        self._family = _GLM_FAMILIES[family]
        self._max_iter = int(max_iter)
        self._tol = abs(float(tol))
        self._fitted: Optional[np.ndarray] = None
        self.feature_names_in_: List[str] = [] if feature_names_in_ is None else list(feature_names_in_)

    def __repr__(self) -> str:
        link, variance = _GLM_NAMES[self._family]
        return f"GLM:\nLink: {link}\nVariance: {variance}"

    def is_fit(self) -> bool:
        return self._fitted is not None and self._fitted.size > 0

    def set_input_features(self, features: List[str]):
        self.feature_names_in_ = list(features)
        return self

    def coeffs(self) -> np.ndarray:
        """A copy of the coefficients (bias excluded)."""
        if not self.is_fit():
            raise ValueError("Matrix is not learned yet.")
        return self._fitted[: self._fitted.size - int(self._add_bias)].copy()

    def bias(self) -> float:
        return float(self._fitted[-1]) if (self.is_fit() and self._add_bias) else 0.0

    def _run(self, X: np.ndarray, y: np.ndarray):
        self._fitted, _ = _glm_fit(self._family, X, y, self._add_bias, self._max_iter, self._tol)
        return self

    def fit(self, X: np.ndarray, y: np.ndarray, null_policy: NullPolicy = "ignore"):
        X_, y_ = _handle_nans_in_np(_as_matrix(X), _as_matrix(y).reshape((-1, 1)), null_policy)
        return self._run(X_, y_)

    def fit_df(self, df: Any, features: List[str], target: str, null_policy: NullPolicy = "skip",
               show_report: bool = False):
        """`show_report` is accepted and ignored, as in the reference."""
        X, y = _df_to_xy(df, list(features), target, null_policy)
        self.feature_names_in_ = list(features)
        return self._run(X, y)

    def _run_by(self, X: np.ndarray, y: np.ndarray, keys: np.ndarray, keep: Optional[np.ndarray], name: str):
        if len(keys) != X.shape[0] or y.shape[0] != X.shape[0]:
            raise ValueError("Dimension mismatch.")
        uniq, gid = _group_ids(np.asarray(keys))        # the groups of every row, before the null policy drops any
        if keep is not None:
            X, y, gid = X[keep], y[keep], gid[keep]
        order, offsets = _key_order(gid, len(uniq))
        # what GLM.fit does on a group's rows: fewer rows than features (none at all included) is an error
        if X.shape[1] == 0 or (np.diff(offsets) < max(X.shape[1], 1)).any():
            raise ValueError("Not enough rows / columns.")
        coeffs, n_iter = _glm_fit_by(self._family, X[order], y[order], offsets, self._add_bias, self._max_iter,
                                     self._tol)
        return {name: uniq, "coeffs": coeffs, "n_iter": n_iter}

    def fit_by(self, X: np.ndarray, y: np.ndarray, group: Any, null_policy: NullPolicy = "ignore") -> Dict[str, Any]:
        """`fit` on every group of rows at once, on the device: group g is the rows whose `group` value is the g-th
        distinct one in first-seen order.  The null policy applies row by row as in `fit`, after the groups are formed.
        Returns {"group": keys, "coeffs": [n_groups, p + bias] float64 with the bias last, "n_iter": [n_groups] int64};
        row g is what `fit` gives on group g's rows, to rounding.  Raises as `fit` would on the first group it cannot fit
        (fewer rows than features).  The model itself is not changed."""
        Xm, ym = _as_matrix(X), _as_matrix(y).reshape((-1, 1))
        if ym.shape[0] != Xm.shape[0]:
            raise ValueError("Dimension mismatch.")
        X_, keep = _nan_rows(Xm, ym, null_policy)
        return self._run_by(X_, ym, np.asarray(group).reshape(-1), keep, "group")

    def fit_df_by(self, df: Any, features: List[str], target: str, by: str,
                  null_policy: NullPolicy = "skip") -> Dict[str, Any]:
        """`fit_df` on every group of `by` at once; the result is keyed by `by` (see `fit_by`)."""
        X, y, keep = _df_rows(df, list(features), target, null_policy)
        return self._run_by(X, y, _key_values(df, by), keep, by)

    def predict(self, X: np.ndarray, linear: bool = False) -> np.ndarray:
        """E[y | X] = g^-1(X beta + bias), or the linear predictor X beta + bias when `linear`; shape (n, 1)."""
        if not self.is_fit():
            raise ValueError("Matrix is not learned yet.")
        Xm = _as_matrix(X)
        out = np.empty((Xm.shape[0], 1), dtype=np.float64)
        xv = _view(Xm)
        _call(lib().pdsb_glm_predict(C.byref(xv), self._fitted.ctypes.data, int(self._fitted.size), int(self._add_bias),
                                     int(self._family), int(bool(linear)), out.ctypes.data))
        return out


# ---------------------------------------------------------------------------------------------------------------
# MixedModel (linear_models.py:956-1121; PyMixedModel, src/pymodels/py_mixed.rs; fit_reml, src/linear/mixed/mod.rs)
# ---------------------------------------------------------------------------------------------------------------
def _group_column(df: Any, name: str) -> Tuple[np.ndarray, np.ndarray]:
    """(values, is_null) of a key column of any type (strings included) out of a Frame / Polars frame / mapping."""
    if hasattr(df, "lazy") and hasattr(df, "collect_schema"):          # polars, when installed
        s = df.lazy().select(name).collect().to_series()
        null = s.is_null().to_numpy()
        return s.to_numpy(), null
    cols = df.columns if hasattr(df, "columns") and isinstance(df.columns, dict) else df
    c = cols[name]
    if hasattr(c, "is_null") and hasattr(c, "to_pylist"):              # pyarrow
        import pyarrow as pa
        import pyarrow.compute as pc

        arr = c.combine_chunks() if hasattr(c, "combine_chunks") else c
        null = np.asarray(arr.is_null().to_numpy(zero_copy_only=False), dtype=bool)
        t = arr.type
        if pa.types.is_integer(t) or pa.types.is_floating(t) or pa.types.is_boolean(t) or pa.types.is_temporal(t):
            return np.asarray(pc.fill_null(arr, pa.scalar(0, type=t) if not pa.types.is_boolean(t) else False)
                              .to_numpy(zero_copy_only=False)), null
        if pa.types.is_string(t) or pa.types.is_large_string(t):
            # the ranks of the distinct strings in sorted order stand in for the strings: same dense codes
            enc = arr.dictionary_encode()
            words = np.asarray(enc.dictionary.to_pylist(), dtype=object)
            rank = np.empty(len(words), dtype=np.int64)
            rank[np.argsort(words, kind="stable")] = np.arange(len(words))
            return rank[pc.fill_null(enc.indices, 0).to_numpy(zero_copy_only=False)], null
        return np.asarray(arr.to_pylist(), dtype=object), null
    a = np.asarray(c)
    if a.dtype == object:
        null = np.array([v is None for v in a], dtype=bool)
    elif a.dtype.kind == "f":
        null = np.isnan(a)
    else:
        null = np.zeros(len(a), dtype=bool)
    return a, null


def _mixed_inputs(Z: np.ndarray, keys: np.ndarray, key_null: np.ndarray, null_policy: NullPolicy):
    """MixedModel.fit_df's preparation (linear_models.py:1066-1094).  Z: the features then the target, nulls as NaN.
    Returns X = [1 | features], y, dense group codes (0-based, in sorted key order), n_groups and between_idx."""
    feats, y = Z[:, :-1], Z[:, -1]
    keep = np.ones(len(y), dtype=bool)
    if null_policy == "skip":
        keep = ~np.isnan(Z).any(axis=1)
    elif null_policy not in ("ignore", "raise"):
        fill = _fill_value(null_policy)
        feats = np.where(np.isnan(feats), fill, feats)
        keep = ~np.isnan(y)
    keep &= ~key_null                                                    # .drop_nulls(subset=[group])
    if not keep.all():
        feats, y, keys = feats[keep], y[keep], keys[keep]
    if null_policy == "raise" and (np.isnan(feats).any() or np.isnan(y).any()):
        raise ValueError("Nulls found in Dataframe.")
    n = len(y)
    X = np.empty((n, feats.shape[1] + 1))
    X[:, 0] = 1.0
    X[:, 1:] = feats
    # one stable sort of the keys gives the dense codes (rank("dense") - 1) and the rows in group order for the
    # between test: a feature is "between" when n_unique(group, f) == n_unique(group), i.e. constant within every
    # group (NaN == NaN)
    codes, n_groups, between = np.zeros(n, dtype=np.int64), 0, [0]
    if n > 0:
        order = np.argsort(keys, kind="stable")
        ks = keys[order]
        new = np.empty(n, dtype=bool)
        new[0] = True
        new[1:] = ks[1:] != ks[:-1]
        cs = np.cumsum(new) - 1
        codes[order] = cs
        n_groups = int(cs[-1]) + 1
        if feats.shape[1] > 0:
            first = feats[order[new]]                                   # each group's first row
            const = np.ones(feats.shape[1], dtype=bool)
            for a in range(0, n, 1 << 16):                              # contiguous row blocks, all features at once
                blk = feats[a:a + (1 << 16)]
                ref = first[codes[a:a + (1 << 16)]]
                const &= ((blk == ref) | (np.isnan(blk) & np.isnan(ref))).all(axis=0)
            between += [int(j) + 1 for j in np.flatnonzero(const)]
    return X, np.ascontiguousarray(y), codes, n_groups, between


def _two_sided_p(t: np.ndarray, df: np.ndarray) -> np.ndarray:
    """student_t_two_sided_pvalue (py_stats.rs:8-11): clamp(2 sf(|t|, df), 0, 1)."""
    sf = lib().pdsb_student_t_sf
    return np.array([min(max(2.0 * sf(abs(float(ti)), float(di)), 0.0), 1.0) for ti, di in zip(t, df)], dtype=np.float64)


def _mixed_fit(X: np.ndarray, y: np.ndarray, codes: np.ndarray, n_groups: int, between: Sequence[int], max_iter: int,
               tol: float):
    """fit_reml on the device: (coeffs, std_errors, dfs, gamma, resid_variance, deviance evaluations)."""
    Xm, ym = _as_matrix(X), _as_matrix(np.asarray(y, dtype=np.float64).reshape(-1, 1))
    c = np.ascontiguousarray(codes, dtype=np.int64).ravel()
    if c.size != Xm.shape[0] or ym.shape[0] != Xm.shape[0]:
        raise ValueError("X, y, and group must have the same number of rows.")
    b = np.ascontiguousarray(between, dtype=np.int64)
    p = Xm.shape[1]
    coeffs, se, dfs = np.empty(p), np.empty(p), np.empty(p)
    gamma, rv, n_evals = C.c_double(0.0), C.c_double(0.0), C.c_int64(0)
    xv, yv = _view(Xm), _view(ym)
    _call(lib().pdsb_mixed_fit(C.byref(xv), C.byref(yv), c.ctypes.data, int(n_groups), b.ctypes.data, int(b.size),
                               int(max_iter), float(tol), coeffs.ctypes.data, se.ctypes.data, dfs.ctypes.data,
                               C.addressof(gamma), C.addressof(rv), C.addressof(n_evals)))
    return coeffs, se, dfs, float(gamma.value), float(rv.value), int(n_evals.value)


class MixedModel:
    """A random-intercept linear mixed model, fit via restricted maximum likelihood (REML).

        y = X @ beta + Z @ u + e,   u ~ N(0, sigma_g^2 I),   e ~ N(0, sigma_e^2 I)

    X is the fixed-effect design (an intercept column plus the given features) and Z the indicator matrix of `group`:
    one random intercept per group level.  Degrees of freedom follow containment, as SAS PROC MIXED does for this
    model: effects constant within every group level (the intercept included) are tested against the group stratum,
    the rest against the residual stratum.

    The fit runs on the device from per-group summaries taken in one pass over the rows; the golden-section search
    over gamma = sigma_g^2 / sigma_e^2 then works on small (p + 1) x (p + 1) matrices.  At most 64 fixed effects
    (intercept included)."""

    def __init__(self):
        self.feature_names_in_: List[str] = []
        self.group_name_in_: Optional[str] = None
        self._coeffs = np.empty(0)
        self._std_errors = np.empty(0)
        self._dfs = np.empty(0)
        self._gamma = 0.0
        self._resid_variance = 0.0
        self._is_fit = False

    def is_fit(self) -> bool:
        return self._is_fit

    @property
    def coeffs_(self) -> np.ndarray:
        return self._coeffs.copy()

    @property
    def std_errors_(self) -> np.ndarray:
        return self._std_errors.copy()

    @property
    def dfs_(self) -> np.ndarray:
        return self._dfs.copy()

    @property
    def gamma_(self) -> float:
        """Variance ratio sigma_g^2 / sigma_e^2 at the REML optimum."""
        return self._gamma

    @property
    def resid_variance_(self) -> float:
        """Residual variance sigma_e^2."""
        return self._resid_variance

    def __repr__(self) -> str:
        if not self.is_fit():
            return "MixedModel (not fitted yet)"
        return (
            "MixedModel(Random Intercept, REML)\n"
            f"Group: {self.group_name_in_}\n"
            f"Variance ratio (group / residual): {self.gamma_:.6g}\n"
            f"{self.report()}"
        )

    def fit_df(self, df: Any, features: List[str], target: str, group: str, null_policy: NullPolicy = "skip",
               max_iter: int = 200, tol: float = 1e-10):
        """Fit on a data frame: `features` are the fixed-effect columns (an intercept is added), `group` the column of
        the random-intercept grouping factor (any key type).  `max_iter` bounds the golden-section steps over gamma and
        `tol` is the bracket width at which the search stops."""
        Z = _columns_of(df, list(features) + [target])
        keys, key_null = _group_column(df, group)
        X, y, codes, n_groups, between = _mixed_inputs(Z, keys, key_null, null_policy)
        (self._coeffs, self._std_errors, self._dfs, self._gamma, self._resid_variance, _) = _mixed_fit(
            X, y, codes, n_groups, between, max_iter, tol)
        self._is_fit = True
        self.feature_names_in_ = list(features)
        self.group_name_in_ = group
        return self

    def report(self):
        """One row per fixed effect (intercept first): effect, estimate, std_err, df, t and the two-sided p-value.  A
        polars DataFrame when polars is installed, this package's `Frame` otherwise."""
        if not self.is_fit():
            raise ValueError("Model is not fit yet.")
        t = self._coeffs / self._std_errors
        data = {"effect": ["Intercept"] + self.feature_names_in_, "estimate": self.coeffs_, "std_err": self.std_errors_,
                "df": self.dfs_, "t": t, "p_value": _two_sided_p(t, self._dfs)}
        try:
            import polars as pl
        except ImportError:
            from .frame import Frame

            return Frame(data)
        return pl.DataFrame(data)
