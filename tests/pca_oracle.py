"""NumPy restatement of pl_singular_values / pl_pca / pl_principal_components (num_ext/pca.rs:39-182) with this
project's documented choices: the SVD of the f64 matrix (np.linalg.svd), every weight vector signed so that its
largest-magnitude entry (the first on ties) is positive (sklearn's svd_flip(u_based_decision=False)), rows with a null
dropped (singular values, pca) or rejected (principal components), and the error cases of the device path."""
from __future__ import annotations

import numpy as np

MAX_FEATURES = 259
NULL_MSG = "Nulls are found in data and this method doesn't allow nulls."
NONFINITE_MSG = "SVD algorithm did not converge."


class PcaError(ValueError):
    pass


def sign_fix(V: np.ndarray) -> np.ndarray:
    """V: p x d, columns = weight vectors.  Flip each column so its largest |entry| (first on ties) is positive."""
    V = np.array(V, dtype=np.float64, copy=True)
    if V.size == 0:
        return V
    idx = np.argmax(np.abs(V), axis=0)
    s = np.sign(V[idx, np.arange(V.shape[1])])
    s[s == 0] = 1.0
    return V * s


def _matrix(cols, valid=None, drop=True):
    X = np.column_stack([np.asarray(c, dtype=np.float64) for c in cols]) if cols else np.zeros((0, 0))
    if valid is not None:
        keep = np.all(np.column_stack(valid), axis=1)
        if not drop and not keep.all():
            raise PcaError(NULL_MSG)
        X = X[keep]
    if X.shape[1] > MAX_FEATURES:
        raise PcaError(f"pca: {X.shape[1]} features; at most {MAX_FEATURES} are supported")
    return X


def _svd(X):
    if not np.all(np.isfinite(X)):
        raise PcaError(NONFINITE_MSG)
    _, s, vt = np.linalg.svd(X, full_matrices=False)
    return s, sign_fix(vt.T)


def singular_values(cols, valid=None) -> np.ndarray:
    X = _matrix(cols, valid)
    if X.shape[0] == 0:
        return np.zeros(0)
    return _svd(X)[0]


def pca(cols, valid=None):
    """-> (singular values [dim], weight vectors [dim x p], row i = vector i)"""
    X = _matrix(cols, valid)
    n, p = X.shape
    if n < p:
        raise PcaError(f"pca: {n} rows < {p} features is not supported")
    s, V = _svd(X)
    return s, V.T


def principal_components(cols, k: int, valid=None) -> np.ndarray:
    """-> n x k"""
    X = _matrix(cols, valid, drop=False)
    n, p = X.shape
    if n < k:
        return np.full((n, k), np.nan)
    if n < p:
        raise PcaError(f"principal_components: {n} rows < {p} features is not supported")
    _, V = _svd(X)
    return X @ V[:, :k]


def explained_var(s: np.ndarray) -> np.ndarray:
    """The reference's list.eval(element ** 2 / (pl.count() - 1)): the count is the list's length."""
    with np.errstate(divide="ignore", invalid="ignore"):
        return s ** 2 / np.float64(len(s) - 1)


def ratio(s: np.ndarray) -> np.ndarray:
    return s / s.sum()
