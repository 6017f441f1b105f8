"""GLM.fit_by / fit_df_by without a GPU: the C declarations, what the Python layer sends the C entry (rows in
first-seen key order, offsets, family, the instance's max_iter and tol), the null policies row by row, groups the
policy empties, the argument checks that run before any device work, and the loud failure without a device."""
import ctypes as C
import re
from pathlib import Path

import numpy as np
import pyarrow as pa
import pytest

from tests.helpers import has_gpu

ROOT = Path(__file__).resolve().parents[1]


def test_header_declares_both_entries():
    h = (ROOT / "include" / "pdsb.h").read_text()
    flat = re.sub(r"\s+", " ", h)
    assert ("int pdsb_dev_grouped_glm_f64(const double* X, int64_t ldx, const double* y, const double* mask, "
            "const int64_t* offsets, int64_t n_groups, int64_t n, int p, int add_bias, int family, double tol, "
            "int64_t max_iter, double* beta, int* status, int64_t* n_iter, void* stream);") in flat
    assert ("int pdsb_glm_fit_by(const pdsb_matrix* X, const pdsb_matrix* y, const int64_t* offsets, int64_t n_groups, "
            "int add_bias, int family, int64_t max_iter, double tol, double* coeffs, int64_t* n_iter, int* status);") in flat
    assert "enum pdsb_glm_status" in flat
    from polars_ds_extension_b200 import _lib

    assert (_lib.GLM_CONVERGED, _lib.GLM_MAX_ITER, _lib.GLM_FAILED, _lib.GLM_EMPTY) == (0, 1, 2, 3)


class _Capture:
    """A stand-in for the library that records what pdsb_glm_fit_by receives and returns zeros."""

    def __init__(self):
        self.calls = []

    def pdsb_glm_fit_by(self, xv, yv, off, ng, bias, family, max_iter, tol, coeffs, n_iter, status):
        def mat(ref):
            m = ref._obj
            a = np.ctypeslib.as_array(C.cast(m.data, C.POINTER(C.c_double)),
                                      shape=(max(1, (m.n_rows - 1) * m.row_stride + (m.n_cols - 1) * m.col_stride + 1),))
            return np.array([[a[i * m.row_stride + j * m.col_stride] for j in range(m.n_cols)] for i in range(m.n_rows)])

        offsets = np.ctypeslib.as_array(C.cast(off, C.POINTER(C.c_int64)), shape=(ng + 1,)).copy()
        q = mat(xv).shape[1] + bias
        np.ctypeslib.as_array(C.cast(coeffs, C.POINTER(C.c_double)), shape=(ng * q,))[:] = 0.0
        np.ctypeslib.as_array(C.cast(n_iter, C.POINTER(C.c_int64)), shape=(ng,))[:] = 1
        self.calls.append(dict(X=mat(xv), y=mat(yv)[:, 0], offsets=offsets, n_groups=ng, add_bias=bias, family=family,
                               max_iter=max_iter, tol=tol))
        return 0


@pytest.fixture
def captured(monkeypatch):
    from polars_ds_extension_b200 import linear_models

    cap = _Capture()
    monkeypatch.setattr(linear_models, "lib", lambda: cap)
    return cap


def _case():
    X = np.arange(16, dtype=np.float64).reshape(8, 2) / 10.0
    y = np.arange(8, dtype=np.float64) + 1.0
    key = np.array(["b", "a", "b", "c", "a", "b", "c", "a"], dtype=object)
    return X, y, key


def test_fit_by_sends_rows_in_first_seen_key_order(captured):
    from polars_ds_extension_b200.linear_models import GLM

    X, y, key = _case()
    m = GLM(add_bias=True, family="gamma", max_iter=17, tol=-3e-7)
    res = m.fit_by(X, y, key)
    (c,) = captured.calls
    order = [0, 2, 5, 1, 4, 7, 3, 6]                      # "b" rows, then "a", then "c", each stable
    assert np.array_equal(c["X"], X[order]) and np.array_equal(c["y"], y[order])
    assert c["offsets"].tolist() == [0, 3, 6, 8] and c["n_groups"] == 3
    assert (c["family"], c["add_bias"], c["max_iter"], c["tol"]) == (3, 1, 17, 3e-7)
    assert list(res["group"]) == ["b", "a", "c"]
    assert res["coeffs"].shape == (3, 3) and res["coeffs"].dtype == np.float64
    assert res["n_iter"].tolist() == [1, 1, 1] and res["n_iter"].dtype == np.int64
    assert not m.is_fit()


@pytest.mark.parametrize("family,code", [("normal", 0), ("gaussian", 0), ("poisson", 1), ("logistic", 2),
                                         ("binomial", 2), ("gamma", 3)])
def test_family_codes(captured, family, code):
    from polars_ds_extension_b200.linear_models import GLM

    X, y, key = _case()
    GLM(family=family).fit_by(X, y, key)
    assert captured.calls[0]["family"] == code and captured.calls[0]["add_bias"] == 0
    assert captured.calls[0]["max_iter"] == 100 and captured.calls[0]["tol"] == 1e-8


def _nulls():
    X, y, key = _case()
    X = X.copy()
    y = y.copy()
    X[2, 1] = np.nan        # a "b" row
    y[4] = np.nan           # an "a" row
    return X, y, key


def test_null_policies_row_by_row(captured):
    from polars_ds_extension_b200.linear_models import GLM

    X, y, key = _nulls()
    m = GLM(add_bias=True)
    m.fit_by(X, y, key, null_policy="skip")
    c = captured.calls[-1]
    assert np.array_equal(c["X"], X[[0, 5, 1, 7, 3, 6]]) and c["offsets"].tolist() == [0, 2, 4, 6]
    m.fit_by(X, y, key, null_policy="zero")                 # X filled, the row with a null y dropped
    c = captured.calls[-1]
    want = np.nan_to_num(X, nan=0.0)[[0, 2, 5, 1, 7, 3, 6]]
    assert np.array_equal(c["X"], want) and c["offsets"].tolist() == [0, 3, 5, 7]
    m.fit_by(X, y, key, null_policy="2.5")
    assert captured.calls[-1]["X"][1, 1] == 2.5
    m.fit_by(X, y, key, null_policy="ignore")
    assert np.isnan(captured.calls[-1]["X"][1, 1]) and captured.calls[-1]["offsets"].tolist() == [0, 3, 6, 8]
    with pytest.raises(ValueError, match="Nulls found in X or y."):
        m.fit_by(X, y, key, null_policy="raise")
    with pytest.raises(ValueError, match="Unknown null_policy"):
        m.fit_by(X, y, key, null_policy="nope")


def test_fit_df_by_null_policies_match_fit_df(captured):
    import polars_ds_extension_b200 as pds
    from polars_ds_extension_b200.linear_models import GLM

    X, y, key = _nulls()
    df = pds.Frame({"a": pa.array(X[:, 0]), "b": pa.array([None if np.isnan(v) else v for v in X[:, 1]], pa.float64()),
                    "y": pa.array([None if np.isnan(v) else v for v in y], pa.float64()),
                    "k": pa.array(list(key))})
    res = GLM(add_bias=False, family="poisson").fit_df_by(df, ["a", "b"], "y", by="k")   # default "skip"
    c = captured.calls[-1]
    assert np.array_equal(c["X"], X[[0, 5, 1, 7, 3, 6]]) and c["offsets"].tolist() == [0, 2, 4, 6]
    assert list(res["k"]) == ["b", "a", "c"] and "group" not in res
    GLM(family="poisson").fit_df_by(df, ["a", "b"], "y", by="k", null_policy="one")
    assert captured.calls[-1]["X"][1, 1] == 1.0 and captured.calls[-1]["offsets"].tolist() == [0, 3, 5, 7]
    with pytest.raises(ValueError, match="Nulls found in Dataframe."):
        GLM().fit_df_by(df, ["a", "b"], "y", by="k", null_policy="raise")


def test_group_emptied_by_skip_raises_as_the_single_fit(captured):
    """GLM.fit on zero rows (or fewer rows than features) raises "Not enough rows / columns." (pdsb_glm_fit); the
    grouped call raises the same before any device work."""
    from polars_ds_extension_b200.linear_models import GLM

    X, y, key = _case()
    X = X.copy()
    X[[3, 6], 0] = np.nan                                   # both "c" rows
    with pytest.raises(ValueError, match=r"^Not enough rows / columns\.$"):
        GLM().fit_by(X, y, key, null_policy="skip")
    with pytest.raises(ValueError, match=r"^Not enough rows / columns\.$"):
        GLM().fit_by(X, y, np.array([0, 0, 0, 0, 0, 0, 0, 1]))          # one row, two features
    assert captured.calls == []


def test_bad_arguments_raise_before_device_work(captured):
    from polars_ds_extension_b200.linear_models import GLM

    X, y, key = _case()
    with pytest.raises(ValueError, match="Dimension mismatch."):
        GLM().fit_by(X, y[:-1], key)
    with pytest.raises(ValueError, match="Dimension mismatch."):
        GLM().fit_by(X, y, key[:-1])
    with pytest.raises(ValueError, match="`max_iter` must be > 1."):
        GLM(max_iter=0)
    with pytest.raises(NotImplementedError):
        GLM(family="tweedie")
    assert captured.calls == []


@pytest.mark.skipif(has_gpu(), reason="checks the host entry's messages on a box without a GPU")
def test_fails_loudly_without_gpu():
    from polars_ds_extension_b200.linear_models import GLM

    X, y, key = _case()
    with pytest.raises(ValueError, match="no usable CUDA device"):
        GLM(family="poisson").fit_by(X, y, key)
    import polars_ds_extension_b200 as pds

    df = pds.Frame({"a": X[:, 0], "b": X[:, 1], "y": y, "k": np.array([1, 2, 1, 3, 2, 1, 3, 2])})
    with pytest.raises(ValueError, match="no usable CUDA device"):
        GLM(family="poisson").fit_df_by(df, ["a", "b"], "y", by="k")
