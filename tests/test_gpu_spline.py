"""smooth_spline on the H100 through the plugin C ABI and the device entry, against tests/spline_oracle.py.

Accuracy rule: err_dev = max|g_dev - g_ld| / max|y| <= max(C err_f64, 1e-13), with err_f64 the same measure for the
sequential f64 banded Cholesky (SciPy) and C = 10 (DESIGN §5)."""
import numpy as np
import pyarrow as pa
import pytest

import polars_ds_extension_b200 as pds
from polars_ds_extension_b200 import _harness
from polars_ds_extension_b200.frame import Frame
from tests import spline_oracle as so

pytestmark = pytest.mark.gpu
C_RULE = 10.0
ROWS_PER_PART = 32          # 16 blocks of 2 unknowns per partition (k14_spline.cu)


def _xs(n, kind, seed):
    """Mean spacing 1: evenly spaced, jittered by up to 0.3, or uniformly random (smallest gap ~ 1 / n)."""
    rng = np.random.default_rng(seed)
    if kind == "even":
        return np.arange(n, dtype=np.float64)
    if kind == "jitter":
        return np.arange(n, dtype=np.float64) + rng.uniform(-0.3, 0.3, n)
    x = np.sort(rng.uniform(0.0, float(n), n))
    assert np.all(np.diff(x) > 0)
    return x


def _ys(x, seed):
    t = x * (10.0 / max(x[-1], 1.0))
    return np.sin(t) + 0.3 * np.cos(31.0 * t) + 0.1 * np.random.default_rng(seed).standard_normal(len(x))


def _dev(x, y, lam):
    out = Frame({"x": x, "y": y}).select(pds.smooth_spline("x", "y", lam))["pl_smooth_spline"]
    assert out.type == pa.float64() and len(out) == len(x)
    return out.to_numpy(zero_copy_only=False)


def _check_rule(x, y, lam):
    g = _dev(x, y, lam)
    g_ld = so.reinsch_ld(x, y, lam)
    err_dev = so.rel_err(g, g_ld, y)
    err_f64 = so.rel_err(so.reinsch_f64(x, y, lam), g_ld, y)
    assert err_dev <= max(C_RULE * err_f64, 1e-13), (err_dev, err_f64)
    return g, err_f64


@pytest.mark.parametrize("lam", [1e-6, 1e-2, 1.0, 1e2, 1e6])
@pytest.mark.parametrize("kind", ["even", "jitter", "random"])
def test_accuracy_rule(kind, lam):
    x = _xs(20_000, kind, 1)
    _check_rule(x, _ys(x, 2), lam)


def test_accuracy_rule_tightly_spaced():
    x = _xs(200_000, "random", 3)
    _, err_f64 = _check_rule(x, _ys(x, 4), 1e2)
    assert err_f64 > 1e-5                  # smallest gap ~1.6e-6: the ill-conditioned case the rule is about


@pytest.mark.parametrize("k", [1, 3, 17])
@pytest.mark.parametrize("d", [-2, -1, 0, 1, 2])
def test_partition_boundaries(k, d):
    n = k * ROWS_PER_PART + 2 + d          # m = n - 2 unknowns around k partitions
    x = _xs(n, "jitter", n)
    y = _ys(x, n)
    for lam in (1e-2, 1e2):
        _check_rule(x, y, lam)


@pytest.mark.parametrize("n", [3, 4, 5])
def test_smallest_inputs(n):
    x = np.array([0.0, 0.7, 1.9, 2.2, 4.0])[:n]
    y = np.array([1.0, -2.0, 0.5, 3.0, 1.5])[:n]
    for lam in (1e-6, 1e-3, 1.0, 1e3):
        _check_rule(x, y, lam)
        assert so.rel_err(_dev(x, y, lam), so.dense_smooth_spline(x, y, lam), y) < 1e-10


@pytest.mark.parametrize("n", [37, 200, 500])
@pytest.mark.parametrize("kind", ["even", "jitter"])
def test_matches_the_dense_reference_form(n, kind):
    x = np.linspace(0.0, 10.0, n)
    if kind == "jitter":
        x = x + np.random.default_rng(n).uniform(-0.3, 0.3, n) * (10.0 / (n - 1))
    y = np.sin(x) + 0.1 * np.random.default_rng(n + 1).standard_normal(n)
    for lam in (1e-3, 1e-1, 10.0, 100.0):
        assert so.rel_err(_dev(x, y, lam), so.dense_smooth_spline(x, y, lam), y) < 1e-8


def test_lambda_zero_is_y_bit_exact():
    x = _xs(10_001, "random", 5)
    y = _ys(x, 6)
    y[17] = np.nan                          # I g = y: the input comes back as it is
    g = _dev(x, y, 0.0)
    np.testing.assert_array_equal(g, y)
    with pytest.raises(pds.PdsbError, match="Input is not increasing."):
        _dev(np.array([0.0, 1.0, 1.0, 2.0]), np.ones(4), 0.0)


@pytest.mark.parametrize("lam", [1e-6, 1.0, 1e6])
def test_linear_data_is_reproduced(lam):
    x = _xs(100_003, "jitter", 7)
    y = 2.5 - 0.75 * x
    assert so.rel_err(_dev(x, y, lam), y, y) < 1e-11


def test_one_million_rows_and_bit_identical_repeats():
    x = _xs(1_000_000, "jitter", 8)
    y = _ys(x, 9)
    g, _ = _check_rule(x, y, 1.0)
    np.testing.assert_array_equal(_dev(x, y, 1.0), g)
    np.testing.assert_array_equal(_dev(x, y, 1.0), g)


def test_ten_million_rows_against_the_f64_baseline():
    x6 = _xs(1_000_000, "jitter", 10)
    y6 = _ys(x6, 11)
    err_f64_6 = so.rel_err(so.reinsch_f64(x6, y6, 1e2), so.reinsch_ld(x6, y6, 1e2), y6)
    x = _xs(10_000_000, "jitter", 12)
    y = _ys(x, 13)
    err = so.rel_err(_dev(x, y, 1e2), so.reinsch_f64(x, y, 1e2), y)
    assert err <= max(C_RULE * err_f64_6, 1e-13), (err, err_f64_6)


def test_reference_errors():
    x = np.linspace(0.0, 1.0, 10)
    y = np.arange(10.0)
    for cols in ({"x": pa.array(x, mask=np.arange(10) == 4), "y": y},
                 {"x": x, "y": pa.array(y, mask=np.arange(10) == 9)}):
        with pytest.raises(pds.PdsbError, match="Input x or y has nulls."):
            Frame(cols).select(pds.smooth_spline("x", "y", 1.0))
    with pytest.raises(pds.PdsbError, match="Must have >= 3 points."):
        _dev(x[:2], y[:2], 1.0)
    with pytest.raises(pds.PdsbError, match="Input is not increasing."):
        _dev(np.array([0.0, 1.0, 1.0, 2.0, 3.0]), y[:5], 1.0)
    xd = x.copy()
    xd[6] = xd[5] - 0.01
    with pytest.raises(pds.PdsbError, match="Input is not increasing."):
        _dev(xd, y, 1.0)
    xl = np.linspace(0.0, 1.0, 100_000)
    xl[-1] = xl[-2]                         # the last gap, in the last partition
    with pytest.raises(pds.PdsbError, match="Input is not increasing."):
        _dev(xl, np.ones(len(xl)), 1.0)
    a = pa.chunked_array([pa.array(x)])
    with pytest.raises(pds.PdsbError, match="Input lengths are not the same."):
        _harness.call_plugin("pl_smooth_spline", [a, a.slice(1)], ["x", "y"], {"lambda": 1.0})
    # a nulls error comes before the lengths error (the reference's order)
    with pytest.raises(pds.PdsbError, match="Input x or y has nulls."):
        _harness.call_plugin("pl_smooth_spline", [pa.chunked_array([pa.array([0.0, None, 2.0])]), a],
                             ["x", "y"], {"lambda": 1.0})
    with pytest.raises(pds.PdsbError, match="must be nonnegative"):
        _harness.call_plugin("pl_smooth_spline", [a, a], ["x", "y"], {"lambda": -1.0})


def test_non_finite_inputs_give_all_nan():
    """NaN / inf y and NaN x: all NaN, as the dense form gives.  An infinite x at an end: all NaN, where the dense form
    gives finite values (DESIGN §5)."""
    n = 5_000
    x = _xs(n, "jitter", 14)
    y = _ys(x, 15)
    for lam in (1e-3, 1.0):
        for bad in (np.nan, np.inf, -np.inf):
            yb = y.copy()
            yb[1234] = bad
            assert np.isnan(_dev(x, yb, lam)).all()
        for pos, bad in ((1234, np.nan), (0, np.nan), (n - 1, np.inf), (0, -np.inf)):
            xb = x.copy()
            xb[pos] = bad
            assert np.isnan(_dev(xb, y, lam)).all()


def test_integer_and_float32_columns_through_the_wrapper():
    x = np.arange(0, 3 * 5_000, 3, dtype=np.int64)
    y = _ys(x.astype(np.float64) / 1000.0, 16).astype(np.float32)
    g = Frame({"x": x, "y": y}).select(pds.smooth_spline("x", "y", 1e3))["pl_smooth_spline"]
    g = g.to_numpy(zero_copy_only=False)
    np.testing.assert_array_equal(g, _dev(x.astype(np.float64), y.astype(np.float64), 1e3))
    a = pa.chunked_array([pa.array(x)])
    with pytest.raises(pds.PdsbError, match="invalid series dtype: expected `Float64`"):
        _harness.call_plugin("pl_smooth_spline", [a, pa.chunked_array([pa.array(y.astype(np.float64))])],
                             ["x", "y"], {"lambda": 1.0})
    with pytest.raises(pds.PdsbError, match="invalid series dtype: expected `Float64`"):
        _harness.call_plugin("pl_smooth_spline", [pa.chunked_array([pa.array(x.astype(np.float64))]),
                                                  pa.chunked_array([pa.array(y)])], ["x", "y"], {"lambda": 1.0})


def test_chunked_and_sliced_inputs_to_the_symbol():
    n = 30_011
    x = _xs(n + 5, "jitter", 17)
    y = _ys(x, 18)
    ref = _dev(x[3:3 + n], y[3:3 + n], 0.5)
    xc = pa.chunked_array([pa.array(x[3:1003]), pa.array(x[1003:1004]), pa.array(x[1004:3 + n])])
    yc = pa.chunked_array([pa.array(y[3:20003]), pa.array(y[20003:3 + n])])
    g = _harness.call_plugin("pl_smooth_spline", [xc, yc], ["x", "y"], {"lambda": 0.5})
    np.testing.assert_array_equal(g.to_numpy(zero_copy_only=False), ref)
    xs = pa.chunked_array([pa.array(x).slice(3, n)])
    ys = pa.chunked_array([pa.array(y[:n + 4]).slice(3, n)])
    g = _harness.call_plugin("pl_smooth_spline", [xs, ys], ["x", "y"], {"lambda": 0.5})
    np.testing.assert_array_equal(g.to_numpy(zero_copy_only=False), ref)


def test_device_entry_matches_the_plugin_path():
    import torch

    n = 123_457
    x = _xs(n, "random", 19)
    y = _ys(x, 20)
    L = pds.lib()
    dx = torch.from_numpy(x).cuda()
    dy = torch.from_numpy(y).cuda()
    g = torch.empty(n, dtype=torch.float64, device="cuda")
    st = torch.full((1,), -1, dtype=torch.int32, device="cuda")
    assert L.pdsb_dev_smooth_spline_f64(dx.data_ptr(), dy.data_ptr(), n, 10.0, g.data_ptr(), st.data_ptr(), None) == 0
    torch.cuda.synchronize()
    assert st.item() == 0
    np.testing.assert_array_equal(g.cpu().numpy(), _dev(x, y, 10.0))
    dx[500] = dx[499]
    assert L.pdsb_dev_smooth_spline_f64(dx.data_ptr(), dy.data_ptr(), n, 10.0, g.data_ptr(), st.data_ptr(), None) == 0
    torch.cuda.synchronize()
    assert st.item() == 1 and torch.isnan(g).all().item()
    assert L.pdsb_dev_smooth_spline_f64(dx.data_ptr(), dy.data_ptr(), 2, 10.0, g.data_ptr(), st.data_ptr(), None) == 1
