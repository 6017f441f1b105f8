"""isotonic_regression on the H100 through the plugin C ABI and the device entry, against tests/isotonic_oracle.py.

Accuracy rule: err = max|g - g_ld| / max|y| with g_ld the long-double solution; err_dev <= max(C err_scipy, FLOOR), with
err_scipy the same measure for SciPy's sequential f64 loop, C = 10 and FLOOR = 1e-12 (DESIGN §5)."""
import numpy as np
import pyarrow as pa
import pytest
from scipy.optimize import isotonic_regression as sp_iso

import polars_ds_extension_b200 as pds
from polars_ds_extension_b200 import _harness
from polars_ds_extension_b200.frame import Frame
from tests import isotonic_oracle as io

pytestmark = pytest.mark.gpu
C_RULE = 10.0
FLOOR = 1e-12
ROWS_PER_PART = 32          # k15_isotonic.cu


def _dev(y, w=None, increasing=True):
    cols = {"y": y} if w is None else {"y": y, "w": w}
    out = Frame(cols).select(pds.isotonic_regression("y", None if w is None else "w", increasing))
    out = out["pl_isotonic_regression"]
    assert out.type == pa.float64() and len(out) == len(y)
    return out.to_numpy(zero_copy_only=False)


def _weights(n, seed):
    return np.random.default_rng(seed).uniform(0.5, 2.0, n)


def _check_rule(y, w, increasing, oracle):
    g = _dev(y, w, increasing)
    ref = oracle(y, w, increasing)
    err_dev = io.rel_err(g, ref, y)
    err_sp = io.rel_err(sp_iso(y, weights=w, increasing=increasing).x, ref, y)
    assert err_dev <= max(C_RULE * err_sp, FLOOR), (err_dev, err_sp)
    d = np.diff(g)
    assert np.all(d >= 0) if increasing else np.all(d <= 0)
    return g


@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("increasing", [True, False])
@pytest.mark.parametrize("kind", io.SHAPES)
def test_accuracy_rule_20k(kind, increasing, weighted):
    n = 20_000
    y = io.shape(kind, n, 1) * (1.0 if increasing else -1.0)
    _check_rule(y, _weights(n, 2) if weighted else None, increasing, io.pava_ld)


@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("increasing", [True, False])
@pytest.mark.parametrize("kind", io.SHAPES)
def test_accuracy_rule_1m(kind, increasing, weighted):
    n = 1_000_000
    y = io.shape(kind, n, 3) * (1.0 if increasing else -1.0)
    _check_rule(y, _weights(n, 4) if weighted else None, increasing, io.blocks_ld)


@pytest.mark.parametrize("kind,weighted", [("walk", False), ("trend", True), ("drop", False)])
def test_accuracy_rule_10m(kind, weighted):
    n = 10_000_000
    y = io.shape(kind, n, 5)
    _check_rule(y, _weights(n, 6) if weighted else None, True, io.blocks_ld)


@pytest.mark.parametrize("increasing", [True, False])
@pytest.mark.parametrize("weighted", [False, True])
def test_integer_data_is_the_correctly_rounded_exact_solution(increasing, weighted):
    """Every partial sum is an exact integer in f64, so every block mean is one correctly rounded division: the output
    must equal the exact solution rounded to f64 bit for bit, which pins the block structure itself."""
    rng = np.random.default_rng(7)
    n = 5_000
    y = (np.cumsum(rng.integers(-20, 21, n)) + rng.integers(-30, 31, n)).astype(np.int64)
    w = rng.integers(1, 10, n) if weighted else None
    g = _dev(y.astype(np.float64), None if w is None else w.astype(np.float64), increasing)
    np.testing.assert_array_equal(g, io.exact_f64(y, w, increasing))


@pytest.mark.parametrize("weighted", [False, True])
def test_invariants(weighted):
    n = 300_007
    rng = np.random.default_rng(8)
    y = np.cumsum(rng.standard_normal(n))
    w = _weights(n, 9) if weighted else np.ones(n)
    g = _dev(y, w if weighted else None)
    assert np.all(np.diff(g) >= 0)
    tot = np.sum(w * y)
    assert abs(np.sum(w * g) - tot) <= 1e-12 * np.sum(np.abs(w * y))
    ys = np.sort(y)
    if weighted:                                   # a one-row block's mean is (w y) / w: y to one rounding each way
        np.testing.assert_allclose(_dev(ys, w), ys, rtol=4.5e-16, atol=0)
    else:
        np.testing.assert_array_equal(_dev(ys), ys)
    yr = ys[::-1].copy()
    mean = np.sum(w * yr) / np.sum(w)
    g = _dev(yr, w if weighted else None)
    assert np.all(g == g[0]) and abs(g[0] - mean) <= 1e-12 * np.max(np.abs(yr))


@pytest.mark.parametrize("k", [1, 2, 3, 7, 64])
@pytest.mark.parametrize("d", [-2, -1, 0, 1, 2])
def test_partition_boundaries(k, d):
    n = k * ROWS_PER_PART + d
    for kind in ("walk", "drop", "sawtooth"):
        y = io.shape(kind, n, n)
        for inc in (True, False):
            _check_rule(y, _weights(n, n) if inc else None, inc, io.pava_ld)


@pytest.mark.parametrize("n", [2, 3])
def test_smallest_inputs(n):
    for y in ([1.0, 0.0, 2.0], [3.0, 2.0, 1.0], [1.0, 2.0, 3.0], [2.0, 2.0, 1.0]):
        y = np.array(y[:n])
        for inc in (True, False):
            for w in (None, np.array([1.0, 3.0, 0.5])[:n]):
                np.testing.assert_allclose(_dev(y, w, inc), sp_iso(y, weights=w, increasing=inc).x, rtol=0, atol=1e-15)


def test_cascades():
    n = 1_000_003
    y = np.arange(n, dtype=np.float64)
    y[-1] = -1e13                                  # every block pooled across every partition and level
    g = _check_rule(y, None, True, io.blocks_ld)
    assert np.all(g == g[0])
    y = -np.arange(n, dtype=np.float64)
    y[0] = -1e13                                   # the mirror image for increasing=False
    g = _check_rule(y, None, False, io.blocks_ld)
    assert np.all(g == g[0])
    _check_rule(io.shape("sawtooth", n, 10), None, True, io.blocks_ld)
    _check_rule(io.shape("runs", n, 11), _weights(n, 12), True, io.blocks_ld)
    _check_rule(io.shape("runs", n, 11), None, False, io.blocks_ld)


def test_short_columns_pass_through():
    for vals in ([], [2.5], [None]):
        a = pa.chunked_array([pa.array(vals, type=pa.float64())])
        out = _harness.call_plugin("pl_isotonic_regression", [a], ["y"], {"has_weights": False, "increasing": True})
        assert out.type == pa.float64() and out.to_pylist() == vals
    # n <= 1 comes back before the weights are looked at
    a = pa.chunked_array([pa.array([None], type=pa.float64())])
    out = _harness.call_plugin("pl_isotonic_regression", [a, pa.chunked_array([pa.array([-1.0, 2.0])])], ["y", "w"],
                               {"has_weights": True, "increasing": False})
    assert out.to_pylist() == [None]


def test_reference_errors_in_order():
    kw = {"has_weights": True, "increasing": True}
    y = pa.chunked_array([pa.array([1.0, 0.0, 2.0, 3.0])])
    yn = pa.chunked_array([pa.array([1.0, None, 2.0, 3.0])])
    with pytest.raises(pds.PdsbError, match="Input should not contain nulls."):
        Frame({"y": yn}).select(pds.isotonic_regression("y"))
    with pytest.raises(pds.PdsbError, match="Input should not contain nulls."):
        _harness.call_plugin("pl_isotonic_regression", [yn, y.slice(1)], ["y", "w"], kw)
    with pytest.raises(pds.PdsbError, match="Weights should not contain nulls and must be the same length as y."):
        _harness.call_plugin("pl_isotonic_regression", [y, y.slice(1)], ["y", "w"], kw)
    with pytest.raises(pds.PdsbError, match="Weight should not contain nulls."):
        Frame({"y": y, "w": pa.chunked_array([pa.array([1.0, None, -2.0, 3.0])])}).select(
            pds.isotonic_regression("y", "w"))
    for bad in (0.0, -1e-300, -5.0):
        w = np.ones(100_000)
        w[77_777] = bad
        with pytest.raises(pds.PdsbError, match="Weight should not contain negative values."):
            _dev(np.arange(100_000.0), w)
    w = np.ones(4)
    w[1] = np.nan                                  # a NaN weight is no error, and gives an all-NaN result
    assert np.isnan(_dev(np.array([1.0, 0.0, 2.0, 3.0]), w)).all()
    w[2] = -1.0                                    # ... unless some weight is <= 0
    with pytest.raises(pds.PdsbError, match="Weight should not contain negative values."):
        _dev(np.array([1.0, 0.0, 2.0, 3.0]), w)
    with pytest.raises(pds.PdsbError, match="invalid series dtype: expected `Float64`"):
        _harness.call_plugin("pl_isotonic_regression", [pa.chunked_array([pa.array([1, 0, 2])])], ["y"],
                             {"has_weights": False, "increasing": True})


def test_non_finite_gives_all_nan():
    n = 50_000
    y = io.shape("walk", n, 13)
    for pos in (0, 12_345, n - 1):
        for bad in (np.nan, np.inf, -np.inf):
            yb = y.copy()
            yb[pos] = bad
            for inc in (True, False):
                assert np.isnan(_dev(yb, None, inc)).all()
            wb = np.ones(n)
            wb[pos] = bad if bad != -np.inf else np.nan
            assert np.isnan(_dev(y, wb)).all()


def test_integer_and_float32_columns_through_the_wrapper():
    n = 40_000
    yi = np.random.default_rng(14).integers(-1000, 1000, n)
    wf = _weights(n, 15).astype(np.float32)
    g = Frame({"y": yi, "w": wf}).select(pds.isotonic_regression("y", "w", increasing=False))["pl_isotonic_regression"]
    np.testing.assert_array_equal(g.to_numpy(zero_copy_only=False),
                                  _dev(yi.astype(np.float64), wf.astype(np.float64), False))


def test_chunked_and_sliced_inputs_to_the_symbol():
    n = 30_011
    y = io.shape("walk", n + 5, 16)
    w = _weights(n + 5, 17)
    ref = _dev(y[3:3 + n], w[3:3 + n])
    kw = {"has_weights": True, "increasing": True}
    yc = pa.chunked_array([pa.array(y[3:1003]), pa.array(y[1003:1004]), pa.array(y[1004:3 + n])])
    wc = pa.chunked_array([pa.array(w[3:20003]), pa.array(w[20003:3 + n])])
    g = _harness.call_plugin("pl_isotonic_regression", [yc, wc], ["y", "w"], kw)
    np.testing.assert_array_equal(g.to_numpy(zero_copy_only=False), ref)
    ys = pa.chunked_array([pa.array(y).slice(3, n)])
    ws = pa.chunked_array([pa.array(w[:n + 4]).slice(3, n)])
    g = _harness.call_plugin("pl_isotonic_regression", [ys, ws], ["y", "w"], kw)
    np.testing.assert_array_equal(g.to_numpy(zero_copy_only=False), ref)


def test_repeats_are_bit_identical():
    n = 2_000_003
    y = io.shape("walk", n, 18)
    w = _weights(n, 19)
    g = _dev(y, w)
    for _ in range(2):
        np.testing.assert_array_equal(_dev(y, w), g)


def test_device_entry_status_bits():
    import torch

    n = 123_457
    y = io.shape("trend", n, 20)
    w = _weights(n, 21)
    L = pds.lib()
    dy = torch.from_numpy(y).cuda()
    dw = torch.from_numpy(w).cuda()
    out = torch.empty(n, dtype=torch.float64, device="cuda")
    st = torch.full((1,), -1, dtype=torch.int32, device="cuda")

    def run(wp, inc=1):
        assert L.pdsb_dev_isotonic_f64(dy.data_ptr(), wp, n, inc, out.data_ptr(), st.data_ptr(), None) == 0
        torch.cuda.synchronize()
        return st.item()

    assert run(dw.data_ptr()) == 0
    np.testing.assert_array_equal(out.cpu().numpy(), _dev(y, w))
    assert run(None, 0) == 0
    np.testing.assert_array_equal(out.cpu().numpy(), _dev(y, None, False))
    dw[500] = 0.0
    assert run(dw.data_ptr()) == 1 and torch.isnan(out).all().item()
    dw[600] = float("nan")
    assert run(dw.data_ptr()) == 3
    dw[500] = 1.0
    assert run(dw.data_ptr()) == 2 and torch.isnan(out).all().item()
    assert L.pdsb_dev_isotonic_f64(dy.data_ptr(), None, 0, 1, out.data_ptr(), st.data_ptr(), None) == 0
    torch.cuda.synchronize()
    assert st.item() == 0
    assert L.pdsb_dev_isotonic_f64(dy.data_ptr(), None, -1, 1, out.data_ptr(), st.data_ptr(), None) == 1
