"""isotonic_regression(...).over(key) on the H100: pl_isotonic_regression_by and pdsb_dev_grouped_isotonic_f64 against
Polars' per-group loop, the single-column entries and tests/isotonic_oracle.py.

The contract: group g is rows [offsets[g], offsets[g+1]) in key order, and its output is bit for bit what
pl_isotonic_regression returns on that group's rows alone (value, validity and the all-NaN rule), so the fast path
equals the loop exactly and no group depends on another group's rows.  Accuracy rule per group as in
test_gpu_isotonic.py: err <= max(C err_scipy, FLOOR), C = 10, FLOOR = 1e-12."""
import ctypes as C
import zlib

import numpy as np
import pyarrow as pa
import pytest
from scipy.optimize import isotonic_regression as sp_iso

import polars_ds_extension_b200 as pds
from polars_ds_extension_b200 import _harness
from polars_ds_extension_b200._lib import check
from polars_ds_extension_b200.frame import Frame
from tests import isotonic_oracle as io
from tests.helpers import group_offsets

pytestmark = pytest.mark.gpu
C_RULE = 10.0
FLOOR = 1e-12
SIZES = [1, 2, 3, 31, 32, 33, 63, 64, 65, 1000, 1023, 1024, 1025] + \
    [32 * 2 ** k + d for k in (2, 3, 5, 6) for d in (-1, 1)] + [20_000]


def _ca(v):
    if isinstance(v, pa.ChunkedArray):
        return v
    if isinstance(v, pa.Array):
        return pa.chunked_array([v])
    return pa.chunked_array([pa.array(np.asarray(v, dtype=np.float64))])


def _by(y, w, offsets, inc=True, offsets_type=pa.int64()):
    """pl_isotonic_regression_by on rows already in group order."""
    ins = [pa.chunked_array([pa.array(np.asarray(offsets), type=offsets_type)]), _ca(y)] + ([_ca(w)] if w is not None else [])
    names = ["__offsets__", "y"] + (["w"] if w is not None else [])
    return _harness.call_plugin("pl_isotonic_regression_by", ins, names, {"has_weights": w is not None, "increasing": inc})


def _one(y, w, inc=True):
    ins = [_ca(y)] + ([_ca(w)] if w is not None else [])
    names = ["y"] + (["w"] if w is not None else [])
    return _harness.call_plugin("pl_isotonic_regression", ins, names, {"has_weights": w is not None, "increasing": inc})


def _loop(y, w, offsets, inc=True):
    """pl_isotonic_regression once per group, concatenated (what Polars' loop returns in key order)."""
    y, w = _ca(y), None if w is None else _ca(w)
    parts = [_one(y.slice(a, b - a), None if w is None else w.slice(a, b - a), inc)
             for a, b in zip(offsets[:-1], offsets[1:])]
    return pa.concat_arrays([p if isinstance(p, pa.Array) else p.combine_chunks() for p in parts])


def _np(a):
    return a.to_numpy(zero_copy_only=False)


def _weights(n, seed):
    return np.random.default_rng(seed).uniform(0.5, 2.0, n)


def _group_data(kind, sizes, seed, inc=True):
    """Each group its own column of the shape, so each group has the shape's structure."""
    return np.concatenate([io.shape(kind, s, seed + i) for i, s in enumerate(sizes)]) * (1.0 if inc else -1.0)


# 1. fast == loop on a frame with interleaved keys ------------------------------------------------------------------
@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("increasing", [True, False])
@pytest.mark.parametrize("kind", io.SHAPES)
def test_fast_over_equals_the_loop(kind, increasing, weighted):
    rng = np.random.default_rng(zlib.crc32(f"{kind}{increasing}{weighted}".encode()))
    sizes = list(SIZES)
    y = _group_data(kind, sizes, 100, increasing)
    keys = np.repeat(np.arange(len(sizes)) * 7 + 3, sizes)
    perm = rng.permutation(len(y))                     # keys interleaved; each group keeps its rows' relative order
    perm = np.concatenate([np.sort(perm[keys[perm] == k]) for k in np.unique(keys)])
    yf, kf = np.empty_like(y), np.empty_like(keys)
    yf[perm], kf[perm] = y, keys
    cols = {"y": yf, "g": kf}
    if weighted:
        cols["w"] = _weights(len(y), 1)
    df = Frame(cols)
    e = pds.isotonic_regression("y", "w" if weighted else None, increasing)
    fast, loop = (df.select(e.over("g", fast=f))["pl_isotonic_regression"] for f in (True, False))
    assert fast.type == pa.float64() and len(fast) == len(y)
    np.testing.assert_array_equal(_np(fast), _np(loop))


# 2. device entry per group == pdsb_dev_isotonic_f64 on the group's rows, status included -----------------------------
def _dev_grouped(y, w, offsets, inc=1, reps=1):
    import torch

    L = pds.lib()
    dy = torch.from_numpy(np.ascontiguousarray(y)).cuda()
    dw = None if w is None else torch.from_numpy(np.ascontiguousarray(w)).cuda()
    doff = torch.from_numpy(np.asarray(offsets, dtype=np.int64)).cuda()
    G = len(offsets) - 1
    outs = []
    for _ in range(reps):
        out = torch.full((len(y),), 7.0, dtype=torch.float64, device="cuda")
        st = torch.full((G,), -1, dtype=torch.int32, device="cuda")
        check(L.pdsb_dev_grouped_isotonic_f64(dy.data_ptr(), None if dw is None else dw.data_ptr(), doff.data_ptr(),
                                              G, len(y), inc, out.data_ptr(), st.data_ptr(), None))
        torch.cuda.synchronize()
        outs.append((out.cpu().numpy(), st.cpu().numpy()))
    return outs if reps > 1 else outs[0]


def _dev_single(y, w, inc=1):
    import torch

    L = pds.lib()
    n = len(y)
    dy = torch.from_numpy(np.ascontiguousarray(y)).cuda()
    dw = None if w is None else torch.from_numpy(np.ascontiguousarray(w)).cuda()
    out = torch.empty(max(n, 1), dtype=torch.float64, device="cuda")
    st = torch.full((1,), -1, dtype=torch.int32, device="cuda")
    assert L.pdsb_dev_isotonic_f64(dy.data_ptr(), None if dw is None else dw.data_ptr(), n, inc, out.data_ptr(),
                                   st.data_ptr(), None) == 0
    torch.cuda.synchronize()
    return out.cpu().numpy()[:n], int(st.item())


@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("inc", [1, 0])
def test_device_entry_equals_the_single_entry_per_group(weighted, inc):
    sizes = [0] + SIZES + [0, 0, 5, 40, 1, 0]
    offsets = group_offsets(sizes)
    y = _group_data("walk", sizes, 200)
    w = _weights(len(y), 2) if weighted else None
    # group 3 a NaN y, group 10 an inf y; with weights, group 5 a w <= 0 and group 11 a NaN w and a w <= 0
    y[offsets[3] + 1] = np.nan
    y[offsets[10] + 500] = np.inf
    if weighted:
        w[offsets[5] + 10] = 0.0
        w[offsets[11]] = np.nan
        w[offsets[11] + 7] = -1.0
    out, st = _dev_grouped(y, w, offsets, inc)
    for g, (a, b) in enumerate(zip(offsets[:-1], offsets[1:])):
        if a == b:
            assert st[g] == 0
            continue
        ref, rst = _dev_single(y[a:b], None if w is None else w[a:b], inc)
        np.testing.assert_array_equal(out[a:b], ref, err_msg=f"group {g}")
        assert st[g] == rst, (g, st[g], rst)
    assert st[3] == 2 and st[10] == 2
    if weighted:
        assert st[5] == 1 and st[11] == 3


# 3. accuracy rule per group; 4. integer data is the correctly rounded exact solution ---------------------------------
@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("kind", ["walk", "trend", "sawtooth", "runs"])
def test_accuracy_rule_per_group(kind, weighted):
    sizes = [s for s in SIZES if s >= 2]
    offsets = group_offsets(sizes)
    y = _group_data(kind, sizes, 300)
    w = _weights(len(y), 3) if weighted else None
    g = _np(_by(y, w, offsets))
    for a, b in zip(offsets[:-1], offsets[1:]):
        ys, ws = y[a:b], None if w is None else w[a:b]
        ref = io.pava_ld(ys, ws)
        err_dev = io.rel_err(g[a:b], ref, ys)
        err_sp = io.rel_err(sp_iso(ys, weights=ws).x, ref, ys)
        assert err_dev <= max(C_RULE * err_sp, FLOOR), (b - a, err_dev, err_sp)
        assert np.all(np.diff(g[a:b]) >= 0)


@pytest.mark.parametrize("increasing", [True, False])
@pytest.mark.parametrize("weighted", [False, True])
def test_integer_data_is_the_exact_solution_per_group(increasing, weighted):
    rng = np.random.default_rng(7)
    sizes = [2, 3, 31, 32, 33, 65, 1000, 1025, 3000]
    offsets = group_offsets(sizes)
    y = (np.cumsum(rng.integers(-20, 21, offsets[-1])) + rng.integers(-30, 31, offsets[-1])).astype(np.int64)
    w = rng.integers(1, 10, offsets[-1]) if weighted else None
    g = _np(_by(y.astype(np.float64), None if w is None else w.astype(np.float64), offsets, increasing))
    for a, b in zip(offsets[:-1], offsets[1:]):
        np.testing.assert_array_equal(g[a:b], io.exact_f64(y[a:b], None if w is None else w[a:b], increasing))


# 5. independence -----------------------------------------------------------------------------------------------------
def test_one_group_does_not_reach_the_others():
    sizes = [33, 1025, 1, 4097, 20_000, 2, 64]
    offsets = group_offsets(sizes)
    y = _group_data("walk", sizes, 400)
    w = _weights(len(y), 4)
    base = _np(_by(y, w, offsets))
    for k in (1, 3, 4):
        a, b = offsets[k], offsets[k + 1]
        others = np.ones(len(y), dtype=bool)
        others[a:b] = False
        ys = y.copy()
        ys[a:b] *= 1e12
        g = _np(_by(ys, w, offsets))
        np.testing.assert_array_equal(g[others], base[others])
        for bad in (np.nan, np.inf, -np.inf):
            yb = y.copy()
            yb[a + (b - a) // 2] = bad
            g = _np(_by(yb, w, offsets))
            np.testing.assert_array_equal(g[others], base[others])
            assert np.isnan(g[a:b]).all()
        wb = w.copy()
        wb[b - 1] = np.nan
        g = _np(_by(y, wb, offsets))
        np.testing.assert_array_equal(g[others], base[others])
        assert np.isnan(g[a:b]).all()


def test_one_row_groups_pass_through():
    # groups: [3 rows], [null y], [NaN y], [y, w <= 0], [y, null w], [y, w = -inf], [2 rows]
    y = pa.array([3.0, 1.0, 2.0, None, np.nan, 5.5, 6.5, 7.5, 4.0, 1.0], type=pa.float64())
    w = pa.array([1.0, 2.0, 1.0, 1.0, 1.0, -2.0, None, -np.inf, 1.0, 3.0], type=pa.float64())
    offsets = [0, 3, 4, 5, 6, 7, 8, 10]
    out = _by(y, w, offsets)
    loop = _loop(y, w, offsets)
    vals = out.to_pylist()
    assert vals[3] is None and np.isnan(vals[4]) and vals[5:8] == [5.5, 6.5, 7.5]
    assert out.null_count == 1 and out.is_valid().to_pylist() == loop.is_valid().to_pylist()
    np.testing.assert_array_equal(_np(out.fill_null(-1.0)), _np(loop.fill_null(-1.0)))
    unweighted = _by(y, None, offsets)
    assert unweighted.to_pylist()[3] is None and unweighted.to_pylist()[5:8] == [5.5, 6.5, 7.5]


# 6. errors -----------------------------------------------------------------------------------------------------------
def test_reference_errors_from_groups_of_two_or_more_rows():
    offsets = [0, 1, 4, 6]
    y = pa.array([None, 1.0, 0.0, 2.0, 3.0, 1.0], type=pa.float64())
    w = pa.array([-1.0, 1.0, 1.0, 1.0, 1.0, 1.0], type=pa.float64())
    _by(y, w, offsets)                                  # the null y and the w <= 0 are in a one-row group: no error
    yn = pa.array([1.0, 1.0, None, 2.0, 3.0, 1.0], type=pa.float64())
    with pytest.raises(pds.PdsbError, match="Input should not contain nulls."):
        _by(yn, None, offsets)
    wn = pa.array([1.0, 1.0, 1.0, 1.0, None, 1.0], type=pa.float64())
    with pytest.raises(pds.PdsbError, match="Weight should not contain nulls."):
        _by(y.fill_null(0.0), wn, offsets)
    for bad in (0.0, -1e-300, -5.0):
        wb = pa.array([1.0, 1.0, 1.0, bad, 1.0, 1.0], type=pa.float64())
        with pytest.raises(pds.PdsbError, match="Weight should not contain negative values."):
            _by(y.fill_null(0.0), wb, offsets)


def test_check_order_across_groups():
    offsets = [0, 3, 6, 9]
    # group 0: w <= 0; group 1: null w; group 2: null y -> the null y is reported first
    y = pa.array([1.0, 0.0, 2.0, 1.0, 0.0, 2.0, 1.0, None, 2.0], type=pa.float64())
    w = pa.array([1.0, -1.0, 1.0, 1.0, None, 1.0, 1.0, 1.0, 1.0], type=pa.float64())
    with pytest.raises(pds.PdsbError, match="Input should not contain nulls."):
        _by(y, w, offsets)
    # without the null y: the null w (group 1) comes before the w <= 0 (group 0)
    with pytest.raises(pds.PdsbError, match="Weight should not contain nulls."):
        _by(y.fill_null(0.0), w, offsets)
    # the loop stops at group 0 with the w <= 0 message (the deviation DESIGN §5 records)
    with pytest.raises(pds.PdsbError, match="Weight should not contain negative values."):
        _loop(y.fill_null(0.0), w, offsets)


def test_bad_offsets_are_refused():
    y = np.arange(10.0)
    for offs in ([0, 6, 4, 10], [0, 5, 9], [0, 5, 11], [1, 5, 10]):
        with pytest.raises(pds.PdsbError, match="grouped isotonic_regression: (bad group offsets|group offsets must be)"):
            _by(y, None, offs)
    with pytest.raises(pds.PdsbError, match="offsets must be one non-null Int64 chunk"):
        _by(y, None, [0, 5, 10], offsets_type=pa.int32())


# 7. one group == pl_isotonic_regression ------------------------------------------------------------------------------
@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("kind", io.SHAPES)
def test_one_group_equals_the_single_call(kind, weighted):
    n = 100_003
    y = io.shape(kind, n, 500)
    w = _weights(n, 5) if weighted else None
    for inc in (True, False):
        np.testing.assert_array_equal(_np(_by(y, w, [0, n], inc)), _np(_one(y, w, inc)))


# 8. large shapes, within the stated scratch bound --------------------------------------------------------------------
class _Pool:
    """High-water mark of the device's default memory pool (where the library's stream-ordered scratch comes from; the
    test's own tensors come from PyTorch's allocator)."""
    USED_MEM_HIGH = 8                                  # CU_MEMPOOL_ATTR_USED_MEM_HIGH

    def __init__(self):
        import torch

        self.cu = C.CDLL("libcuda.so.1")
        dev = C.c_int()
        assert self.cu.cuDeviceGet(C.byref(dev), torch.cuda.current_device()) == 0
        self.pool = C.c_void_p()
        assert self.cu.cuDeviceGetDefaultMemPool(C.byref(self.pool), dev) == 0

    def reset(self):
        z = C.c_uint64(0)
        assert self.cu.cuMemPoolSetAttribute(self.pool, self.USED_MEM_HIGH, C.byref(z)) == 0

    def high(self):
        v = C.c_uint64(0)
        assert self.cu.cuMemPoolGetAttribute(self.pool, self.USED_MEM_HIGH, C.byref(v)) == 0
        return v.value


def _scratch_bound(offsets):
    """pdsb.h: about 25 n + 140 P + 80 n_groups bytes, P = the groups' partitions of 32 rows."""
    sizes = np.diff(offsets)
    P = int(np.sum((sizes + 31) // 32))
    return 25 * int(offsets[-1]) + 140 * P + 80 * len(sizes) + (16 << 20)


def _run_large(y, offsets, sample_groups):
    pool = _Pool()
    pool.reset()
    out, st = _dev_grouped(y, None, offsets)
    used = pool.high()
    assert used <= _scratch_bound(offsets), (used, _scratch_bound(offsets))
    assert (st == 0).all()
    for g in sample_groups:
        a, b = offsets[g], offsets[g + 1]
        ref, _ = _dev_single(y[a:b], None)
        np.testing.assert_array_equal(out[a:b], ref, err_msg=f"group {g}")
    d = np.diff(out) >= 0
    d[offsets[1:-1] - 1] = True                        # no order across a group boundary
    assert d.all()
    return out


@pytest.mark.parametrize("big", [False, True])
def test_a_million_groups_of_100(big):
    sizes = np.full(1_000_000, 100, dtype=np.int64)
    if big:
        sizes = np.concatenate([sizes[:500_000], [10_000_000], sizes[500_000:]])
    offsets = group_offsets(sizes)
    rng = np.random.default_rng(8)
    y = np.cumsum(rng.standard_normal(int(offsets[-1])))
    sample = list(rng.choice(len(sizes), 100, replace=False)) + [0, len(sizes) - 1] + ([500_000] if big else [])
    _run_large(y, offsets, sample)


def test_ten_million_one_row_groups():
    n = 10_000_000
    y = np.random.default_rng(9).standard_normal(n)
    out = _run_large(y, np.arange(n + 1, dtype=np.int64), [0, 12_345, n - 1])
    np.testing.assert_array_equal(out, y)


# 9. chunked and sliced inputs; 10. repeats ---------------------------------------------------------------------------
def test_chunked_and_sliced_inputs():
    sizes = [1, 33, 1000, 2, 20_000, 65]
    offsets = group_offsets(sizes)
    n = int(offsets[-1])
    y = io.shape("walk", n + 5, 16)
    w = _weights(n + 5, 17)
    ref = _np(_by(y[3:3 + n], w[3:3 + n], offsets))
    yc = pa.chunked_array([pa.array(y[3:40]), pa.array(y[40:41]), pa.array(y[41:3 + n])])
    wc = pa.chunked_array([pa.array(w[3:20003]), pa.array(w[20003:3 + n])])
    np.testing.assert_array_equal(_np(_by(yc, wc, offsets)), ref)
    ys = pa.chunked_array([pa.array(y).slice(3, n)])
    ws = pa.chunked_array([pa.array(w[:n + 4]).slice(3, n)])
    np.testing.assert_array_equal(_np(_by(ys, ws, offsets)), ref)


def test_repeats_are_bit_identical():
    rng = np.random.default_rng(18)
    sizes = rng.integers(1, 5000, 2000)
    offsets = group_offsets(sizes)
    y = np.cumsum(rng.standard_normal(int(offsets[-1])))
    w = _weights(len(y), 19)
    runs = _dev_grouped(y, w, offsets, reps=3)
    for out, st in runs[1:]:
        np.testing.assert_array_equal(out, runs[0][0])
        np.testing.assert_array_equal(st, runs[0][1])
