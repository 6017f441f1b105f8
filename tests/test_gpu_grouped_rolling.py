"""rolling_lin_reg over groups on the H100: pdsb_dev_grouped_rolling_lin_reg_* against pdsb_dev_online_lin_reg_* on each
group's rows, and pdsb_host_grouped_rolling against pdsb_host_online(rolling = 1) on each group's rows.

The contract: group g is rows [offsets[g], offsets[g+1]) in key order, and its coefficients, pred and validity are bit
for bit what the single call returns on that group's rows alone, on every pass-C route, in calls whose groups need two
different plans, and independently of every other group's rows."""
import ctypes as C
import zlib

import numpy as np
import pyarrow as pa
import pytest

from polars_ds_extension_b200._lib import Column, HostResult, LrKwargs, PdsbError, check, lib
from tests.helpers import group_offsets

pytestmark = pytest.mark.gpu

PACKED, LANE, GENERIC = 1, 2, 3
WINDOWS = [2, 63, 64, 511, 512, 1023, 1024, 1025, 3000]


def _data(n, p, f64, seed, nan_rows=0):
    rng = np.random.default_rng(seed)
    dt = np.float64 if f64 else np.float32
    X = rng.standard_normal((n, p)).astype(dt)
    y = (X.astype(np.float64) @ (np.arange(p) % 5 - 2.0) + 0.5 + 0.1 * rng.standard_normal(n)).astype(dt)
    if nan_rows:
        X[rng.choice(n, nan_rows, replace=False), rng.integers(0, p)] = np.nan
        y[rng.choice(n, nan_rows, replace=False)] = np.nan
    return X, y


def _route():
    return int(lib().pdsb_last_online_path())


def _expected_route(f64, q, window, skip):
    if q > 12:
        return GENERIC
    return PACKED if (not f64 and q <= 9 and window >= 64 and not skip) else LANE


def _iview(t):
    import torch

    return t.reshape(-1).view(torch.int64 if t.dtype == torch.float64 else torch.int32)


def _dev(X, y, off, window, min_rows, bias, lam, skip):
    """(grouped outputs, the device tensors) for host arrays X (n, p), y, offsets and per-group skip flags."""
    import torch
    from polars_ds_extension_b200 import device as dev

    Xd = torch.from_numpy(np.ascontiguousarray(X.T)).cuda()
    yd = torch.from_numpy(np.ascontiguousarray(y)).cuda()
    sk = None if skip is None else torch.tensor(np.asarray(skip, dtype=np.uint8), device="cuda")
    out = dev.grouped_rolling_lin_reg(Xd, yd, torch.from_numpy(np.asarray(off, dtype=np.int64)).cuda(), window, min_rows,
                                      add_bias=bias, l2_reg=lam, skip=sk)
    torch.cuda.synchronize()
    return out, Xd, yd


def _single(Xd, yd, a, b, window, min_rows, bias, lam, skip):
    import torch
    from polars_ds_extension_b200 import device as dev

    out = dev.online_lin_reg(Xd[:, a:b].contiguous(), yd[a:b].contiguous(), window, min_rows, add_bias=bias, l2_reg=lam,
                             skip=bool(skip))
    torch.cuda.synchronize()
    return out


def _same_as_single(grouped, Xd, yd, off, window, min_rows, bias, lam, skip, groups=None):
    import torch

    co, pr, va = grouped
    for g in (range(len(off) - 1) if groups is None else groups):
        a, b = int(off[g]), int(off[g + 1])
        if b == a:
            continue
        sg = 0 if skip is None else int(skip[g])
        c1, p1, v1 = _single(Xd, yd, a, b, window, min_rows, bias, lam, sg)
        assert torch.equal(v1, va[a:b]), (g, "valid")
        assert torch.equal(_iview(c1), _iview(co[a:b])), (g, "coeffs")
        assert torch.equal(_iview(p1), _iview(pr[a:b])), (g, "pred")


def _sizes(window):
    return [max(1, window - 1), window, window + 1, 1023, 1024, 1025, 2047, 2048, 2049]


# 1. every pass-C route: the device entry equals the single entry per group, and the route is the single call's ---------
# (f64, p, bias, every group skips)
CONFIGS = [(False, 8, True, False), (False, 3, True, True), (False, 10, True, False), (True, 3, True, False),
           (True, 2, False, True), (False, 13, False, False), (True, 13, True, True)]


@pytest.mark.parametrize("lam", [0.0, 0.5])
@pytest.mark.parametrize("window", WINDOWS)
@pytest.mark.parametrize("f64,p,bias,skip_all", CONFIGS)
def test_device_entry_equals_the_single_entry_on_every_route(f64, p, bias, skip_all, window, lam):
    q = p + int(bias)
    sizes = _sizes(window)
    off = group_offsets(sizes)
    X, y = _data(int(off[-1]), p, f64, seed=zlib.crc32(f"{f64}{p}{window}".encode()), nan_rows=40 if skip_all else 0)
    skip = [1] * len(sizes) if skip_all else None
    min_rows = q + 1 if skip_all else 0
    grouped, Xd, yd = _dev(X, y, off, window, min_rows, bias, lam, skip)
    assert _route() == _expected_route(f64, q, window, skip_all)
    _same_as_single(grouped, Xd, yd, off, window, min_rows, bias, lam, skip)
    if sizes[0] < window:                               # the group shorter than the window has no valid row
        assert int(grouped[2][: off[1]].sum()) == 0


# 2. two plans in one call: every row of the class table ------------------------------------------------------------------
# (p with a bias, window, the no-skip class's route)
TABLE = [(8, 256, PACKED), (8, 600, PACKED), (8, 1500, PACKED), (11, 1500, LANE)]


@pytest.mark.parametrize("p,window,ns_route", TABLE)
def test_mixed_skip_classes_run_both_plans(p, window, ns_route):
    q = p + 1
    sizes = [window + 3, 3 * 1024 + 17, 1024, 2 * window + 1, 5000, window - 1, 4097, 1500]
    off = group_offsets(sizes)
    X, y = _data(int(off[-1]), p, False, seed=window + p, nan_rows=60)
    skip = [g % 2 for g in range(len(sizes))]
    grouped, Xd, yd = _dev(X, y, off, window, q, True, 0.25, skip)
    assert _route() == LANE                              # the skip class's pass C, launched last
    # the single calls of the no-skip groups take the other kernel, so both ran
    _single(Xd, yd, int(off[0]), int(off[1]), window, q, True, 0.25, 0)
    assert _route() == ns_route
    _same_as_single(grouped, Xd, yd, off, window, q, True, 0.25, skip)


@pytest.mark.parametrize("present", [0, 1])
def test_one_class_present_runs_its_own_plan(present):
    sizes = [700, 1500, 2100]
    off = group_offsets(sizes)
    X, y = _data(int(off[-1]), 8, False, seed=6, nan_rows=20)
    skip = [present] * len(sizes)
    grouped, Xd, yd = _dev(X, y, off, 256, 10, True, 0.0, skip)
    assert _route() == (LANE if present else PACKED)
    _same_as_single(grouped, Xd, yd, off, 256, 10, True, 0.0, skip)


# 3. the host entry against pdsb_host_online(rolling = 1) per group -------------------------------------------------------
def _host_call(cols, kw, f32, offsets=None):
    """(coeffs, pred, valid) numpy arrays of pdsb_host_online (offsets None) or pdsb_host_grouped_rolling."""
    from polars_ds_extension_b200 import device as dev

    L = lib()
    keep: list = []
    cc = (Column * len(cols))(*[dev._column(c, None, False, keep) for c in cols])
    k = LrKwargs(bias=int(kw["bias"]), null_policy=kw["null_policy"].encode(), n=kw["n"], lambda_=kw["lambda"],
                 min_size=kw["min_size"])
    r = HostResult()
    if offsets is None:
        check(L.pdsb_host_online(cc, len(cols), C.byref(k), int(f32), 1, C.byref(r)))
    else:
        off = (C.c_int64 * len(offsets))(*[int(v) for v in offsets])
        check(L.pdsb_host_grouped_rolling(cc, len(cols), off, len(offsets) - 1, C.byref(k), int(f32), C.byref(r)))
    try:
        it = np.uint32 if r.is_f32 else np.uint64
        n, q = r.n_rows, r.n_coef
        co = np.ctypeslib.as_array(C.cast(r.coeffs, C.POINTER(C.c_uint32 if r.is_f32 else C.c_uint64)), (n * q,)).copy()
        pr = np.ctypeslib.as_array(C.cast(r.pred, C.POINTER(C.c_uint32 if r.is_f32 else C.c_uint64)), (n,)).copy()
        va = (np.ones(n, dtype=np.uint8) if not r.valid else
              np.ctypeslib.as_array(C.cast(r.valid, C.POINTER(C.c_uint8)), (n,)).copy())
        return co.view(it), pr.view(it), va
    finally:
        L.pdsb_host_result_free(C.byref(r))


def _cols(X, y, null_y=None, null_x=None):
    return [pa.chunked_array([pa.array(y, mask=null_y)])] + [
        pa.chunked_array([pa.array(X[:, j], mask=null_x if j == 0 else None)]) for j in range(X.shape[1])]


def _loop(cols, off, kw, f32):
    parts = [_host_call([c.slice(a, b - a) for c in cols], kw, f32) for a, b in zip(off[:-1], off[1:])]
    return tuple(np.concatenate([pt[i] for pt in parts]) for i in range(3))


def _kw(window, bias, lam=0.0, policy="raise", min_size=0):
    return {"null_policy": policy, "n": int(window), "bias": bool(bias), "lambda": float(lam), "min_size": int(min_size)}


@pytest.mark.parametrize("policy,where", [("raise", "none"), ("skip", "both"), ("skip", "x"), ("zero", "y"),
                                          ("one", "x"), ("2.5", "both"), ("ignore", "both"), ("ignore", "nan")])
@pytest.mark.parametrize("f32,p,bias", [(True, 3, True), (True, 8, True), (False, 4, True), (True, 13, False)])
def test_host_entry_equals_the_single_host_call_per_group(f32, p, bias, policy, where):
    sizes = [300, 1100, 64 + 7, 2050, 500, 1500]
    off = group_offsets(sizes)
    n = int(off[-1])
    rng = np.random.default_rng(zlib.crc32(f"{policy}{where}{p}".encode()))
    X, y = _data(n, p, not f32, seed=p, nan_rows=40 if where == "nan" else 0)
    null_y = np.zeros(n, dtype=bool)
    null_x = np.zeros(n, dtype=bool)
    if where in ("y", "both"):
        null_y[rng.choice(n, n // 20, replace=False)] = True
    if where in ("x", "both"):
        null_x[rng.choice(n, n // 20, replace=False)] = True
    for g in (1, 4):                                    # groups 1 and 4 have no nulls
        null_y[off[g]:off[g + 1]] = False
        null_x[off[g]:off[g + 1]] = False
    cols = _cols(X, y, null_y if null_y.any() else None, null_x if null_x.any() else None)
    kw = _kw(64, bias, 0.1, policy, min_size=p + 2)
    fast, loop = _host_call(cols, kw, f32, off), _loop(cols, off, kw, f32)
    for a, b, name in zip(fast, loop, ("coeffs", "pred", "valid")):
        assert a.shape == b.shape and np.array_equal(a, b), name


def _err(fn):
    with pytest.raises(PdsbError) as ei:
        fn()
    return str(ei.value)


@pytest.mark.parametrize("case", ["empty", "nulls", "features", "window_zero", "window_size", "features_then_nulls"])
def test_first_error_matches_the_loop(case):
    p, bias = 3, True
    sizes = {"empty": [50, 0, 50], "nulls": [50, 50, 50], "features": [50, 3, 50], "window_zero": [50, 50, 50],
             "window_size": [50, 6, 50], "features_then_nulls": [50, 3, 50]}[case]
    off = group_offsets(sizes)
    n = int(off[-1])
    X, y = _data(n, p, False, seed=2)
    null_y = np.zeros(n, dtype=bool)
    if case in ("nulls", "features_then_nulls"):
        null_y[off[2] + 1] = True
    kw = _kw(0 if case == "window_zero" else 10, bias)
    cols = _cols(X, y, null_y if null_y.any() else None)
    fast, loop = _err(lambda: _host_call(cols, kw, True, off)), _err(lambda: _loop(cols, off, kw, True))
    assert fast == loop
    want = {"empty": "Empty data", "nulls": "Nulls found in data", "features": "#Data < #features",
            "window_zero": "window / start_with must be >= 1", "window_size": "#Data < window size",
            "features_then_nulls": "#Data < #features"}[case]
    assert want in fast


@pytest.mark.parametrize("offsets", [[0, 50, 99], [0, 60, 50, 100], [1, 50, 100], [0, 50, 101]])
def test_bad_offsets_are_refused(offsets):
    X, y = _data(100, 2, True, seed=4)
    with pytest.raises(PdsbError, match="grouped rolling_lin_reg"):
        _host_call(_cols(X, y), _kw(3, False), False, offsets)


# 4. edge cases ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("f64,p,window,route", [(False, 3, 1500, PACKED), (True, 3, 700, LANE)])
def test_one_group_of_1100_chains_is_the_single_call(f64, p, window, route):
    n = 1100 * 1024 + 5                                  # the group scan carries across a 1024-chain chunk
    X, y = _data(n, p, f64, seed=3)
    grouped, Xd, yd = _dev(X, y, [0, n], window, 0, True, 0.0, None)
    assert _route() == route
    _same_as_single(grouped, Xd, yd, [0, n], window, 0, True, 0.0, None)


@pytest.mark.parametrize("window", [100, 101])
@pytest.mark.parametrize("p", [7, 8])                 # 8 and 9 coefficients: even and odd D of the packed kernel
def test_groups_at_odd_rows(p, window):
    sizes = [1, 333, 1201, 2048 + 77, 515, 1024, 3]   # odd first rows for most groups
    off = group_offsets(sizes)
    X, y = _data(int(off[-1]), p, False, seed=p * window)
    grouped, Xd, yd = _dev(X, y, off, window, 0, True, 0.0, None)
    assert _route() == PACKED
    assert any(o % 2 for o in off[:-1])
    _same_as_single(grouped, Xd, yd, off, window, 0, True, 0.0, None)


@pytest.mark.parametrize("f64,p,window,skip", [(False, 3, 256, None), (False, 8, 256, [0, 1, 0, 1, 0]),
                                               (True, 6, 40, None), (True, 13, 300, [1, 0, 1, 0, 1])])
def test_other_groups_do_not_matter_and_repeats_are_identical(f64, p, window, skip):
    import torch

    sizes = [400, 1500, 37, 2100, 1064]
    off = group_offsets(sizes)
    X, y = _data(int(off[-1]), p, f64, seed=8, nan_rows=10)
    a, Xd, yd = _dev(X, y, off, window, p + 2, True, 0.1, skip)
    again, _, _ = _dev(X, y, off, window, p + 2, True, 0.1, skip)
    for u, v in zip(a, again):
        assert torch.equal(_iview(u) if u.is_floating_point() else u, _iview(v) if v.is_floating_point() else v)
    X2, y2 = X.copy(), y.copy()
    X2[off[1]:off[2]] *= 3.0
    y2[off[1]:off[2]] = -y2[off[1]:off[2]]
    b, _, _ = _dev(X2, y2, off, window, p + 2, True, 0.1, skip)
    for g in (0, 2, 3, 4):
        s, e = int(off[g]), int(off[g + 1])
        assert torch.equal(_iview(a[0][s:e]), _iview(b[0][s:e])) and torch.equal(_iview(a[1][s:e]), _iview(b[1][s:e]))
        assert torch.equal(a[2][s:e], b[2][s:e])
    assert not torch.equal(_iview(a[0][off[1]:off[2]]), _iview(b[0][off[1]:off[2]]))


def test_a_million_groups_of_100_rows():
    import torch
    from polars_ds_extension_b200 import device as dev

    G, m, p, w = 1_000_000, 100, 2, 20
    rng = np.random.default_rng(12)
    X = torch.randn((p, G * m), dtype=torch.float32, device="cuda", generator=torch.Generator("cuda").manual_seed(1))
    y = X[0] * 0.5 - X[1] + 0.1
    off = torch.arange(0, G * m + 1, m, dtype=torch.int64, device="cuda")
    co, pr, va = dev.grouped_rolling_lin_reg(X, y, off, w, 0, add_bias=True)
    torch.cuda.synchronize()
    assert _route() == LANE
    for g in sorted(rng.choice(G, 64, replace=False).tolist()) + [0, G - 1]:
        a, b = g * m, (g + 1) * m
        c1, p1, v1 = dev.online_lin_reg(X[:, a:b].contiguous(), y[a:b].contiguous(), w, 0, add_bias=True)
        torch.cuda.synchronize()
        assert torch.equal(v1, va[a:b]) and torch.equal(_iview(c1), _iview(co[a:b])), g
        assert torch.equal(_iview(p1), _iview(pr[a:b])), g
    assert int(va.sum()) == G * (m - w + 1)


@pytest.mark.parametrize("skip_half", [False, True])
def test_launch_count_does_not_grow_with_the_groups(skip_half):
    L = lib()
    counts = []
    for G in (10, 10_000):
        sizes = [300] * G
        off = group_offsets(sizes)
        X, y = _data(int(off[-1]), 8, False, seed=G)
        skip = [g % 2 for g in range(G)] if skip_half else None
        before = int(L.pdsb_kernel_launch_count())
        _dev(X, y, off, 128, 0, True, 0.0, skip)
        counts.append(int(L.pdsb_kernel_launch_count()) - before)
    assert counts[0] == counts[1], counts


def test_window_below_one_is_refused():
    import torch

    X = torch.zeros((2, 10), dtype=torch.float32, device="cuda")
    off = torch.tensor([0, 5, 10], dtype=torch.int64, device="cuda")
    from polars_ds_extension_b200 import device as dev

    with pytest.raises(PdsbError, match="window must be >= 1"):
        dev.grouped_rolling_lin_reg(X, X[0], off, 0, 0)


# 5. any nonzero skip byte is the skip class, and every output row is written -----------------------------------------
@pytest.mark.parametrize("f64,p,window", [(False, 8, 256), (False, 8, 1500), (False, 11, 1500), (True, 3, 256),
                                          (False, 3, 40), (False, 13, 300)])
def test_nonzero_skip_bytes_are_the_skip_class(f64, p, window):
    import torch

    q = p + 1
    sizes = [window + 3, 3 * 1024 + 17, 1024, 2 * window + 1, 2050, 1500]
    off = group_offsets(sizes)
    n = int(off[-1])
    X, y = _data(n, p, f64, seed=window * 3 + p, nan_rows=30)
    flags = [0, 2, 255, 0, 1, 7]
    Xd = torch.from_numpy(np.ascontiguousarray(X.T)).cuda()
    yd = torch.from_numpy(np.ascontiguousarray(y)).cuda()
    dt = Xd.dtype
    # sentinels: outputs the call leaves unwritten keep these bits, which no fit produces
    co = torch.full((n, q), 12345.0, dtype=dt, device="cuda")
    pr = torch.full((n,), 12345.0, dtype=dt, device="cuda")
    va = torch.full((n,), 0xAB, dtype=torch.uint8, device="cuda")
    sk = torch.tensor(flags, dtype=torch.uint8, device="cuda")
    offd = torch.from_numpy(off).cuda()
    fn = getattr(lib(), f"pdsb_dev_grouped_rolling_lin_reg_{'f64' if f64 else 'f32'}")
    check(fn(C.c_void_p(Xd.data_ptr()), n, C.c_void_p(yd.data_ptr()), n, p, 1, window, q, 0.25,
             C.c_void_p(offd.data_ptr()), len(sizes), C.c_void_p(sk.data_ptr()), C.c_void_p(co.data_ptr()),
             C.c_void_p(pr.data_ptr()), C.c_void_p(va.data_ptr()), None))
    torch.cuda.synchronize()
    assert _route() == _expected_route(f64, q, window, True)
    assert bool(((va == 0) | (va == 1)).all()), "a row was left unwritten"
    _same_as_single((co, pr, va), Xd, yd, off, window, q, True, 0.25, [int(f != 0) for f in flags])
