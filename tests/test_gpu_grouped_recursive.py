"""recursive_lin_reg(...).over(key) on the H100: pl_recursive_lr_by(_f32) and pdsb_dev_grouped_recursive_lin_reg_* against
Polars' per-group loop and the single-column entries.

The contract: group g is rows [offsets[g], offsets[g+1]) in key order, and its output is bit for bit what
pl_recursive_lr(_f32) returns on that group's rows alone (coefficients, pred, validity, NaN and null placement), so the
fast path equals the loop exactly, on every pass-C route, and no group depends on another group's rows."""
import zlib

import numpy as np
import pyarrow as pa
import pytest

import polars_ds_extension_b200 as pds
import polars_ds_extension_b200.config as cfg
from polars_ds_extension_b200 import _harness
from polars_ds_extension_b200._lib import PdsbError, lib
from tests.helpers import group_offsets

pytestmark = pytest.mark.gpu

PACKED, LANE, GENERIC = 1, 2, 3
# (f64, p, bias) -> the pass-C kernel it must take: packed f32 up to 9 coefficients, lane-per-moment up to 12, generic
ROUTES = [(False, 3, True, PACKED), (False, 8, True, PACKED), (False, 9, True, LANE), (False, 12, False, LANE),
          (True, 2, True, LANE), (True, 12, False, LANE), (False, 13, False, GENERIC), (True, 13, True, GENERIC)]
SIZES = [31, 32, 33, 63, 64, 65, 1023, 1024, 1025, 2047, 2048, 2049, 3000]


def _data(n, p, f64, seed, nan_rows=0):
    rng = np.random.default_rng(seed)
    dt = np.float64 if f64 else np.float32
    X = rng.standard_normal((n, p)).astype(dt)
    y = (X.astype(np.float64) @ (np.arange(p) % 5 - 2.0) + 0.5 + 0.1 * rng.standard_normal(n)).astype(dt)
    if nan_rows:
        X[rng.choice(n, nan_rows, replace=False), rng.integers(0, p)] = np.nan
        y[rng.choice(n, nan_rows, replace=False)] = np.nan
    return X, y


def _cols(X, y, null_y=None, null_x=None):
    yc = pa.array(y, mask=null_y)
    xs = [pa.array(X[:, j], mask=null_x if j == 0 else None) for j in range(X.shape[1])]
    return [pa.chunked_array([yc])] + [pa.chunked_array([x]) for x in xs]


def _kw(start, bias, lam=0.0, policy="raise"):
    return {"null_policy": policy, "n": int(start), "bias": bool(bias), "lambda": float(lam), "min_size": 0}


def _names(k):
    return ["y"] + [f"x{j}" for j in range(k - 1)]


def _by(cols, offsets, kw, f64):
    ins = [pa.chunked_array([pa.array(np.asarray(offsets, dtype=np.int64))])] + cols
    return _harness.call_plugin("pl_recursive_lr_by" + ("" if f64 else "_f32"), ins, ["__offsets__"] + _names(len(cols)), kw)


def _one(cols, kw, f64):
    return _harness.call_plugin("pl_recursive_lr" + ("" if f64 else "_f32"), cols, _names(len(cols)), kw)


def _loop(cols, offsets, kw, f64):
    """pl_recursive_lr once per group, concatenated (what Polars' loop returns in key order)."""
    parts = [_one([c.slice(a, b - a) for c in cols], kw, f64) for a, b in zip(offsets[:-1], offsets[1:])]
    return pa.concat_arrays(parts)


def _bits(arr):
    """(coeff validity, coeff bits of the valid rows, pred validity, pred bits of the valid rows)."""
    co, pr = arr.flatten()                              # the struct's offset applied (a slice of a result)
    cv = np.asarray(co.is_valid().to_numpy(zero_copy_only=False), dtype=bool)
    pv = np.asarray(pr.is_valid().to_numpy(zero_copy_only=False), dtype=bool)
    flat = co.flatten().to_numpy(zero_copy_only=False)
    pf = pr.filter(pa.array(pv)).to_numpy(zero_copy_only=False)
    it = np.uint32 if flat.dtype == np.float32 else np.uint64
    return cv, flat.view(it), pv, pf.view(it)


def _same(a, b, what=""):
    for x, y, name in zip(_bits(a), _bits(b), ("coeff validity", "coeffs", "pred validity", "pred")):
        assert x.shape == y.shape and np.array_equal(x, y), f"{what}: {name} differ"


def _route():
    return int(lib().pdsb_last_online_path())


# 1. every route: fast == loop, bit for bit, and the intended kernel ---------------------------------------------------
@pytest.mark.parametrize("lam", [0.0, 0.5])
@pytest.mark.parametrize("f64,p,bias,route", ROUTES)
def test_fast_equals_the_loop_on_every_route(f64, p, bias, route, lam):
    q = p + int(bias)
    start = q + 2
    sizes = [start] + SIZES
    off = group_offsets(sizes)
    X, y = _data(int(off[-1]), p, f64, seed=p * 7 + int(bias) + int(f64) * 100)
    cols, kw = _cols(X, y), _kw(start, bias, lam)
    fast = _by(cols, off, kw, f64)
    assert _route() == route
    _same(fast, _loop(cols, off, kw, f64), f"route {route}")
    assert len(fast) == off[-1]


# 2. the frame: shuffled keys, over(key, fast=True) against over(key) ----------------------------------------------
@pytest.mark.parametrize("f64", [False, True])
def test_frame_over_fast_equals_over(monkeypatch, f64):
    monkeypatch.setattr(cfg, "LIN_REG_EXPR_F64", f64)
    rng = np.random.default_rng(11)
    sizes = [40, 700, 1025, 2100, 64, 33]
    X, y = _data(sum(sizes), 4, f64, seed=5)
    g = rng.permutation(np.repeat(np.arange(len(sizes)), sizes))
    df = pds.Frame({"y": y, **{f"x{j}": X[:, j] for j in range(4)}, "g": g})
    e = pds.recursive_lin_reg("x0", "x1", "x2", "x3", target="y", start_with=6, add_bias=True, l2_reg=0.1)
    fast, loop = (df.select(e.over("g", fast=f))[e.symbol] for f in (True, False))
    _same(fast, loop, "frame")


# 3. group lengths: exactly start_with, one group == the single call, > 1024 chains in one group -------------------
@pytest.mark.parametrize("f64,p,bias,route", [(False, 3, True, PACKED), (True, 3, False, LANE)])
def test_one_group_is_the_single_call(f64, p, bias, route):
    n = 1024 * 1024 + 77 * 1024 + 5                     # 1100 chains: the group scan carries across 1024-chain chunks
    X, y = _data(n, p, f64, seed=3)
    cols, kw = _cols(X, y), _kw(4, bias)
    fast = _by(cols, [0, n], kw, f64)
    assert _route() == route
    _same(fast, _one(cols, kw, f64), "one group")


@pytest.mark.parametrize("f64,p,bias,route", [(False, 3, True, PACKED), (True, 5, True, LANE), (False, 13, True, GENERIC)])
def test_long_group_among_short_ones(f64, p, bias, route):
    q = p + int(bias)
    sizes = [q, 1024 * 1025 + 3, q + 1, 100] if route != GENERIC else [q, 40 * 1024 + 9, q + 1, 100]
    off = group_offsets(sizes)
    X, y = _data(int(off[-1]), p, f64, seed=9)
    cols, kw = _cols(X, y), _kw(q, bias, 0.25)
    fast = _by(cols, off, kw, f64)
    assert _route() == route
    _same(fast, _loop(cols, off, kw, f64), "long group")


# 4. null policies, groups with and without nulls mixed in one call -------------------------------------------------
def _null_case(policy, where, n, rng):
    null_y = np.zeros(n, dtype=bool)
    null_x = np.zeros(n, dtype=bool)
    if where in ("y", "both"):
        null_y[rng.choice(n, n // 20, replace=False)] = True
    if where in ("x", "both"):
        null_x[rng.choice(n, n // 20, replace=False)] = True
    return null_y, null_x


@pytest.mark.parametrize("policy,where", [("skip", "both"), ("skip", "x"), ("zero", "y"), ("one", "x"), ("2.5", "both"),
                                          ("ignore", "both"), ("ignore", "nan")])
@pytest.mark.parametrize("f64,p,bias,route", [(False, 3, True, PACKED), (True, 4, True, LANE), (False, 10, False, LANE),
                                              (True, 13, False, GENERIC)])
def test_null_policies(f64, p, bias, route, policy, where):
    q = p + int(bias)
    sizes = [q + 3, 500, 1100, 64, 2050, 40]
    off = group_offsets(sizes)
    n = int(off[-1])
    rng = np.random.default_rng(zlib.crc32(f"{policy}{where}{p}".encode()))
    X, y = _data(n, p, f64, seed=p, nan_rows=40 if where == "nan" else 0)
    null_y, null_x = _null_case(policy, where, n, rng)
    for g in (1, 4):                                    # groups 1 and 4 have no nulls
        null_y[off[g]:off[g + 1]] = False
        null_x[off[g]:off[g + 1]] = False
    cols, kw = _cols(X, y, null_y, null_x), _kw(q + 1, bias, 0.0, policy)
    fast = _by(cols, off, kw, f64)
    assert _route() == route
    _same(fast, _loop(cols, off, kw, f64), f"{policy} {where}")


def test_raise_with_nulls_fails_like_the_loop():
    X, y = _data(300, 3, False, seed=1)
    null_y = np.zeros(300, dtype=bool)
    null_y[250] = True
    cols, kw = _cols(X, y, null_y), _kw(4, True)
    with pytest.raises(PdsbError, match="Nulls found in data"):
        _by(cols, [0, 100, 200, 300], kw, False)
    # a group without nulls on its own is fine, so the loop gets through the first two groups as well
    _same(_by([c.slice(0, 200) for c in cols], [0, 100, 200], kw, False),
          _loop([c.slice(0, 200) for c in cols], [0, 100, 200], kw, False), "raise, no nulls")


# 5. the first error across groups is the loop's; bad offsets are refused -------------------------------------------
def _err(fn):
    with pytest.raises(PdsbError) as ei:
        fn()
    return str(ei.value)


@pytest.mark.parametrize("case", ["features_then_nulls", "nulls_then_features", "window", "start_zero"])
def test_first_error_matches_the_loop(case):
    p, bias = 3, True
    sizes = {"features_then_nulls": [50, 3, 50], "nulls_then_features": [50, 50, 3], "window": [50, 6, 50],
             "start_zero": [50, 50, 50]}[case]
    off = group_offsets(sizes)
    n = int(off[-1])
    X, y = _data(n, p, False, seed=2)
    null_y = np.zeros(n, dtype=bool)
    null_y[off[1] + 1 if case == "nulls_then_features" else off[2] + 1] = True
    kw = _kw(0 if case == "start_zero" else 10, bias)
    cols = _cols(X, y, null_y)
    fast, loop = _err(lambda: _by(cols, off, kw, False)), _err(lambda: _loop(cols, off, kw, False))
    assert fast == loop
    want = {"features_then_nulls": "#Data < #features", "nulls_then_features": "Nulls found in data",
            "window": "#Data < window size", "start_zero": "start_with must be >= 1"}[case]
    assert want in fast


@pytest.mark.parametrize("offsets", [[0, 50, 99], [0, 60, 50, 100], [1, 50, 100], [0, 50, 101]])
def test_bad_offsets_are_refused(offsets):
    X, y = _data(100, 2, True, seed=4)
    with pytest.raises(PdsbError, match="grouped recursive_lin_reg"):
        _by(_cols(X, y), offsets, _kw(3, False), True)


# 6. the device entry against pdsb_dev_online_lin_reg_* on each group's slice ---------------------------------------
@pytest.mark.parametrize("f64,p,bias,route", ROUTES)
def test_device_entry_equals_the_single_entry_per_group(f64, p, bias, route):
    import torch
    from polars_ds_extension_b200 import device as dev

    q = p + int(bias)
    sizes = [q + 1, 1, 0, 31, 1024, 1025, 2049, 64, 65]
    off = group_offsets(sizes)
    n = int(off[-1])
    X, y = _data(n, p, f64, seed=p + 40, nan_rows=30)
    Xd = torch.from_numpy(np.ascontiguousarray(X.T)).cuda()
    yd = torch.from_numpy(y).cuda()
    skip = torch.tensor(np.arange(len(sizes)) % 2, dtype=torch.uint8, device="cuda")
    lam = 0.3
    co, pr, va = dev.grouped_recursive_lin_reg(Xd, yd, torch.from_numpy(off).cuda(), min_rows=2, add_bias=bias,
                                               l2_reg=lam, skip=skip)
    torch.cuda.synchronize()
    assert _route() == route
    for g, (a, b) in enumerate(zip(off[:-1], off[1:])):
        if b == a:
            continue
        c1, p1, v1 = dev.online_lin_reg(Xd[:, a:b].contiguous(), yd[a:b].contiguous(), 0, 2, add_bias=bias, l2_reg=lam,
                                        skip=bool(g % 2))
        torch.cuda.synchronize()
        assert torch.equal(v1, va[a:b]), g
        assert torch.equal(c1.view(-1).view(torch.int32 if not f64 else torch.int64),
                           co[a:b].reshape(-1).view(torch.int32 if not f64 else torch.int64)), g
        assert torch.equal(p1.view(torch.int32 if not f64 else torch.int64),
                           pr[a:b].view(torch.int32 if not f64 else torch.int64)), g


# 7. independence from the other groups, repeats, many short groups --------------------------------------------------
@pytest.mark.parametrize("f64,p,bias,route", [(False, 3, True, PACKED), (True, 6, False, LANE), (True, 13, True, GENERIC)])
def test_other_groups_do_not_matter_and_repeats_are_identical(f64, p, bias, route):
    sizes = [100, 1500, 37, 2100, 64]
    off = group_offsets(sizes)
    X, y = _data(int(off[-1]), p, f64, seed=8)
    kw = _kw(p + 2, bias, 0.1)
    a = _by(_cols(X, y), off, kw, f64)
    assert _route() == route
    _same(a, _by(_cols(X, y), off, kw, f64), "repeat")
    X2, y2 = X.copy(), y.copy()
    X2[off[1]:off[2]] *= 3.0
    y2[off[1]:off[2]] = -y2[off[1]:off[2]]
    b = _by(_cols(X2, y2), off, kw, f64)
    for g in (0, 2, 3, 4):
        sl = slice(int(off[g]), int(off[g + 1]))
        _same(a.slice(sl.start, sl.stop - sl.start), b.slice(sl.start, sl.stop - sl.start), f"group {g}")
    assert not np.array_equal(_bits(a.slice(off[1], sizes[1]))[1], _bits(b.slice(off[1], sizes[1]))[1])


def test_a_million_groups_of_100_rows():
    import torch
    from polars_ds_extension_b200 import device as dev

    G, m, p = 1_000_000, 100, 2
    rng = np.random.default_rng(12)
    X = torch.randn((p, G * m), dtype=torch.float32, device="cuda", generator=torch.Generator("cuda").manual_seed(1))
    y = X[0] * 0.5 - X[1] + 0.1
    off = torch.arange(0, G * m + 1, m, dtype=torch.int64, device="cuda")
    co, pr, va = dev.grouped_recursive_lin_reg(X, y, off, min_rows=5, add_bias=True)
    torch.cuda.synchronize()
    assert _route() == PACKED
    for g in sorted(rng.choice(G, 64, replace=False).tolist()) + [0, G - 1]:
        a, b = g * m, (g + 1) * m
        c1, p1, v1 = dev.online_lin_reg(X[:, a:b].contiguous(), y[a:b].contiguous(), 0, 5, add_bias=True)
        torch.cuda.synchronize()
        assert torch.equal(v1, va[a:b]) and torch.equal(c1.view(torch.int32), co[a:b].view(torch.int32)), g
        assert torch.equal(p1.view(torch.int32), pr[a:b].view(torch.int32)), g
    assert int(va.sum()) == G * (m - 4)
