"""group_by().agg(query_ar_coeffs(...), fast=True) on the device (pl_ar_coeffs_by, K5's AR pass).

The main contract: per group, the coefficients and their validity are bit for bit what pl_lr_by(_f32) returns on the
group's lagged columns materialised on the host (target x_t for t = L .. m-1, features x_{t-1} .. x_{t-L}, taken within
the group; feature nulls filled, target nulls left null and dropped by pl_lr_by's "skip").  Then: against Polars' loop
and numpy.linalg.lstsq, the errors, the device entry, independence, repeats and 1e6 groups."""
import numpy as np
import pyarrow as pa
import pytest

import polars_ds_extension_b200 as pds
import polars_ds_extension_b200.config as cfg
from polars_ds_extension_b200 import _harness
from polars_ds_extension_b200 import Frame
from tests.helpers import group_offsets

pytestmark = pytest.mark.gpu

LAGS = list(range(1, 13)) + [16, 33, 64]


def _kwargs(lag, bias, policy, f32):
    cfg_f64 = cfg.LIN_REG_EXPR_F64
    try:
        cfg.LIN_REG_EXPR_F64 = not f32
        return dict(pds.lin_reg("a", target="y", add_bias=bias, null_policy=policy).kwargs)
    finally:
        cfg.LIN_REG_EXPR_F64 = cfg_f64


def _sizes(lag):
    q = lag + 1
    return [0, 1, max(lag - 1, 0), lag, lag + 1, q, q + 1, 31, 32, 33, 8191, 8192, 8193, 2 * 8192 - 1, 2 * 8192 + 1,
            100_003]


def _series(n, f32, seed):
    # a moving average, x_t = e_t + 0.3 e_{t-1} - 0.1 e_{t-2}: correlated lags, yet far from lin_reg's rank gate at 64 lags
    # (the gate reads the uncentred Gram, so a level large against the noise would null the long fits)
    e = np.random.default_rng(seed).standard_normal(n + 2)
    x = e[2:] + 0.3 * e[1:-1] - 0.1 * e[:-2]
    return x.astype(np.float32 if f32 else np.float64)


def _fast(x: pa.Array, offsets, lag, kw, f32):
    return _harness.call_plugin("pl_ar_coeffs_by" + ("_f32" if f32 else ""),
                                [pa.array(np.asarray(offsets, np.int64)), x], ["__offsets__", "x"], dict(kw, lag=lag))


def _materialised(xv, valid, offsets, lag, fill, f32):
    """The lagged columns of every group: (sliced offsets, target, features), nulls as the single pl_lr treats them."""
    dt = np.float32 if f32 else np.float64
    offsets = np.asarray(offsets, np.int64)
    m = np.diff(offsets)
    k = np.maximum(m - lag, 0)
    so = group_offsets(k)
    tidx = np.concatenate([np.arange(a + lag, b) for a, b in zip(offsets[:-1], offsets[1:])] + [np.zeros(0, np.int64)])
    tidx = tidx.astype(np.int64)
    y = pa.array(xv[tidx].astype(dt), mask=~valid[tidx])
    feats = []
    for i in range(1, lag + 1):
        v = xv[tidx - i].astype(dt)
        ok = valid[tidx - i]
        if fill is None:
            feats.append(pa.array(v, mask=~ok))
        else:
            feats.append(pa.array(np.where(ok, v, dt(fill)).astype(dt)))
    return so, y, feats


def _reference(xv, valid, offsets, lag, kw, f32):
    """pl_lr_by(_f32) on the materialised lagged columns: fill policies fill the features here and pl_lr_by drops the
    null targets with "skip"; "skip" leaves both null."""
    pol = kw["null_policy"]
    fill = None if pol in ("skip", "raise") else (0.0 if pol == "zero" else 1.0 if pol == "one" else float(pol))
    if fill is not None and f32:
        fill = float(np.float32(np.float64(pol)) if pol not in ("zero", "one") else fill)
    so, y, feats = _materialised(xv, valid, offsets, lag, fill, f32)
    names = ["__offsets__", "y"] + [str(i) for i in range(1, lag + 1)]
    return _harness.call_plugin("pl_lr_by" + ("_f32" if f32 else ""), [pa.array(so), y] + feats, names,
                                dict(kw, null_policy="skip"))


def _bits(arr: pa.Array):
    """(validity, bit patterns of the valid rows' coefficients) of a List result."""
    arr = arr.combine_chunks() if isinstance(arr, pa.ChunkedArray) else arr
    valid = np.asarray(arr.is_valid().to_numpy(zero_copy_only=False), dtype=bool)
    offs = arr.offsets.to_numpy()
    vals = arr.values.to_numpy(zero_copy_only=False)
    row = np.repeat(np.arange(len(arr)), np.diff(offs))
    v = vals[offs[0]:offs[-1]][valid[row]]
    return valid, v.view(np.uint32 if v.dtype == np.float32 else np.uint64)


def _same(a, b, what):
    va, ba = _bits(a)
    vb, bb = _bits(b)
    assert np.array_equal(va, vb), f"{what}: validity differs in {np.flatnonzero(va != vb)[:10]}"
    assert ba.shape == bb.shape and np.array_equal(ba, bb), \
        f"{what}: coefficient bits differ at {np.flatnonzero(ba != bb)[:10] if ba.shape == bb.shape else 'shape'}"


def _column(xv, valid):
    return pa.array(xv, mask=None if valid.all() else ~valid)


@pytest.mark.parametrize("f32", [True, False], ids=["f32", "f64"])
@pytest.mark.parametrize("bias", [True, False], ids=["bias", "nobias"])
@pytest.mark.parametrize("lag", LAGS)
def test_bits_equal_pl_lr_by_on_the_lagged_columns(f32, bias, lag):
    sizes = _sizes(lag)
    rng = np.random.default_rng(1000 + lag)
    sizes = sizes + list(rng.integers(0, 3 * lag + 70, 40))
    rng.shuffle(sizes)
    offsets = group_offsets(sizes)
    xv = _series(int(offsets[-1]), f32, lag)
    valid = np.ones(len(xv), bool)
    kw = _kwargs(lag, bias, "raise", f32)
    got = _fast(_column(xv, valid), offsets, lag, kw, f32)
    assert len(got) == len(sizes)
    _same(got, _reference(xv, valid, offsets, lag, kw, f32), f"lag {lag}")
    valid_groups = _bits(got)[0]
    target_rows = np.asarray(sizes) - lag
    assert not valid_groups[target_rows < lag + bias].any()      # fewer target rows than coefficients: null
    assert valid_groups[target_rows >= 8000].all()


def _null_layout(offsets, lag, rng):
    n = int(offsets[-1])
    valid = rng.random(n) > 0.03
    for g, (a, b) in enumerate(zip(offsets[:-1], offsets[1:])):
        if b - a < 3:
            continue
        kind = g % 4
        if kind == 0:
            valid[a] = False                                    # the group's first row
        elif kind == 1:
            valid[b - 1] = False                                # its last row
        elif kind == 2:
            s = min(a + lag + 5, b - 1)
            valid[s:min(s + lag, b)] = False                    # every row of a lag window
        else:
            valid[a:b] = True                                   # a group without nulls
    return valid


@pytest.mark.parametrize("f32", [True, False], ids=["f32", "f64"])
@pytest.mark.parametrize("policy", ["zero", "one", "0.3", "-2.5e-3", "skip"])
@pytest.mark.parametrize("lag", [1, 3, 10, 11, 33])
def test_null_policies(f32, policy, lag):
    rng = np.random.default_rng(7 * lag)
    sizes = [lag, lag + 1, lag + 2, 40, 200, 8193, 3 * lag + 1, 500, 1, 0, 1000, 77]
    offsets = group_offsets(sizes)
    xv = _series(int(offsets[-1]), f32, 3 + lag)
    valid = _null_layout(offsets, lag, rng)
    xv_raw = np.where(valid, xv, xv.dtype.type(12345.0))        # a null's slot holds garbage the kernel must not see
    kw = _kwargs(lag, True, policy, f32)
    got = _fast(_column(xv_raw, valid), offsets, lag, kw, f32)
    _same(got, _reference(xv, valid, offsets, lag, kw, f32), f"{policy} lag {lag}")


@pytest.mark.parametrize("f32", [True, False], ids=["f32", "f64"])
@pytest.mark.parametrize("lag", [2, 10, 12])
def test_non_finite_values_drop_their_rows(f32, lag):
    sizes = [300, 64, 5000, 8193, 40]
    offsets = group_offsets(sizes)
    xv = _series(int(offsets[-1]), f32, 11)
    for pos, v in [(0, np.nan), (5, np.inf), (301, -np.inf), (364 + 100, np.nan), (364 + 4999, np.inf),
                   (364 + 5000 + 17, np.nan), (364 + 5000 + 18, np.nan)]:
        xv[pos] = v
    xv[-40:] = np.nan                                           # a group with no finite row
    valid = np.ones(len(xv), bool)
    for policy in ("raise", "zero"):
        kw = _kwargs(lag, True, policy, f32)
        got = _fast(_column(xv, valid), offsets, lag, kw, f32)
        _same(got, _reference(xv, valid, offsets, lag, kw, f32), f"non-finite {policy}")
        assert not _bits(got)[0][-1]


def _ar_lstsq(x, lag, bias):
    cols = [x[lag - i: len(x) - i] for i in range(1, lag + 1)]
    A = np.column_stack(cols + ([np.ones(len(x) - lag)] if bias else []))
    return np.linalg.lstsq(A, x[lag:], rcond=None)[0]


@pytest.mark.parametrize("f64", [True, False], ids=["f64", "f32"])
@pytest.mark.parametrize("lag,bias", [(1, True), (3, True), (5, False), (12, True)])
def test_against_the_loop_and_lstsq(monkeypatch, f64, lag, bias):
    monkeypatch.setattr(cfg, "LIN_REG_EXPR_F64", f64)
    rng = np.random.default_rng(lag)
    n_groups = 40
    sizes = rng.integers(lag + 30, 3000, n_groups)
    key = np.repeat(np.arange(n_groups) * 7 % 41, sizes)
    x = _series(len(key), False, lag + 50)
    shuffle = rng.permutation(len(key))             # shuffled keys: a group's series is its rows in frame order
    key, x = key[shuffle], x[shuffle]
    df = Frame({"x": x, "k": key})
    e = pds.query_ar_coeffs("x", lag=lag, add_bias=bias)
    fast = df.group_by("k").agg(e, fast=True)
    loop = df.group_by("k").agg(e, fast=False)
    assert list(fast["k"]) == list(loop["k"])
    tol = 1e-10 if f64 else 1e-4
    from tests.parity_rule import rel

    for i, k in enumerate(fast["k"]):
        f = np.asarray(fast[e.out_name][i].as_py())
        lp = np.asarray(loop[e.out_name][i][0].as_py())
        assert rel(f, lp) <= tol, (k, rel(f, lp))
        xs = x[key == k] if f64 else x[key == k].astype(np.float32).astype(np.float64)
        assert rel(f, _ar_lstsq(xs, lag, bias)) <= tol, (k, "lstsq")


def test_errors():
    offsets = group_offsets([50, 60])
    x = np.arange(110.0)
    valid = np.ones(110, bool)
    valid[70] = False
    with pytest.raises(pds.PdsbError, match="Nulls found in data"):
        _fast(_column(x, valid), offsets, 2, _kwargs(2, True, "raise", False), False)
    for offs, msg in [([0, 50, 100], "bad group offsets"), ([0, 60, 50, 110], "non-decreasing"),
                      ([5, 50, 110], "bad group offsets")]:
        with pytest.raises(pds.PdsbError, match=msg):
            _fast(pa.array(x), offs, 2, _kwargs(2, True, "raise", False), False)
    with pytest.raises(pds.PdsbError, match="1 to 64 lags"):
        _fast(pa.array(x), offsets, 65, _kwargs(65, True, "raise", False), False)
    with pytest.raises(pds.PdsbError, match="1 to 64 lags"):
        _fast(pa.array(x), offsets, 0, _kwargs(0, True, "raise", False), False)
    df = Frame({"x": _series(2000, False, 1), "k": np.repeat([0, 1], 1000)})
    e = pds.query_ar_coeffs("x", lag=65)
    with pytest.raises(pds.PdsbError, match="1 to 64 lags"):
        df.group_by("k").agg(e, fast=True)
    loop = df.group_by("k").agg(e, fast=False)[e.out_name]     # the loop still fits 65 lags
    assert len(loop) == 2 and len(loop[0][0].as_py()) == 66


@pytest.mark.parametrize("f32", [True, False], ids=["f32", "f64"])
@pytest.mark.parametrize("lag", [4, 33])
def test_device_entry(f32, lag):
    import torch

    from polars_ds_extension_b200 import device

    sizes = [lag, 5000, 8193, 123, 20_000, lag + 3]
    offsets = group_offsets(sizes)
    xv = _series(int(offsets[-1]), f32, 99)
    valid = np.ones(len(xv), bool)
    valid[[10, 5003, 5004, 13_000]] = False
    dt = torch.float32 if f32 else torch.float64
    xf = np.where(valid, xv, 0).astype(xv.dtype)                   # the "zero" fill
    xd = torch.tensor(xf, dtype=dt, device="cuda")
    md = torch.tensor(valid.astype(xv.dtype), dtype=dt, device="cuda")
    od = torch.tensor(offsets, device="cuda")
    beta, status = device.grouped_ar_coeffs(xd, od, lag, add_bias=True, mask=md)
    torch.cuda.synchronize()
    kw = _kwargs(lag, True, "zero", f32)
    plug = _fast(_column(xf, valid), offsets, lag, kw, f32)
    vb, bb = _bits(plug)
    assert np.array_equal(vb, status.cpu().numpy() == 0)
    b = beta.cpu().numpy()[vb].astype(np.float32 if f32 else np.float64).ravel()
    assert np.array_equal(b.view(bb.dtype), bb)
    # pdsb_dev_grouped_lin_reg on the lagged columns materialised on the device
    so, y, feats = _materialised(xf, valid, offsets, lag, 0.0, f32)
    yv = np.where(np.asarray(y.is_valid()), y.to_numpy(zero_copy_only=False), np.nan)
    n = len(yv)
    X = torch.stack([torch.tensor(f.to_numpy(zero_copy_only=False), dtype=dt, device="cuda") for f in feats])
    b2, s2 = device.grouped_lin_reg(X, torch.tensor(yv, dtype=dt, device="cuda"), torch.tensor(so, device="cuda"),
                                    add_bias=True, singular_x_tol=1e-6 if f32 else 1e-12)
    assert X.shape[1] == n
    assert torch.equal(s2, status)
    ok = (status == 0).cpu().numpy()
    assert np.array_equal(b2.cpu().numpy()[ok].view(np.uint64), beta.cpu().numpy()[ok].view(np.uint64))


@pytest.mark.parametrize("f32", [True, False], ids=["f32", "f64"])
def test_independence_and_repeats(f32):
    lag = 6
    sizes = [1000, 20_000, 333, 9000]
    offsets = group_offsets(sizes)
    xv = _series(int(offsets[-1]), f32, 5)
    valid = np.ones(len(xv), bool)
    kw = _kwargs(lag, True, "raise", f32)
    a = _fast(_column(xv, valid), offsets, lag, kw, f32)
    for _ in range(3):
        _same(_fast(_column(xv, valid), offsets, lag, kw, f32), a, "repeat")
    x2 = xv.copy()
    x2[offsets[1]:offsets[2]] *= xv.dtype.type(1.5)
    x2[offsets[1] + 7] = xv.dtype.type(3.0)
    b = _fast(_column(x2, valid), offsets, lag, kw, f32)
    for g in (0, 2, 3):
        _same(a.slice(g, 1), b.slice(g, 1), f"group {g}")
    assert not np.array_equal(_bits(a.slice(1, 1))[1], _bits(b.slice(1, 1))[1])
    # the same group alone, and behind other groups, gives the same bits
    for g in range(4):
        lo, hi = offsets[g], offsets[g + 1]
        alone = _fast(_column(xv[lo:hi], valid[lo:hi]), [0, hi - lo], lag, kw, f32)
        _same(alone, a.slice(g, 1), f"group {g} alone")


def test_one_million_groups():
    lag, f32 = 8, True
    n_groups, m = 1_000_000, 100
    offsets = np.arange(n_groups + 1, dtype=np.int64) * m
    rng = np.random.default_rng(3)
    xv = rng.standard_normal(n_groups * m).astype(np.float32)
    valid = np.ones(len(xv), bool)
    kw = _kwargs(lag, True, "raise", f32)
    got = _fast(pa.array(xv), offsets, lag, kw, f32)
    assert len(got) == n_groups and got.null_count == 0
    pick = np.sort(rng.choice(n_groups, 300, replace=False))
    rows = np.concatenate([np.arange(g * m, (g + 1) * m) for g in pick])
    ref = _reference(xv[rows], valid[rows], np.arange(len(pick) + 1, dtype=np.int64) * m, lag, kw, f32)
    _same(got.take(pa.array(pick)), ref, "sampled groups")
