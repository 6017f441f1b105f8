"""group_by(key).agg(lin_reg(weights=w)) and lin_reg(weights=w, return_pred=True).over(key) on the device: pl_wls_by and
pl_wls_pred_by fit every group's weighted least squares in one launch sequence (K5 with the weighted moments pass).
Checked bit for bit against pl_lr_by with unit weights, against Polars' per-group loop of single weighted pl_lr calls and
the f64 oracle under tests/parity_rule.py, against exact rational solutions on integer data, for the predict pass, the
null policies and error messages of DESIGN §5 item 33, independence, repeatability and the launch count."""
import numpy as np
import pyarrow as pa
import pytest
import torch

import polars_ds_extension_b200 as pds
import polars_ds_extension_b200.config as cfg
from polars_ds_extension_b200 import Frame, _harness
from polars_ds_extension_b200 import device as dev
from polars_ds_extension_b200._lib import lib
from tests.backends import OracleBackend, PluginBackend
from tests.exact_oracle import Design, accept, exact_moments, exact_solve, f32_chain_ok, gram, int_design
from tests.helpers import group_offsets
from tests.parity_rule import F32_TOL, FLOOR, accept_f32, accept_f64, rel

pytestmark = pytest.mark.gpu

ORC = OracleBackend()


def _xs(p):
    return [f"x{i}" for i in range(p)]


def _data(seed, sizes, p, dt, wlo=0.5, whi=2.0):
    """Features X (n, p), target y, positive weights w of groups of the given sizes in group order, each row's group."""
    rng = np.random.default_rng(seed)
    gid = np.repeat(np.arange(len(sizes)), sizes)
    n = len(gid)
    X = rng.standard_normal((n, p)) + 0.3 * np.sin(np.arange(p) + gid[:, None])
    y = X @ np.cos(np.arange(p)) + 0.2 * rng.standard_normal(n) + 0.5 * np.cos(gid)
    w = rng.uniform(wlo, whi, n)
    return X.astype(dt), y.astype(dt), w.astype(dt), gid


def _kw(p, f64, **kw):
    """The kwargs a weighted lin_reg expression carries."""
    f = cfg.LIN_REG_EXPR_F64
    try:
        cfg.LIN_REG_EXPR_F64 = f64
        return pds.lin_reg(*_xs(p), target="y", weights="w", **kw).kwargs
    finally:
        cfg.LIN_REG_EXPR_F64 = f


def _arr(v, mask=None):
    return pa.array(v, mask=mask)


def _wls(w, y, X, offs, kw, f32, pred=False, wmask=None, ymask=None, xmask=None):
    ins = [pa.array(np.asarray(offs, dtype=np.int64)), _arr(w, wmask), _arr(y, ymask)]
    ins += [_arr(X[:, i], None if xmask is None else xmask[i]) for i in range(X.shape[1])]
    sym = ("pl_wls_pred_by" if pred else "pl_wls_by") + ("_f32" if f32 else "")
    return _harness.call_plugin(sym, ins, ["__offsets__", "w", "y"] + _xs(X.shape[1]), kw)


def _by(y, X, offs, kw, f32):
    ins = [pa.array(np.asarray(offs, dtype=np.int64)), pa.array(y)] + [pa.array(X[:, i]) for i in range(X.shape[1])]
    return _harness.call_plugin("pl_lr_by" + ("_f32" if f32 else ""), ins, ["__offsets__", "y"] + _xs(X.shape[1]), kw)


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint32 if a.dtype == np.float32 else np.uint64)


def _same_bits(lst_a, lst_b, what):
    """Two LargeList columns of the same fixed stride: the same validity and the same value bits everywhere."""
    va = np.asarray(lst_a.is_valid().to_numpy(zero_copy_only=False), dtype=bool)
    vb = np.asarray(lst_b.is_valid().to_numpy(zero_copy_only=False), dtype=bool)
    assert np.array_equal(va, vb), f"{what}: validity differs in groups {np.flatnonzero(va != vb)[:10]}"
    a, b = lst_a.values.to_numpy(zero_copy_only=False), lst_b.values.to_numpy(zero_copy_only=False)
    assert a.dtype == b.dtype and a.shape == b.shape, what
    q = len(a) // max(len(lst_a), 1)
    keep = np.repeat(va, q)
    bad = np.flatnonzero(_bits(a)[keep] != _bits(b)[keep])
    assert bad.size == 0, f"{what}: {bad.size} coefficients differ, first at {bad[:5]}"
    return int(va.sum())


def _groups(res):
    return [None if not res[g].is_valid else np.asarray(res[g].as_py(), dtype=np.float64) for g in range(len(res))]


# ---- 1. unit weights: bit for bit pl_lr_by with l2_reg = 0 and singular_x_tol = 0 ----
@pytest.mark.parametrize("p", [1, 4, 8, 10, 11, 40, 64])
@pytest.mark.parametrize("bias", [True, False])
@pytest.mark.parametrize("f64", [True, False])
def test_unit_weights_are_pl_lr_by_bit_for_bit(f64, bias, p):
    """p <= 10 on the register kernel, p >= 11 on the tile kernel; groups of q - 1, q and q + 1 rows, around one trip of
    the register kernel (128 rows) and one 8192-row item, and longer.  w * z == z exactly for w = 1, so every moment is
    the same FMA chain as pl_lr_by's."""
    q = p + int(bias)
    sizes = [q - 1, q, q + 1, 127, 128, 129, 8191, 8192, 8193, 16385, 20000]
    X, y, _, _ = _data(300 + p, sizes, p, np.float64 if f64 else np.float32)
    w = np.ones(len(y), dtype=y.dtype)
    offs = group_offsets(sizes)
    kw = _kw(p, f64, add_bias=bias)
    kw_by = dict(kw, weighted=False, l2_reg=0.0, singular_x_tol=0.0)
    n_valid = _same_bits(_wls(w, y, X, offs, kw, not f64), _by(y, X, offs, kw_by, not f64), f"p={p} bias={bias}")
    assert n_valid >= len(sizes) - 1


# ---- 2. against the per-group loop and the f64 oracle ----
def _frame(X, y, w, gid, wmask=None, ymask=None, xmask=None):
    cols = {f"x{i}": _arr(X[:, i], None if xmask is None else xmask[i]) for i in range(X.shape[1])}
    return Frame(cols | {"y": _arr(y, ymask), "w": _arr(w, wmask), "g": gid})


def _floor32(Xg, wg, bias):
    A = np.column_stack([Xg.astype(np.float64)] + ([np.ones(len(Xg))] if bias else []))
    G = (A * wg.astype(np.float64)[:, None]).T @ A
    return max(FLOOR, float(np.linalg.cond(G)) * 2.0 ** -24)


def _accept(monkeypatch, f64, got, sub, make, floor, what):
    """One group's fast result against the single weighted call (the loop) and the oracle: the parity rule for f64; for
    f32 the grouped report's rule, with the floor max(2e-6, cond(X'WX) 2^-24)."""
    monkeypatch.setattr(cfg, "LIN_REG_EXPR_F64", f64)
    loop = PluginBackend().normalize(make(), sub.evaluate(make()))
    o = ORC.eval(sub, make())
    assert got is not None and loop is not None and o is not None, what
    if f64:
        accept_f64(got, o, what)
        accept_f64(got, np.asarray(loop, np.float64), f"{what} loop")
        return
    monkeypatch.setattr(cfg, "LIN_REG_EXPR_F64", True)
    truth = ORC.eval(sub, make())
    monkeypatch.setattr(cfg, "LIN_REG_EXPR_F64", False)
    if floor <= FLOOR:
        _, eo, _ = accept_f32(got, o, truth, what)
    else:
        eg, eo, ego = rel(got, truth), rel(o, truth), rel(got, o)
        assert eg <= max(eo, floor), f"{what}: {eg:.3e} from the f64 truth, the f32 restatement {eo:.3e}, floor {floor:.3e}"
        if eo <= F32_TOL:
            assert ego <= max(F32_TOL, 2 * floor), f"{what}: |gpu - oracle_f32| = {ego:.3e}"
    if eo <= F32_TOL:
        assert rel(got, loop) <= max(F32_TOL, 2 * floor), (what, "loop", rel(got, loop))


@pytest.mark.parametrize("p", [3, 8, 12, 40])
@pytest.mark.parametrize("bias", [True, False])
@pytest.mark.parametrize("f64", [True, False])
def test_matches_loop_and_oracle(monkeypatch, f64, bias, p):
    q = p + int(bias)
    sizes = [10 * q + 3, 2000, 8193]
    X, y, w, gid = _data(400 + p, sizes, p, np.float64 if f64 else np.float32)
    df = _frame(X, y, w, gid)
    make = lambda: pds.lin_reg(*_xs(p), target="y", add_bias=bias, weights="w")     # noqa: E731
    monkeypatch.setattr(cfg, "LIN_REG_EXPR_F64", f64)
    fast = _groups(df.group_by("g").agg(make(), fast=True)[make().out_name])
    assert len(fast) == len(sizes)
    for g in range(len(sizes)):
        sel = gid == g
        _accept(monkeypatch, f64, fast[g], df.filter(sel), make, _floor32(X[sel], w[sel], bias),
                f"{'f64' if f64 else 'f32'} p={p} bias={bias} group {g}")


# ---- 3. exact data ----
@pytest.mark.parametrize("p,bias", [(1, True), (3, True), (8, False), (10, True), (12, True), (30, False)])
def test_exact_integer_data(p, bias):
    """Integer X in [-8, 8], |y| <= 72 and weights 1..4: every moment is an integer the f64 and f32 chains (at most 260
    rows per lane, or 32-row tiles) sum exactly, and beta is held to exact_oracle.accept against the exact rational
    solution."""
    q = p + int(bias)
    sizes = [q - 1, q + 2, 50, 300, 9000]
    offs = group_offsets(sizes)
    d = int_design(900 + p, int(offs[-1]), p, tag=False, weights=True)
    for dtype in (torch.float64, torch.float32):
        if dtype == torch.float32 and not f32_chain_ok(d, 8192 // 32 + 128):
            continue
        X = torch.from_numpy(np.ascontiguousarray(d.X.T.astype(np.float64))).to(dtype).cuda()
        y = torch.from_numpy(d.Y[:, 0].astype(np.float64)).to(dtype).cuda()
        w = torch.from_numpy(d.w.astype(np.float64)).to(dtype).cuda()
        beta, status = dev.grouped_wls_lin_reg(X, y, w, torch.from_numpy(offs).cuda(), add_bias=bias)
        beta, status = beta.cpu().numpy(), status.cpu().numpy()
        for g, (s, e) in enumerate(zip(offs[:-1], offs[1:])):
            if e - s < q:
                assert status[g] != 0 and np.isnan(beta[g]).all(), (dtype, g)
                continue
            M = exact_moments(Design(d.X[s:e], d.Y[s:e], d.w[s:e]))
            G, b = gram(M, p, 1, bias)
            assert status[g] == 0, (dtype, g)
            accept(beta[g], exact_solve(G, b), G, b, "qr", f"{dtype} p={p} group {g}")


# ---- 4. predictions ----
@pytest.mark.parametrize("p", [4, 12])
@pytest.mark.parametrize("f64", [True, False])
def test_pred_rows_are_the_predict_pass_on_the_fit(f64, p):
    dt = np.float64 if f64 else np.float32
    sizes = [p, 3000, 1, 9000, 257]
    X, y, w, _ = _data(500 + p, sizes, p, dt)
    offs = group_offsets(sizes)
    res = _wls(w, y, X, offs, _kw(p, f64, add_bias=True, return_pred=True), not f64, pred=True)
    Xt = torch.from_numpy(np.ascontiguousarray(X.T)).cuda()
    yt, wt, ot = torch.from_numpy(y).cuda(), torch.from_numpy(w).cuda(), torch.from_numpy(offs).cuda()
    beta, status = dev.grouped_wls_lin_reg(Xt, yt, wt, ot, add_bias=True)
    pred, resid, valid = dev.grouped_predict(Xt, yt, ot, beta, status, add_bias=True)
    v = valid.cpu().numpy().astype(bool)
    assert np.array_equal(np.asarray(res.field("pred").is_valid().to_numpy(zero_copy_only=False), bool), v)
    for name, ref in (("pred", pred), ("resid", resid)):
        got = res.field(name).to_numpy(zero_copy_only=False)
        assert np.array_equal(_bits(got[v]), _bits(ref.cpu().numpy()[v])), name
    # the same coefficients as pl_wls_by
    coeffs = _wls(w, y, X, offs, _kw(p, f64, add_bias=True), not f64)
    for g in range(len(sizes)):
        if status[g].item() == 0:
            assert np.array_equal(np.asarray(coeffs[g].as_py(), dt), beta[g].cpu().numpy().astype(dt)), g


@pytest.mark.parametrize("f64", [True, False])
def test_over_matches_the_loop(monkeypatch, f64):
    p = 5
    sizes = [400, 2500, 9000]
    X, y, w, gid = _data(600, sizes, p, np.float64 if f64 else np.float32)
    perm = np.random.default_rng(601).permutation(len(y))
    df = _frame(X[perm], y[perm], w[perm], gid[perm])
    monkeypatch.setattr(cfg, "LIN_REG_EXPR_F64", f64)
    e = pds.lin_reg(*_xs(p), target="y", add_bias=True, weights="w", return_pred=True)
    fast, loop = (df.select(e.over("g", fast=f))[e.out_name] for f in (True, False))
    for k in ("pred", "resid"):
        a, b = (r.field(k).to_numpy(zero_copy_only=False) for r in (fast, loop))
        assert fast.field(k).null_count == loop.field(k).null_count == 0
        for g in range(len(sizes)):
            sel = gid[perm] == g
            floor = F32_TOL if f64 else max(F32_TOL, 2 * _floor32(X[gid == g], w[gid == g], True))
            assert rel(a[sel], b[sel]) <= (1e-6 if f64 else floor), (k, g, rel(a[sel], b[sel]))


# ---- 5. errors and nulls ----
def _error(fn):
    with pytest.raises(pds.PdsbError) as ei:
        fn()
    return str(ei.value)


def _fast_and_loop(df, e):
    return (lambda: df.group_by("g").agg(e, fast=True)), (lambda: df.group_by("g").agg(e, fast=False))


@pytest.mark.parametrize("f64", [True, False])
def test_failures_match_the_loop(monkeypatch, f64):
    """Every failure of Polars' loop, with its message, for coefficients and predictions."""
    monkeypatch.setattr(cfg, "LIN_REG_EXPR_F64", f64)
    p, sizes = 3, [40, 50, 60]
    X, y, w, gid = _data(700, sizes, p, np.float64 if f64 else np.float32)
    n = len(y)
    ynull = np.zeros(n, bool)
    ynull[55] = True                                  # group 1
    xnull = [np.zeros(n, bool) for _ in range(p)]
    xnull[1][95] = True                               # group 2
    cases = [
        ("raise, null y", dict(ymask=ynull), "raise", "Nulls found in data"),
        ("raise, null x", dict(xmask=xnull), "raise", "Nulls found in data"),
        ("skip, null y", dict(ymask=ynull), "skip", "Shape of weights is not the same as the data."),
        ("skip, null x", dict(xmask=xnull), "skip", "Shape of weights is not the same as the data."),
        ("fill, null y", dict(ymask=ynull), "0.5", "Shape of weights is not the same as the data."),
    ]
    for what, masks, policy, msg in cases:
        df = _frame(X, y, w, gid, **masks)
        for ret in (False, True):
            e = pds.lin_reg(*_xs(p), target="y", add_bias=True, weights="w", null_policy=policy, return_pred=ret)
            if ret:
                fast = lambda: df.select(e.over("g", fast=True))          # noqa: E731
                loop = lambda: df.select(e.over("g", fast=False))         # noqa: E731
            else:
                fast, loop = _fast_and_loop(df, e)
            fe, le = _error(fast), _error(loop)
            assert fe == le and msg in fe, (what, ret, fe, le)
    # small weights: the single call counts fewer rows than coefficients
    df = _frame(X, y, np.full(n, 0.01, X.dtype), gid, ymask=ynull)
    fast, loop = _fast_and_loop(df, pds.lin_reg(*_xs(p), target="y", add_bias=True, weights="w"))
    assert _error(fast) == _error(loop) and "#Data < #features" in _error(fast)
    # a weight column of another length
    short = lambda: _wls(w[:-1], y, X, group_offsets(sizes), _kw(p, f64, add_bias=True), not f64)     # noqa: E731
    assert "Shape of weights is not the same as the data." in _error(short)


@pytest.mark.parametrize("f64", [True, False])
def test_fills_and_null_weights(monkeypatch, f64):
    """A fill of the features runs and matches the loop.  A null weight, and a null y or x under "ignore", arrive as NaN
    and drop their row, as a NaN value does (pl_lr_by's rule): that group's fit is the fit of its other rows, and the
    other groups are bit for bit the fit without the nulls."""
    monkeypatch.setattr(cfg, "LIN_REG_EXPR_F64", f64)
    p, sizes = 3, [400, 500, 600]
    X, y, w, gid = _data(710, sizes, p, np.float64 if f64 else np.float32)
    n = len(y)
    offs = group_offsets(sizes)
    xnull = [np.zeros(n, bool) for _ in range(p)]
    xnull[0][[3, 450]] = True                         # groups 0 and 1
    wnull = np.zeros(n, bool)
    wnull[1000] = True                                # group 2
    kw = _kw(p, f64, add_bias=True)
    base = _groups(_wls(w, y, X, offs, kw, not f64))
    df = _frame(X, y, w, gid, xmask=xnull)
    e = pds.lin_reg(*_xs(p), target="y", add_bias=True, weights="w", null_policy="0.25")
    fast = _groups(df.group_by("g").agg(e, fast=True)[e.out_name])
    loop = df.group_by("g").agg(e, fast=False)[e.out_name]
    for g in range(len(sizes)):
        assert rel(fast[g], np.asarray(loop[g][0].as_py(), np.float64)) <= (1e-6 if f64 else F32_TOL), g
    for policy, masks, dropped in (("ignore", dict(xmask=xnull), [3, 450]), ("skip", dict(wmask=wnull), [1000]),
                                   ("ignore", dict(wmask=wnull), [1000])):
        df = _frame(X, y, w, gid, **masks)
        e = pds.lin_reg(*_xs(p), target="y", add_bias=True, weights="w", null_policy=policy)
        fast = _groups(df.group_by("g").agg(e, fast=True)[e.out_name])
        keep = np.ones(n, bool)
        keep[dropped] = False
        for g in range(len(sizes)):
            s, t = offs[g], offs[g + 1]
            if keep[s:t].all():
                assert np.array_equal(fast[g], base[g]), (policy, g)
                continue
            k = keep[s:t]
            one = _groups(_wls(w[s:t][k], y[s:t][k], X[s:t][k], [0, int(k.sum())], kw, not f64))[0]
            assert rel(fast[g], one) <= (1e-12 if f64 else F32_TOL), (policy, g, rel(fast[g], one))


@pytest.mark.parametrize("f64", [True, False])
def test_nonfinite_rows_drop_and_short_groups_are_null(f64):
    """A NaN / inf in a kept row's x, y or w drops that row (pl_lr_by's rule): the group's fit is the fit of the other
    rows.  A group with fewer kept rows than coefficients, an empty group included, is null."""
    p, dt = 4, np.float64 if f64 else np.float32
    sizes = [300, 300, 300, 300, 0, 6, 300]
    X, y, w, _ = _data(720, sizes, p, dt)
    offs = group_offsets(sizes)
    X[10, 1] = np.nan                                 # group 0
    y[320] = np.inf                                   # group 1
    w[650] = np.nan                                   # group 2
    w[920] = -np.inf                                  # group 3
    w[1200:1203] = np.nan                             # group 5: 3 kept rows < q = 5
    kw = _kw(p, f64, add_bias=True)
    got = _groups(_wls(w, y, X, offs, kw, not f64))
    assert got[4] is None and got[5] is None and all(got[g] is not None for g in (0, 1, 2, 3, 6))
    bad = ~(np.isfinite(X).all(axis=1) & np.isfinite(y) & np.isfinite(w))
    for g in (0, 1, 2, 3):
        s, e = offs[g], offs[g + 1]
        keep = ~bad[s:e]
        one = _groups(_wls(w[s:e][keep], y[s:e][keep], X[s:e][keep], [0, int(keep.sum())], kw, not f64))[0]
        assert rel(got[g], one) <= (1e-12 if f64 else F32_TOL), (g, rel(got[g], one))


# ---- 6. independence, repeatability and cost ----
@pytest.mark.parametrize("f64", [True, False])
def test_a_group_is_the_same_whatever_shares_the_call(f64):
    p, dt = 6, np.float64 if f64 else np.float32
    sizes = [500, 9000, 3, 20000, 128, 700]
    X, y, w, _ = _data(730, sizes, p, dt)
    offs = group_offsets(sizes)
    kw = _kw(p, f64, add_bias=True)
    res = _wls(w, y, X, offs, kw, not f64)
    assert res.equals(_wls(w, y, X, offs, kw, not f64))
    for g in (0, 1, 3, 5):
        s, e = offs[g], offs[g + 1]
        one = _wls(w[s:e], y[s:e], X[s:e], [0, e - s], kw, not f64)
        assert one[0].values.equals(res[g].values), g
    # another group's data changes that group only
    X2 = X.copy()
    X2[offs[3]:offs[4]] *= dt(1.5)
    res2 = _wls(w, y, X2, offs, kw, not f64)
    for g in range(len(sizes)):
        same = res2[g].values.equals(res[g].values) if res[g].is_valid else not res2[g].is_valid
        assert same == (g != 3), g


@pytest.mark.parametrize("p", [5, 20])
def test_as_many_launches_as_pl_lr_by(p):
    sizes = [5, 9000, 3, 700]
    X, y, w, _ = _data(740, sizes, p, np.float64)
    offs = group_offsets(sizes)
    kw = _kw(p, True, add_bias=True)
    counts = {}
    for name, call in (("by", lambda: _by(y, X, offs, dict(kw, weighted=False), False)),
                       ("wls", lambda: _wls(w, y, X, offs, kw, False))):
        c0 = lib().pdsb_kernel_launch_count()
        call()
        counts[name] = lib().pdsb_kernel_launch_count() - c0
    assert counts["wls"] == counts["by"] > 0, counts


def test_million_groups_of_100_rows():
    n_groups, m, p = 1_000_000, 100, 3
    rng = np.random.default_rng(750)
    X = rng.standard_normal((n_groups * m, p), dtype=np.float32)
    y = X @ np.array([0.5, -1.0, 0.25], np.float32) + 0.1 * rng.standard_normal(n_groups * m, dtype=np.float32)
    w = rng.uniform(0.5, 2.0, n_groups * m).astype(np.float32)
    offs = np.arange(0, n_groups * m + 1, m, dtype=np.int64)
    kw = _kw(p, False, add_bias=True)
    res = _wls(w, y, X, offs, kw, True)
    assert len(res) == n_groups and res.null_count == 0
    for g in (0, 4242, n_groups - 1):
        lo, hi = offs[g], offs[g + 1]
        assert _wls(w[lo:hi], y[lo:hi], X[lo:hi], [0, m], kw, True)[0].values.equals(res[g].values), g
