"""group_by(key).agg(lin_reg(target=[...])) on the device: pl_lr_multi_by fits every group's t targets in one launch
sequence, K5's moments pass run once over [y_1 .. y_{t-1}, x.., y_0] and one factorisation per group for all t
right-hand sides.  Checked bit for bit against pl_lr_by run on each target alone, against the CPU oracle and Polars'
per-group loop (one pl_lr_multi call per group) under tests/parity_rule.py, and for group sizes, gating, independence,
nulls, non-finite rows, input errors, the device entry, chunked input and the launch count."""
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
from tests.helpers import group_offsets
from tests.parity_rule import F32_TOL, accept_f32, accept_f64, rel

pytestmark = pytest.mark.gpu

ORC = OracleBackend()


def _data(seed, sizes, p, t, dt):
    """Targets Y (n, t), features X (n, p) of groups of the given sizes in group order, and each row's group id."""
    rng = np.random.default_rng(seed)
    gid = np.repeat(np.arange(len(sizes)), sizes)
    n = len(gid)
    X = rng.standard_normal((n, p)) + 0.3 * np.sin(np.arange(p) + gid[:, None])
    B = np.cos(np.arange(p)[:, None] + 1.7 * np.arange(t)[None, :])
    Y = X @ B + 0.2 * rng.standard_normal((n, t)) + 0.5 * np.cos(gid[:, None] + np.arange(t)[None, :])
    return Y.astype(dt), X.astype(dt), gid


def _xs(p):
    return [f"x{i}" for i in range(p)]


def _expr(p, t, **kw):
    return pds.lin_reg(*_xs(p), target=[f"y{c}" for c in range(t)], **kw)


def _single(p, **kw):
    """pl_lr's kwargs for the same fit of one target (what pl_lr_by is called with)."""
    kw.pop("null_policy", None)
    return pds.lin_reg(*_xs(p), target="y0", **kw).kwargs


def _col(v, chunks=None, mask=None):
    if chunks is None:
        return pa.array(v, mask=mask)
    return pa.chunked_array([pa.array(v[a:b], mask=None if mask is None else mask[a:b])
                             for a, b in zip(chunks[:-1], chunks[1:])])


def _multi(Y, X, offs, kw, f32, chunks=None, ymask=None, xmask=None):
    t, p = Y.shape[1], X.shape[1]
    ins = [pa.array(np.asarray(offs, dtype=np.int64))]
    ins += [_col(Y[:, c], chunks, None if ymask is None else ymask[c]) for c in range(t)]
    ins += [_col(X[:, i], chunks, None if xmask is None else xmask[i]) for i in range(p)]
    names = ["__offsets__"] + [f"target_{c}" for c in range(t)] + _xs(p)
    return _harness.call_plugin("pl_lr_multi_by" + ("_f32" if f32 else ""), ins, names, kw)


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


def _check_against_by(Y, X, offs, kw_multi, kw_by, f32, what, y_for_by=None):
    """Target c of pl_lr_multi_by == pl_lr_by on [y_c, x...] bit for bit (y_for_by(c) replaces y_c there)."""
    res = _multi(Y, X, offs, kw_multi, f32)
    assert res.type.num_fields == Y.shape[1]
    assert [res.type.field(c).name for c in range(Y.shape[1])] == [f"target_{c}" for c in range(Y.shape[1])]
    n_valid = 0
    for c in range(Y.shape[1]):
        ref = _by(Y[:, c] if y_for_by is None else y_for_by(c), X, offs, kw_by, f32)
        n_valid = _same_bits(res.field(c), ref, f"{what} target {c}")
    return res, n_valid


# ---- 1. bit for bit against pl_lr_by per target ----
@pytest.mark.parametrize("p,t", [(8, 3), (12, 4), (40, 8)])
@pytest.mark.parametrize("solver", ["qr", "choleskey"])
@pytest.mark.parametrize("l2", [0.0, 0.5])
@pytest.mark.parametrize("bias", [True, False])
@pytest.mark.parametrize("f64", [True, False])
def test_bits_match_pl_lr_by_per_target(monkeypatch, f64, bias, l2, solver, p, t):
    """(8, 3): both on K5's register kernel; (12, 4) and (40, 8): both on its tile kernel.  Groups of 1, q - 1 and q rows,
    and sizes around K5's 8192-row items.  The groups of up to q + 5 rows are null or not as pl_lr_by's are (the rank gate
    compares |X'X| with the product of its diagonal, which few rows per coefficient bring below the tolerance); from 300
    rows on every group has a fit."""
    monkeypatch.setattr(cfg, "LIN_REG_EXPR_F64", f64)
    q = p + int(bias)
    sizes = [1, q - 1, q, q + 5, 300, 8191, 8192, 8193, 16385]
    Y, X, _ = _data(100 + p + t, sizes, p, t, np.float64 if f64 else np.float32)
    kw = dict(add_bias=bias, l2_reg=l2, solver=solver)
    _, n_valid = _check_against_by(Y, X, group_offsets(sizes), _expr(p, t, **kw).kwargs, _single(p, **kw), not f64,
                                   f"p={p} t={t}")
    assert n_valid >= 5


# ---- 2. against the oracle and Polars' loop ----
def _fast_groups(df, e):
    res = df.group_by("g").agg(e, fast=True)[e.out_name]
    assert pa.types.is_struct(res.type)
    return [{res.type.field(c).name: (None if not res.field(c)[g].is_valid
                                      else np.asarray(res.field(c)[g].as_py(), dtype=np.float64))
             for c in range(res.type.num_fields)} for g in range(len(res))]


def _check_group(monkeypatch, f64, sub, make, got, what):
    monkeypatch.setattr(cfg, "LIN_REG_EXPR_F64", f64)
    loop = PluginBackend().normalize(make(), sub.evaluate(make()))
    o = ORC.eval(sub, make())
    if not f64:
        monkeypatch.setattr(cfg, "LIN_REG_EXPR_F64", True)
        truth = ORC.eval(sub, make())
        monkeypatch.setattr(cfg, "LIN_REG_EXPR_F64", False)
    assert list(got) == list(o) == list(loop), what
    for k, g in got.items():
        assert g is not None and o[k] is not None and loop[k] is not None, (what, k)
        lp = np.asarray(loop[k], np.float64)
        if f64:
            accept_f64(g, o[k], f"{what}:{k}")
            accept_f64(g, lp, f"{what}:{k} loop")
        else:
            _, eo, _ = accept_f32(g, o[k], truth[k], f"{what}:{k}")
            if eo <= F32_TOL:
                assert rel(g, lp) <= F32_TOL, (what, k, "loop", rel(g, lp))


def _frame(Y, X, gid, ymask=None, xmask=None):
    cols = {f"y{c}": pa.array(Y[:, c], mask=None if ymask is None else ymask[c]) for c in range(Y.shape[1])}
    cols |= {f"x{i}": pa.array(X[:, i], mask=None if xmask is None else xmask[i]) for i in range(X.shape[1])}
    return Frame(cols | {"g": gid})


@pytest.mark.parametrize("p,t", [(8, 3), (8, 8), (10, 2), (12, 4), (40, 8), (57, 8)])
@pytest.mark.parametrize("bias", [True, False])
@pytest.mark.parametrize("f64", [True, False])
def test_matches_oracle_and_loop(monkeypatch, f64, bias, p, t):
    """(8, 8) and (10, 2) run the tile kernel here and pl_lr_by's register kernel there; (57, 8) is the widest batched
    fit, p + t = 65.  Every group has ten rows per coefficient or more, so that none meets the rank gate."""
    q = p + int(bias)
    sizes = [10 * q + 3, 2000, 8193]
    Y, X, gid = _data(200 + p + t, sizes, p, t, np.float64 if f64 else np.float32)
    df = _frame(Y, X, gid)
    make = lambda: _expr(p, t, add_bias=bias)       # noqa: E731
    monkeypatch.setattr(cfg, "LIN_REG_EXPR_F64", f64)
    fast = _fast_groups(df, make())
    assert len(fast) == len(sizes)
    for g in range(len(sizes)):
        _check_group(monkeypatch, f64, df.filter(gid == g), make, fast[g],
                     f"{'f64' if f64 else 'f32'} p={p} t={t} bias={bias} group {g}")


# ---- 3. group sizes ----
@pytest.mark.parametrize("p,t", [(8, 3), (12, 4)])
def test_one_group_of_1e5_rows(monkeypatch, p, t):
    monkeypatch.setattr(cfg, "LIN_REG_EXPR_F64", False)
    sizes = [100_000]
    Y, X, gid = _data(7 + p, sizes, p, t, np.float32)
    kw = dict(add_bias=True)
    res, n_valid = _check_against_by(Y, X, group_offsets(sizes), _expr(p, t, **kw).kwargs, _single(p, **kw), True,
                                     "1e5")
    assert n_valid == 1
    _check_group(monkeypatch, False, _frame(Y, X, gid), lambda: _expr(p, t, **kw),
                 _fast_groups(_frame(Y, X, gid), _expr(p, t, **kw))[0], "1e5 rows")


def test_million_groups_of_100_rows():
    n_groups, m, p, t = 1_000_000, 100, 3, 2
    rng = np.random.default_rng(17)
    X = rng.standard_normal((n_groups * m, p), dtype=np.float32)
    Y = np.column_stack([X @ np.array([0.5, -1.0, 0.25], np.float32), X[:, 0] - X[:, 2]])
    Y += 0.1 * rng.standard_normal((n_groups * m, t), dtype=np.float32)
    offs = np.arange(0, n_groups * m + 1, m, dtype=np.int64)
    kw = dict(add_bias=True)
    cfg_f64 = cfg.LIN_REG_EXPR_F64
    try:
        cfg.LIN_REG_EXPR_F64 = False
        kw_multi, kw_by = _expr(p, t, **kw).kwargs, _single(p, **kw)
    finally:
        cfg.LIN_REG_EXPR_F64 = cfg_f64
    res, n_valid = _check_against_by(Y, X, offs, kw_multi, kw_by, True, "1e6 groups")
    assert len(res) == n_groups and n_valid == n_groups
    for g in (0, 4242, n_groups - 1):          # alone, a group gives the same bits
        lo, hi = offs[g], offs[g + 1]
        one = _multi(Y[lo:hi], X[lo:hi], np.array([0, m], dtype=np.int64), kw_multi, True)
        for c in range(t):
            assert one.field(c)[0].values.equals(res.field(c)[g].values), (g, c)


# ---- 4. gating and independence ----
@pytest.mark.parametrize("solver", ["qr", "choleskey"])
@pytest.mark.parametrize("f64", [True, False])
def test_gated_groups_are_null_for_every_target_and_the_others_unchanged(monkeypatch, f64, solver):
    monkeypatch.setattr(cfg, "LIN_REG_EXPR_F64", f64)
    p, t = 5, 3
    sizes = [400, 300, 4, 9000, 500, 2, 700]
    dt = np.float64 if f64 else np.float32
    Y, X, _ = _data(41, sizes, p, t, dt)
    offs = group_offsets(sizes)
    X[offs[1]:offs[2], 3] = X[offs[1]:offs[2], 1]                      # group 1: a duplicated column
    X[offs[4]:offs[5], 2] = 0                                          # group 4: an all-zero column
    kw = dict(add_bias=True, solver=solver)
    km, kb = _expr(p, t, **kw).kwargs, _single(p, **kw)
    res, _ = _check_against_by(Y, X, offs, km, kb, not f64, "gating")
    for c in range(t):
        valid = res.field(c).is_valid().to_pylist()
        assert valid == [True, False, False, True, False, False, True], (c, valid)
    # a different group 3 changes group 3 only
    Y2, X2 = Y.copy(), X.copy()
    Y2[offs[3]:offs[4]] = Y2[offs[3]:offs[4]][::-1] * dt(1.5)
    X2[offs[3]:offs[4]] += dt(0.25)
    res2 = _multi(Y2, X2, offs, km, not f64)
    for c in range(t):
        for g in range(len(sizes)):
            same = res2.field(c)[g].values.equals(res.field(c)[g].values) if res.field(c)[g].is_valid else True
            assert same == (g != 3), (c, g)


# ---- 5. nulls and non-finite values ----
def _error(fn):
    with pytest.raises(pds.PdsbError) as ei:
        fn()
    return str(ei.value)


@pytest.mark.parametrize("f64", [True, False])
def test_null_policies_fail_as_the_loop_does(monkeypatch, f64):
    monkeypatch.setattr(cfg, "LIN_REG_EXPR_F64", f64)
    p, t = 3, 2
    sizes = [50, 60, 70]
    Y, X, gid = _data(51, sizes, p, t, np.float64 if f64 else np.float32)
    n = len(gid)
    null_at = np.arange(n) == 75
    cases = [
        ("raise", None, [null_at, None, None], "Nulls found in data"),
        ("raise", [null_at, None], None, "Nulls found in data"),
        ("skip", None, [null_at, None, None], "The null policy is not supported by multi-target linear regression."),
        ("ignore", [None, null_at], None, "The null policy is not supported by multi-target linear regression."),
        ("zero", [None, null_at], None,
         "Filling null doesn't work for multi-target lstsq when there are nulls in any of the targets."),
        ("1.5", [null_at, None], [null_at, None, None],
         "Filling null doesn't work for multi-target lstsq when there are nulls in any of the targets."),
    ]
    for policy, ymask, xmask, msg in cases:
        df = _frame(Y, X, gid, ymask, xmask)
        e = _expr(p, t, add_bias=True, null_policy=policy)
        loop = _error(lambda: df.group_by("g").agg(e))
        fast = _error(lambda: df.group_by("g").agg(e, fast=True))
        assert fast == loop == f"the plugin failed with message: {msg}", (policy, fast, loop)
    # no null anywhere: every policy fits
    for policy in ("raise", "skip", "ignore", "zero"):
        assert len(_frame(Y, X, gid).group_by("g").agg(_expr(p, t, null_policy=policy), fast=True)["coeffs"]) == 3


@pytest.mark.parametrize("fill", ["zero", "one", "-2.5"])
@pytest.mark.parametrize("f64", [True, False])
def test_fill_with_feature_nulls(monkeypatch, f64, fill):
    """Nulls in the features only are filled: against the loop and the oracle, and bit for bit against pl_lr_by on the
    columns filled beforehand."""
    monkeypatch.setattr(cfg, "LIN_REG_EXPR_F64", f64)
    p, t = 6, 3
    sizes = [500, 3000, 9000]
    dt = np.float64 if f64 else np.float32
    Y, X, gid = _data(53, sizes, p, t, dt)
    rng = np.random.default_rng(54)
    xmask = [rng.random(len(gid)) < 0.05 for _ in range(p)]
    value = {"zero": 0.0, "one": 1.0}.get(fill, None)
    value = dt(float(fill)) if value is None else dt(value)
    Xf = X.copy()
    for i in range(p):
        Xf[xmask[i], i] = value
    kw = dict(add_bias=True)
    res = _multi(Y, X, group_offsets(sizes), _expr(p, t, null_policy=fill, **kw).kwargs, not f64, xmask=xmask)
    for c in range(t):
        _same_bits(res.field(c), _by(Y[:, c], Xf, group_offsets(sizes), _single(p, **kw), not f64),
                   f"{fill} target {c}")
    df = _frame(Y, X, gid, xmask=xmask)
    make = lambda: _expr(p, t, null_policy=fill, **kw)          # noqa: E731
    fast = _fast_groups(df, make())
    for g in range(len(sizes)):
        _check_group(monkeypatch, f64, df.filter(gid == g), make, fast[g], f"fill {fill} group {g}")


@pytest.mark.parametrize("p,t", [(4, 3), (14, 3)])
@pytest.mark.parametrize("f64", [True, False])
def test_nonfinite_rows_are_dropped_for_every_target(monkeypatch, f64, p, t):
    """A NaN or inf anywhere in a row drops the row from its group for every target: bit for bit pl_lr_by on y_c with
    every such row made NaN, and against the oracle on the group without those rows."""
    monkeypatch.setattr(cfg, "LIN_REG_EXPR_F64", f64)
    sizes = [600, 8200, 3000]
    dt = np.float64 if f64 else np.float32
    Y, X, gid = _data(57, sizes, p, t, dt)
    rng = np.random.default_rng(58)
    n = len(gid)
    bad = rng.random(n) < 0.04
    rows = np.flatnonzero(bad)
    for k, r in enumerate(rows):
        v = [np.nan, np.inf, -np.inf][k % 3]
        if k % 2:
            Y[r, k % t] = v
        else:
            X[r, k % p] = v
    kw = dict(add_bias=True)
    offs = group_offsets(sizes)

    def y_dropped(c):
        y = Y[:, c].copy()
        y[bad] = np.nan
        return y

    _check_against_by(Y, X, offs, _expr(p, t, **kw).kwargs, _single(p, **kw), not f64, "non-finite", y_dropped)
    df = _frame(Y, X, gid)
    make = lambda: _expr(p, t, **kw)            # noqa: E731
    fast = _fast_groups(df, make())
    for g in range(len(sizes)):
        _check_group(monkeypatch, f64, df.filter((gid == g) & ~bad), make, fast[g], f"non-finite group {g}")


# ---- 6. bad input ----
@pytest.mark.parametrize("f64", [True, False])
def test_bad_input(f64):
    p, t = 2, 2
    Y, X, _ = _data(61, [10, 10, 10], p, t, np.float64 if f64 else np.float32)
    km, kb = _expr(p, t, add_bias=True).kwargs, _single(p, add_bias=True)
    for offs in ([0, 20, 10, 30], [0, 40, 35, 30], [0, 10, 20, 29], [1, 10, 20, 30]):
        by = _error(lambda: _by(Y[:, 0], X, offs, kb, not f64))
        assert _error(lambda: _multi(Y, X, offs, km, not f64)) == by, offs
    for lt in (0, 4, -3):
        assert _error(lambda: _multi(Y, X, [0, 10, 20, 30], dict(km, last_target_idx=lt), not f64)) == \
            "the plugin failed with message: last_target_idx out of range"
    X58 = np.random.default_rng(62).standard_normal((30, 58)).astype(X.dtype)
    Y8 = np.random.default_rng(63).standard_normal((30, 8)).astype(X.dtype)
    msg = _error(lambda: _multi(Y8, X58, [0, 10, 20, 30], dict(km, last_target_idx=8), not f64))
    assert "8 targets and 58 features" in msg and "1 to 65" in msg, msg
    # p + t = 65 is accepted
    _multi(Y8, X58[:, :57], [0, 10, 20, 30], dict(km, last_target_idx=8), not f64)


# ---- 7. device entry, repeat calls, chunked input, launch count ----
@pytest.mark.parametrize("p,t", [(8, 3), (12, 4)])
@pytest.mark.parametrize("f32", [False, True])
def test_device_entry_matches_the_plugin(f32, p, t):
    sizes = [100, 3, 9000, 40, 8193]
    dt = np.float32 if f32 else np.float64
    Y, X, _ = _data(71, sizes, p, t, dt)
    offs = group_offsets(sizes)
    singular_x_tol = 1e-6 if f32 else 1e-12
    Z = torch.tensor(np.ascontiguousarray(np.column_stack([Y, X]).T), device="cuda")
    beta, status = dev.grouped_lin_reg_multi(Z, torch.tensor(offs, device="cuda"), t, add_bias=True,
                                             singular_x_tol=singular_x_tol)
    torch.cuda.synchronize()
    assert beta.shape == (len(sizes), t, p + 1)
    st = status.cpu().numpy()
    assert st.tolist() == [0, 1, 0, 0, 0]
    b = beta.cpu().numpy()
    assert np.isnan(b[1]).all()
    cfg_f64 = cfg.LIN_REG_EXPR_F64
    try:
        cfg.LIN_REG_EXPR_F64 = not f32
        kw = _expr(p, t, add_bias=True).kwargs
    finally:
        cfg.LIN_REG_EXPR_F64 = cfg_f64
    assert kw["singular_x_tol"] == singular_x_tol
    res = _multi(Y, X, offs, kw, f32)
    for c in range(t):
        for g in (0, 2, 3, 4):
            assert np.array_equal(_bits(np.asarray(res.field(c)[g].as_py(), dt)), _bits(b[g, c].astype(dt))), (c, g)


@pytest.mark.parametrize("f64", [True, False])
def test_repeatable_and_chunked_inputs(f64):
    p, t = 6, 3
    sizes = np.random.default_rng(88).integers(50, 5000, 40).tolist()
    Y, X, _ = _data(89, sizes, p, t, np.float64 if f64 else np.float32)
    n = len(Y)
    offs = group_offsets(sizes)
    kw = _expr(p, t, add_bias=True).kwargs
    one = _multi(Y, X, offs, kw, not f64)
    assert one.equals(_multi(Y, X, offs, kw, not f64))
    assert _multi(Y, X, offs, kw, not f64, chunks=[0, 1, 1000, 1001, n // 2 + 3, n]).equals(one)
    ins = [pa.array(offs)]
    ins += [pa.array(np.concatenate([c[:13], c, c[:5]])).slice(13, n) for c in list(Y.T) + list(X.T)]
    names = ["__offsets__"] + [f"target_{c}" for c in range(t)] + _xs(p)
    assert _harness.call_plugin("pl_lr_multi_by" + ("" if f64 else "_f32"), ins, names, kw).equals(one)


@pytest.mark.parametrize("p,t", [(8, 3), (8, 8), (12, 4)])
def test_no_more_launches_than_pl_lr_by(p, t):
    Y, X, gid = _data(31, [5, 9000, 3, 700], p, t, np.float64)
    offs = group_offsets([5, 9000, 3, 700])
    counts = {}
    for name, call in (("by", lambda: _by(Y[:, 0], X, offs, _single(p, add_bias=True), False)),
                       ("multi", lambda: _multi(Y, X, offs, _expr(p, t, add_bias=True).kwargs, False))):
        c0 = lib().pdsb_kernel_launch_count()
        call()
        counts[name] = lib().pdsb_kernel_launch_count() - c0
    assert 0 < counts["multi"] <= counts["by"], counts
