"""group_by(key).agg(lin_reg_report) on the device (K17): pl_lin_reg_report_by reports every group in one launch
sequence.  Checked against Polars' per-group loop (fast=False: one pl_lin_reg_report call per group, var(y) from
t.var()) and against the CPU oracle per group, at a leverage of 0.9, with skipped nulls, for independence from the
other groups and reproducibility, for its error messages, and K9 (the single report, whose per-row HC weight and
finalize rule K17 shares) against the bits it returned before the two rules were shared.

f32 groups: pass 1 is pl_lr_by's (f32 products summed in short f32 chains, then f64), so a group's normal equations
carry f32 rounding amplified by cond(X'X).  The parity rule's floor (2e-6, two correctly rounded f32 answers) is
therefore taken as max(2e-6, cond(X'X) 2^-24) of the group's kept rows, and for the fields that depend on an hc2 / hc3
standard error (se, t, p, the interval) times 1 + k / (1 - max h) (k = 1 for hc2, 2 for hc3), the amplification of an
error in the leverage h by 1 / (1 - h)^k.  For a well-conditioned group that is the rule as written; only the few-row
groups (q + 1 rows and the like) get a wider floor."""
from pathlib import Path

import numpy as np
import pyarrow as pa
import pytest
import torch

import polars_ds_extension_b200 as pds
import polars_ds_extension_b200.config as cfg
from polars_ds_extension_b200 import Frame, _harness
from polars_ds_extension_b200 import device as dev
from tests.backends import OracleBackend
from tests.helpers import chunked, group_offsets
from tests.parity_rule import F32_TOL, FLOOR, accept_f32, accept_f64, rel

pytestmark = pytest.mark.gpu

ORC = OracleBackend()
STD_ERRS = ["se", "hc0", "hc1", "hc2", "hc3"]
SE_NAME = {"se": "std_err", "hc0": "hc0_se", "hc1": "hc1_se", "hc2": "hc2_se", "hc3": "hc3_se"}
FIELDS = ["beta", "SE", "t", "p>|t|", "0.025", "0.975", "r2", "adj_r2"]


def _groups(seed, sizes, p, dt):
    """y, X, group ids, rows in group order: per group y = X beta_g + b_g + heteroscedastic noise, every beta_g
    coefficient away from zero."""
    rng = np.random.default_rng(seed)
    ys, Xs = [], []
    for g, m in enumerate(sizes):
        X = rng.standard_normal((m, p)) + 0.3 * np.sin(np.arange(p) + g)
        beta = (0.6 + 0.3 * np.cos(np.arange(p) + 2 * g)) * np.where(np.arange(p) % 2, 1.0, -1.0)
        y = X @ beta + 0.5 * np.cos(g) + 0.5 * rng.standard_normal(m) * (1.0 + 0.5 * np.abs(X[:, 0]))
        ys.append(y)
        Xs.append(X)
    return np.concatenate(ys).astype(dt), np.concatenate(Xs).astype(dt), np.repeat(np.arange(len(sizes)), sizes)


def _frame(y, X, gid, **extra):
    return Frame({"y": y} | {f"x{i}": X[:, i] for i in range(X.shape[1])} | {"g": gid} | extra)


def _expr(p, **kw):
    return pds.lin_reg_report(*[f"x{i}" for i in range(p)], target="y", **kw)


def _rep(sa, se):
    """A report struct array -> {field: values}, the std_err field under "SE"."""
    d = {f.name: sa.field(i) for i, f in enumerate(sa.type)}
    out = {"features": d["features"].to_pylist()}
    for k in FIELDS:
        out[k] = d[SE_NAME[se] if k == "SE" else k].to_numpy(zero_copy_only=False).astype(np.float64)
    return out


def _fast(df, e, se):
    res = df.group_by("g").agg(e, fast=True)[e.out_name or e.symbol]
    return [None if not res[i].is_valid else _rep(res[i].values, se) for i in range(len(res))]


def _slow(df, e, se):
    return [_rep(r, se) for r in df.group_by("g").agg(e, fast=False)[e.out_name or e.symbol]]


def _oracle(sub, e, se):
    o = ORC.eval(sub, e)
    out = {"features": o["features"]}
    for k in FIELDS:
        out[k] = np.broadcast_to(np.asarray(o[SE_NAME[se] if k == "SE" else k], np.float64), o["beta"].shape)
    return out


def _call_by(y, X, offsets, kw, chunks=1, f32=False):
    ins = ([pa.array(np.asarray(offsets, dtype=np.int64)), chunked(y, chunks)]
           + [chunked(X[:, i], chunks) for i in range(X.shape[1])])
    names = ["__offsets__", "y"] + [f"x{i}" for i in range(X.shape[1])]
    return _harness.call_plugin("pl_lin_reg_report_by" + ("_f32" if f32 else ""), ins, names, kw)


def _finite_parts(what, *vs):
    """The non-finite entries (inf / NaN) must sit at the same places with the same values; returns the finite mask."""
    fin = np.isfinite(vs[0])
    for v in vs[1:]:
        assert np.array_equal(np.isfinite(v), fin), what
        assert np.array_equal(v[~fin], vs[0][~fin], equal_nan=True), what
    return fin


def _floor32(Xg, bias, se):
    """The f32 floors (the fields without, with the standard error) of a group with kept rows Xg."""
    A = np.column_stack([Xg.astype(np.float64)] + ([np.ones(len(Xg))] if bias else []))
    G = A.T @ A
    base = max(FLOOR, float(np.linalg.cond(G)) * 2.0 ** -24)
    k = {"hc2": 1, "hc3": 2}.get(se, 0)
    if not k:
        return base, base
    h = np.einsum("ij,ji->i", A, np.linalg.solve(G, A.T))
    return base, base * (1.0 + k / max(1.0 - float(h.max()), 1e-12))


def _accept32(g, o32, truth, floor, what):
    if floor <= FLOOR:
        return accept_f32(g, o32, truth, what)[1]
    eg, eo, ego = rel(g, truth), rel(o32, truth), rel(g, o32)
    assert eg <= max(eo, floor), f"{what}: {eg:.3e} from the f64 truth, the f32 restatement {eo:.3e}, floor {floor:.3e}"
    if eo <= F32_TOL:
        assert ego <= max(F32_TOL, 2 * floor), f"{what}: |gpu - oracle_f32| = {ego:.3e}"
    return eo


def _check(f64, got, loop, o, truth, what, floors=(FLOOR, FLOOR)):
    """Every field of a group's report: against the oracle by the parity rule (p-values by the ln p rule of
    test_gpu_wide._assert_report) and against the per-group loop.  floors: the f32 floors of the group (_floor32)."""
    assert got["features"] == loop["features"] == o["features"], what
    for k in FIELDS:
        floor = floors[1] if k in ("SE", "t", "p>|t|", "0.025", "0.975") else floors[0]
        g, lp, ov, tv = got[k], loop[k], o[k], truth[k]
        fin = _finite_parts(f"{what}:{k}", g, lp, ov, tv)
        if not fin.any():
            continue
        g, lp, ov, tv = g[fin], lp[fin], ov[fin], tv[fin]
        if k == "p>|t|":
            lg, lo, lt, ll = (np.log(np.maximum(v, 1e-300)) for v in (g, ov, tv, lp))
            eg, eo = np.max(np.abs(lg - lt) / np.abs(lt)), np.max(np.abs(lo - lt) / np.abs(lt))
            assert eg <= (1e-6 if f64 else max(eo, floor)), (what, k, eg, eo)
            if f64 or eo <= F32_TOL:
                assert np.max(np.abs(lg - ll) / np.abs(ll)) <= (1e-6 if f64 else max(F32_TOL, 2 * floor)), \
                    (what, k, "loop")
            continue
        if f64:
            accept_f64(g, ov, f"{what}:{k}")
            accept_f64(g, lp, f"{what}:{k} loop")
        else:
            eo = _accept32(g, ov, tv, floor, f"{what}:{k}")
            if eo <= F32_TOL:            # a group the f32 restatement itself resolves: the loop must agree too
                assert rel(g, lp) <= max(F32_TOL, 2 * floor), (what, k, "loop", rel(g, lp))


def _three(monkeypatch, f64, sub, make, se):
    monkeypatch.setattr(cfg, "LIN_REG_EXPR_F64", f64)
    o = _oracle(sub, make(), se)
    if f64:
        return o, o
    monkeypatch.setattr(cfg, "LIN_REG_EXPR_F64", True)
    truth = _oracle(sub, make(), se)
    monkeypatch.setattr(cfg, "LIN_REG_EXPR_F64", False)
    return o, truth


def _compare_all(monkeypatch, f64, df, gid, X, bias, make, se, sizes, q, what):
    monkeypatch.setattr(cfg, "LIN_REG_EXPR_F64", f64)
    e = make()
    fast, slow = _fast(df, e, se), _slow(df, e, se)
    assert len(fast) == len(slow) == len(sizes)
    for g, m in enumerate(sizes):
        assert fast[g] is not None, (what, g)
        if m == q:
            # no residual degree of freedom: only beta is defined (the rest is rounding noise divided by zero), and
            # in f32 a square system of random rows resolves it too coarsely to compare
            assert fast[g]["features"] == slow[g]["features"]
            if f64:
                assert rel(fast[g]["beta"], slow[g]["beta"]) <= 1e-6, (what, g)
            continue
        o, truth = _three(monkeypatch, f64, df.filter(gid == g), make, se)
        monkeypatch.setattr(cfg, "LIN_REG_EXPR_F64", f64)
        floors = (FLOOR, FLOOR) if f64 else _floor32(X[gid == g], bias, se)
        _check(f64, fast[g], slow[g], o, truth, f"{what} group {g} ({m} rows)", floors)


# ---- 1. fast group_by against the loop and the oracle, group sizes on both sides of the item boundaries ----
@pytest.mark.parametrize("f64", [True, False])
@pytest.mark.parametrize("bias", [True, False])
@pytest.mark.parametrize("p", [1, 4, 8, 10, 11, 40, 64])
def test_fast_report_matches_loop_and_oracle(monkeypatch, f64, bias, p):
    q = p + int(bias)
    sizes = [q, q + 1, 127, 128, 129, 1000, 8191, 8192, 8193, 16385, 20000]
    y, X, gid = _groups(300 + p, sizes, p, np.float64 if f64 else np.float32)
    df = _frame(y, X, gid)
    for se in STD_ERRS:
        _compare_all(monkeypatch, f64, df, gid, X, bias, lambda: _expr(p, add_bias=bias, std_err=se), se, sizes, q,
                     f"{'f64' if f64 else 'f32'} p={p} bias={bias} {se}")


# ---- 2. hc2 / hc3 with a row of leverage 0.9 ----
@pytest.mark.parametrize("se", ["hc2", "hc3"])
@pytest.mark.parametrize("p", [4, 11])
def test_high_leverage_row(monkeypatch, se, p):
    from tests.test_gpu_wide import _high_leverage

    sizes = [500, 700, 900]
    y, X, gid = _groups(41 + p, sizes, p, np.float64)
    xs = [f"x{i}" for i in range(p)]
    lo, hi = 500, 1200
    sub = _high_leverage(Frame({c: X[lo:hi, i] for i, c in enumerate(xs)}), xs, p)
    X = X.copy()
    for i, c in enumerate(xs):
        X[lo:hi, i] = sub[c].to_numpy()
    A = np.column_stack([X[lo:hi], np.ones(hi - lo)])
    assert abs(A[0] @ np.linalg.solve(A.T @ A, A[0]) - 0.9) < 1e-9
    _compare_all(monkeypatch, True, _frame(y, X, gid), gid, X, True, lambda: _expr(p, add_bias=True, std_err=se), se,
                 sizes, p + 1, f"leverage {se} p={p}")


# ---- 3. nulls with "skip" ----
@pytest.mark.parametrize("f64", [True, False])
@pytest.mark.parametrize("se", ["se", "hc1", "hc3"])
def test_skipped_nulls(monkeypatch, f64, se):
    p = 5
    sizes = [400, 900, 3000, 9000, 60, 12]
    dt = np.float64 if f64 else np.float32
    y, X, gid = _groups(61, sizes, p, dt)
    rng = np.random.default_rng(62)
    n = len(y)
    xnull = [rng.random(n) < 0.05 for _ in range(p)]
    ynull = rng.random(n) < 0.05
    o = group_offsets(np.bincount(gid))
    # group 1: y is set on rows where x0 is null, so var(y) spans rows the fit drops
    xnull[0][o[1]:o[1] + 200] = True
    ynull[o[1]:o[1] + 200] = False
    # group 4: 60 rows, all but 4 dropped (fewer kept rows than coefficients -> a null list)
    xnull[2][o[4]:o[4] + 56] = True
    cols = {"y": pa.array(y, mask=ynull)} | {f"x{i}": pa.array(X[:, i], mask=xnull[i]) for i in range(p)}
    df = Frame(cols | {"g": gid})
    monkeypatch.setattr(cfg, "LIN_REG_EXPR_F64", f64)
    make = lambda: _expr(p, add_bias=True, std_err=se, null_policy="skip")     # noqa: E731
    e = make()
    fast, slow = _fast(df, e, se), _slow(df, e, se)
    assert fast[4] is None
    for g in (0, 1, 2, 3, 5):
        assert fast[g] is not None, g
        o_, truth = _three(monkeypatch, f64, df.filter(gid == g), make, se)
        monkeypatch.setattr(cfg, "LIN_REG_EXPR_F64", f64)
        kept = (gid == g) & ~ynull & ~np.any(np.column_stack(xnull), axis=1)
        floors = (FLOOR, FLOOR) if f64 else _floor32(X[kept], True, se)
        _check(f64, fast[g], slow[g], o_, truth, f"nulls {se} group {g}", floors)
    # the loop's r2 uses var(y) over every non-null y of the group, rows with a null x included
    assert rel(fast[1]["r2"], slow[1]["r2"]) <= (1e-12 if f64 else 1e-5)


@pytest.mark.parametrize("f32", [False, True])
def test_empty_group_through_the_abi(f32):
    p = 3
    dt = np.float32 if f32 else np.float64
    y, X, gid = _groups(71, [300, 500], p, dt)
    offs = np.array([0, 0, 300, 300, 800, 800], dtype=np.int64)          # groups 0, 2 and 4 are empty
    kw = _expr(p, add_bias=True, std_err="hc1").kwargs
    res = _call_by(y, X, offs, kw, f32=f32)
    assert pa.types.is_large_list(res.type) and len(res) == 5
    assert [res[i].is_valid for i in range(5)] == [False, True, False, True, False]
    assert res.null_count == 3
    ref = _call_by(y, X, np.array([0, 300, 800], dtype=np.int64), kw, f32=f32)
    for a, b in ((1, 0), (3, 1)):
        assert res[a].values.equals(ref[b].values)
    item = res.type.value_type
    assert item.field(2).name == "hc1_se" and item.field(1).type == (pa.float32() if f32 else pa.float64())
    assert res[1].values.field("features").to_pylist() == ["x0", "x1", "x2", "__bias__"]


# ---- 4. independence, reproducibility, chunked inputs ----
@pytest.mark.parametrize("f64", [True, False])
@pytest.mark.parametrize("se", ["se", "hc3"])
def test_independent_reproducible_and_chunk_invariant(f64, se):
    p = 8
    sizes = [129, 8193, 3000, 20000, 77]
    dt = np.float64 if f64 else np.float32
    y, X, gid = _groups(91, sizes, p, dt)
    offs = group_offsets(np.bincount(gid))
    kw = _expr(p, add_bias=True, std_err=se).kwargs
    f32 = not f64
    a = _call_by(y, X, offs, kw, f32=f32)
    b = _call_by(y, X, offs, kw, f32=f32)
    assert a.equals(b)
    c = _call_by(y, X, offs, kw, chunks=7, f32=f32)
    assert a.equals(c)
    y2, X2 = y.copy(), X.copy()
    lo, hi = offs[2], offs[3]
    y2[lo:hi] = y2[lo:hi][::-1] * dt(1.5)
    X2[lo:hi] = X2[lo:hi] + dt(0.25)
    d = _call_by(y2, X2, offs, kw, f32=f32)
    for g in range(len(sizes)):
        if g == 2:
            assert not d[g].values.equals(a[g].values)
        else:
            assert d[g].values.equals(a[g].values), g


def test_device_entry_matches_the_plugin():
    p, se = 6, 4
    sizes = [100, 6, 9000]
    y, X, gid = _groups(95, sizes, p, np.float64)
    offs = group_offsets(np.bincount(gid))
    out, status = dev.grouped_report(torch.tensor(X.T.copy(), device="cuda"), torch.tensor(y, device="cuda"),
                                     torch.tensor(offs, device="cuda"), add_bias=True, se_type=se)
    assert status.cpu().tolist() == [0, 1, 0]
    o = out.cpu().numpy()
    assert np.isnan(o[1]).all()
    res = _call_by(y, X, offs, _expr(p, add_bias=True, std_err="hc3").kwargs)
    for g in (0, 2):
        v = res[g].values
        got = np.stack([v.field(i).to_numpy(zero_copy_only=False) for i in range(1, 9)])
        assert np.array_equal(got, o[g])



@pytest.mark.parametrize("se", [0, 3])
@pytest.mark.parametrize("p", [4, 14])
def test_device_entry_launch_count(p, se):
    """Seven launches whatever p and std_err: one work list (count, scan, item -> rows and group) shared by the moments
    pass and pass 3, the moments, the solve, pass 3 and the finalize."""
    from polars_ds_extension_b200._lib import lib

    y, X, gid = _groups(43, [200, 9000, 5], p, np.float64)
    c0 = lib().pdsb_kernel_launch_count()
    dev.grouped_report(torch.tensor(X.T.copy(), device="cuda"), torch.tensor(y, device="cuda"),
                       torch.tensor(group_offsets(np.bincount(gid)), device="cuda"), add_bias=True, se_type=se)
    assert lib().pdsb_kernel_launch_count() - c0 == 7

# ---- 5. errors ----
def test_errors(monkeypatch):
    p = 3
    y, X, gid = _groups(97, [50, 60], p, np.float64)
    kw = _expr(p, add_bias=True).kwargs
    with pytest.raises(pds.PdsbError, match="bad group offsets"):
        _call_by(y, X, np.array([0, 50, 100], dtype=np.int64), kw)
    with pytest.raises(pds.PdsbError, match="non-decreasing"):
        _call_by(y, X, np.array([0, 70, 60, 110], dtype=np.int64), kw)
    ym = pa.array(y, mask=np.arange(len(y)) == 3)
    ins = [pa.array(group_offsets(np.bincount(gid))), ym] + [pa.array(X[:, i]) for i in range(p)]
    names = ["__offsets__", "y"] + [f"x{i}" for i in range(p)]
    with pytest.raises(pds.PdsbError, match="Nulls found in data"):
        _harness.call_plugin("pl_lin_reg_report_by", ins, names, kw)
    with pytest.raises(pds.PdsbError, match="only null_policy='skip'"):
        _harness.call_plugin("pl_lin_reg_report_by", ins, names, kw | {"null_policy": "zero"})
    with pytest.raises(pds.PdsbError, match="weighted fits are not batched"):
        _call_by(y, X, group_offsets(np.bincount(gid)), kw | {"weighted": True})
    df = _frame(y, X, gid, w=np.ones(len(y)))
    with pytest.raises(ValueError, match="fast group_by is only available for lin_reg coefficients"):
        df.group_by("g").agg(pds.lin_reg_report("x0", target="y", weights="w"), fast=True)
    X65 = np.random.default_rng(98).standard_normal((len(y), 65))
    with pytest.raises(pds.PdsbError, match="at most 64"):
        _call_by(y, X65, group_offsets(np.bincount(gid)), kw)


# ---- 6. K9 unchanged ----
def test_single_report_bits_unchanged():
    from tests.golden import make_report_bits as mk

    golden = np.load(Path(__file__).parent / "golden" / "report_bits.npz")
    assert len(golden.files) == len(mk.CASES) * len(mk.STD_ERRS)
    try:
        for dt, bias, pol in mk.CASES:
            cfg.LIN_REG_EXPR_F64 = dt == "f64"
            df, xs = mk.report_frame(dt, pol == "skip")
            for se in mk.STD_ERRS:
                res = df.evaluate(pds.lin_reg_report(*xs, target="y", add_bias=bias, null_policy=pol, std_err=se))
                got, want = mk.report_values(res), golden[mk.key(dt, bias, pol, se)]
                assert got.dtype == want.dtype and np.array_equal(got.view(np.uint8), want.view(np.uint8)), \
                    mk.key(dt, bias, pol, se)
    finally:
        cfg.LIN_REG_EXPR_F64 = True
