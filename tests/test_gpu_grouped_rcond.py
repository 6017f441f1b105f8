"""group_by(key).agg(lin_reg_w_rcond) on the device (K19): pl_lr_w_rcond_by fits every group in one launch sequence.
Checked per group against Polars' per-group loop (one pl_lr_w_rcond call on the group's rows) and against the CPU oracle,
on full-rank and rank-deficient groups, with skipped nulls and dropped non-finite rows, for its error messages, for
independence from the other groups, reproducibility and chunking, through the device entry, and at 1e6 groups.

Every group's data is built so that the cut is not on a knife edge: each eigenvalue of its (ridged) Gram is either at
least 100 times the threshold tol * sqrt(lambda_max) or at most 0.01 times it (an exactly singular direction counts as
0), for the tolerance of the f32 and the f64 rule alike (_check_margin).  The f32 floor of the parity rule is
max(2e-6, cond 2^-24), cond the ratio of the largest to the smallest kept eigenvalue (for the singular values of a
group with a nearly collinear direction, 2^-11: _check_margin)."""
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
CUT = 1e-7           # an rcond that cuts the exactly singular directions and keeps every other one
NEAR_CUT = 1e-2      # an rcond that cuts the nearly collinear direction of "near"


def _groups(seed, sizes, p, dt, kind="full"):
    """y, X, group ids.  kind: "full" (full rank), "dup" (x1 = x0), "const" (x0 = 2 in every row: with a bias, a column
    the ones column spans exactly, as 2 * 1 is exact), "near" (x1 = x0 + 1e-3 z).  A group of a few rows per feature
    gets orthogonal columns, orthogonal to the ones column as well where it has more rows than features: a square
    system of random rows would have eigenvalues anywhere near the cut.  Every x is a multiple of 1/4 and small, so
    each product and each partial sum of X'X is exact in f32: an exactly singular Gram stays exactly singular in every
    summation order, the loop's and the oracle's included."""
    rng = np.random.default_rng(seed)
    ys, Xs = [], []
    for g, m in enumerate(sizes):
        if p <= m <= 4 * p + 8:
            lead = [np.ones((m, 1))] if m > p else []
            Q = np.linalg.qr(np.column_stack(lead + [rng.standard_normal((m, p))]))[0]
            X = np.sqrt(m) * Q[:, len(lead):]
        else:
            X = rng.standard_normal((m, p)) + 0.3 * np.sin(np.arange(p) + g)
        X = np.round(4 * X) / 4
        beta = (0.6 + 0.3 * np.cos(np.arange(p) + 2 * g)) * np.where(np.arange(p) % 2, 1.0, -1.0)
        y = X @ beta + 0.5 * np.cos(g) + 0.5 * rng.standard_normal(m)
        if kind == "dup":
            X[:, 1] = X[:, 0]
        elif kind == "const":
            X[:, 0] = 2.0
        elif kind == "near":
            X[:, 1] = X[:, 0] + 1e-3 * rng.standard_normal(m)
        ys.append(y)
        Xs.append(X)
    return np.concatenate(ys).astype(dt), np.concatenate(Xs).astype(dt), np.repeat(np.arange(len(sizes)), sizes)


def _expr(p, **kw):
    return pds.lin_reg_w_rcond(*[f"x{i}" for i in range(p)], target="y", **kw)


def _frame(y, X, gid):
    return Frame({"y": y} | {f"x{i}": X[:, i] for i in range(X.shape[1])} | {"g": gid})


def _gram(Xk, bias, l2):
    A = np.column_stack([Xk.astype(np.float64)] + ([np.ones(len(Xk))] if bias else []))
    G = A.T @ A
    G[np.arange(Xk.shape[1]), np.arange(Xk.shape[1])] += l2
    return G


def _tol(rcond, m, q, f32):
    if f32:
        return max(float(np.float32(rcond)), float(np.finfo(np.float32).eps) * max(m, q))
    return max(rcond, float(np.finfo(np.float64).eps) * max(m, q))


def _check_margin(Xk, m, bias, l2, rcond, f32, what):
    """The cut of this group is not on a knife edge (module docstring); returns the f32 floors of its coefficients and of
    its singular values."""
    lam = np.linalg.eigvalsh(_gram(Xk, bias, l2))
    lmax = max(float(lam.max()), 0.0)
    lam = np.where(np.abs(lam) <= 1e-11 * lmax, 0.0, lam)            # exactly singular directions
    for f in ((True, False) if f32 else (False,)):
        thr = _tol(rcond, m, len(lam), f) * np.sqrt(lmax)
        assert np.all((lam >= 100 * thr) | (lam <= 0.01 * thr)), (what, f, lam.min(), thr)
    kept = lam[lam >= 100 * _tol(rcond, m, len(lam), f32) * np.sqrt(lmax)]
    floor = max(FLOOR, float(kept.max() / kept.min()) * 2.0 ** -24)
    # a cut direction that is not exactly singular ("near") has an eigenvalue at the f32 Gram's rounding level, c 2^-24
    # lambda_max: its singular value is resolved only to sqrt(c 2^-24) of the largest one
    sv_floor = max(floor, 2.0 ** -11) if np.any(lam[lam < 100 * _tol(rcond, m, len(lam), f32) * np.sqrt(lmax)] > 0) \
        else floor
    return floor, sv_floor


def _struct(v):
    return {k: np.asarray(v[k], dtype=np.float64) for k in ("coeffs", "singular_values")}


def _fast(df, e):
    res = df.group_by("g").agg(e, fast=True)[e.out_name or e.symbol]
    assert pa.types.is_large_list(res.type)
    return [None if not res[i].is_valid else _struct(res[i].as_py()[0]) for i in range(len(res))]


def _loop(sub, e):
    return _struct(sub.evaluate(e)[0].as_py())


def _accept32(g, o32, truth, floor, what):
    if floor <= FLOOR:
        return accept_f32(g, o32, truth, what)[1]
    eg, eo, ego = rel(g, truth), rel(o32, truth), rel(g, o32)
    assert eg <= max(eo, floor), f"{what}: {eg:.3e} from the f64 truth, the f32 restatement {eo:.3e}, floor {floor:.3e}"
    if eo <= F32_TOL:
        assert ego <= max(F32_TOL, 2 * floor), f"{what}: |gpu - oracle_f32| = {ego:.3e}"
    return eo


def _check_group(monkeypatch, f64, sub, make, got, floors, what):
    monkeypatch.setattr(cfg, "LIN_REG_EXPR_F64", f64)
    loop = _loop(sub, make())
    o = ORC.eval(sub, make())
    if not f64:
        monkeypatch.setattr(cfg, "LIN_REG_EXPR_F64", True)
        truth = ORC.eval(sub, make())
        monkeypatch.setattr(cfg, "LIN_REG_EXPR_F64", False)
    for k, floor in zip(("coeffs", "singular_values"), floors):
        g, lp, ov = got[k], loop[k], np.asarray(o[k], np.float64)
        assert g.shape == lp.shape == ov.shape, (what, k)
        if f64:
            accept_f64(g, ov, f"{what}:{k}")
            accept_f64(g, lp, f"{what}:{k} loop")
        else:
            eo = _accept32(g, ov, np.asarray(truth[k], np.float64), floor, f"{what}:{k}")
            if eo <= F32_TOL:
                assert rel(g, lp) <= max(F32_TOL, 2 * floor), (what, k, "loop", rel(g, lp))


# (kind, rcond, l2): a full-rank group at the eps floor and with a ridge, exactly singular groups cut by CUT (with a
# ridge nothing is singular any more: l2 = 1e3 lifts those directions well above f32's eps floor at 16385 rows), and a
# nearly collinear direction cut by NEAR_CUT
RIDGE = 1e3
CASES = [("full", 0.0, 0.0), ("full", 0.0, RIDGE), ("dup", CUT, 0.0), ("dup", CUT, RIDGE), ("const", CUT, 0.0),
         ("const", CUT, RIDGE), ("near", NEAR_CUT, 0.0)]


# ---- 1. fast group_by against the loop and the oracle ----
@pytest.mark.parametrize("f64", [True, False])
@pytest.mark.parametrize("bias", [True, False])
@pytest.mark.parametrize("kind,rcond,l2", CASES)
@pytest.mark.parametrize("p", [1, 8, 64])
def test_fast_matches_loop_and_oracle(monkeypatch, f64, bias, kind, rcond, l2, p):
    if (kind in ("dup", "near") and p < 2) or (kind == "const" and not bias):
        pytest.skip("this kind of rank deficiency needs two features / a bias")
    q = p + int(bias)
    sizes = [1, q - 1, q, q + 5, 300, 8191, 8192, 8193, 16385] if kind != "near" else [300, 8191, 8193, 16385]
    sizes = [m for m in sizes if m >= 1]
    dt = np.float64 if f64 else np.float32
    y, X, gid = _groups(500 + p + 7 * len(kind), sizes, p, dt, kind)
    df = _frame(y, X, gid)
    make = lambda: _expr(p, add_bias=bias, rcond=rcond, l2_reg=l2)      # noqa: E731
    monkeypatch.setattr(cfg, "LIN_REG_EXPR_F64", f64)
    fast = _fast(df, make())
    assert len(fast) == len(sizes)
    for g, m in enumerate(sizes):
        what = f"{'f64' if f64 else 'f32'} p={p} bias={bias} {kind} l2={l2} group {g} ({m} rows)"
        if m < q:
            assert fast[g] is None, what
            continue
        assert fast[g] is not None, what
        floors = _check_margin(X[gid == g], m, bias, l2, rcond, not f64, what)
        _check_group(monkeypatch, f64, df.filter(gid == g), make, fast[g], floors, what)


def _call_by(y, X, offsets, kw, chunks=1, f32=False, ymask=None):
    ins = ([pa.array(np.asarray(offsets, dtype=np.int64)), chunked(y, chunks, ymask)]
           + [chunked(X[:, i], chunks) for i in range(X.shape[1])])
    names = ["__offsets__", "y"] + [f"x{i}" for i in range(X.shape[1])]
    return _harness.call_plugin("pl_lr_w_rcond_by" + ("_f32" if f32 else ""), ins, names, kw)


# ---- 2. empty groups ----
@pytest.mark.parametrize("f32", [False, True])
def test_empty_groups_through_the_abi(f32):
    p = 3
    y, X, _ = _groups(71, [300, 500], p, np.float32 if f32 else np.float64)
    offs = np.array([0, 0, 300, 300, 800, 800], dtype=np.int64)          # groups 0, 2 and 4 are empty
    kw = _expr(p, add_bias=True, rcond=1e-6).kwargs
    res = _call_by(y, X, offs, kw, f32=f32)
    assert len(res) == 5 and [res[i].is_valid for i in range(5)] == [False, True, False, True, False]
    item = res.type.value_type
    T = pa.float32() if f32 else pa.float64()
    assert [item.field(i).name for i in range(2)] == ["coeffs", "singular_values"]
    assert item.field(0).type.value_type == T
    ref = _call_by(y, X, np.array([0, 300, 800], dtype=np.int64), kw, f32=f32)
    for a, b in ((1, 0), (3, 1)):
        assert res[a].values.equals(ref[b].values)
        assert len(res[a].as_py()) == 1 and len(res[a].as_py()[0]["coeffs"]) == p + 1


# ---- 3. nulls with "skip" and non-finite values ----
@pytest.mark.parametrize("f64", [True, False])
def test_skipped_nulls_and_dropped_nonfinite_rows(monkeypatch, f64):
    p = 5
    sizes = [400, 900, 3000, 9000, 60]
    dt = np.float64 if f64 else np.float32
    y, X, gid = _groups(61, sizes, p, dt)
    rng = np.random.default_rng(62)
    n = len(y)
    xnull = [rng.random(n) < 0.05 for _ in range(p)]
    ynull = rng.random(n) < 0.05
    o = group_offsets(np.bincount(gid))
    xnull[2][o[4]:o[4] + 56] = True              # group 4: 60 rows, all but 4 dropped -> a null list
    bad = rng.random(n) < 0.03                    # NaN / inf in kept rows: dropped from their group
    X = X.copy()
    X[bad, 1] = np.nan
    X[np.flatnonzero(bad)[::2], 3] = np.inf
    cols = {"y": pa.array(y, mask=ynull)} | {f"x{i}": pa.array(X[:, i], mask=xnull[i]) for i in range(p)}
    df = Frame(cols | {"g": gid})
    monkeypatch.setattr(cfg, "LIN_REG_EXPR_F64", f64)
    make = lambda: _expr(p, add_bias=True, rcond=1e-6, null_policy="skip")     # noqa: E731
    fast = _fast(df, make())
    assert fast[4] is None
    drop = ynull | np.any(np.column_stack(xnull), axis=1) | bad
    for g in range(4):
        # the loop sees the group without its non-finite rows (a NaN would poison its fit); the threshold's eps floor
        # depends on the row count, which the margin keeps away from the cut
        sub = df.filter((gid == g) & ~bad)
        floors = _check_margin(X[(gid == g) & ~drop], sizes[g], True, 0.0, 1e-6, not f64, f"nulls group {g}")
        _check_group(monkeypatch, f64, sub, make, fast[g], floors, f"nulls group {g}")


# ---- 4. errors ----
def test_errors():
    p = 3
    y, X, gid = _groups(97, [50, 60], p, np.float64)
    kw = _expr(p, add_bias=True, null_policy="skip").kwargs
    with pytest.raises(pds.PdsbError, match="bad group offsets"):
        _call_by(y, X, np.array([0, 50, 100], dtype=np.int64), kw)
    with pytest.raises(pds.PdsbError, match="non-decreasing"):
        _call_by(y, X, np.array([0, 70, 60, 110], dtype=np.int64), kw)
    ymask = np.arange(len(y)) == 3
    with pytest.raises(pds.PdsbError, match="Nulls found in data"):
        _call_by(y, X, group_offsets(np.bincount(gid)), kw | {"null_policy": "raise"}, ymask=ymask)
    for fill in ("zero", "1.5"):
        with pytest.raises(pds.PdsbError, match="only null_policy='skip' is supported with nulls"):
            _call_by(y, X, group_offsets(np.bincount(gid)), kw | {"null_policy": fill}, ymask=ymask)
    X65 = np.random.default_rng(98).standard_normal((len(y), 65))
    with pytest.raises(pds.PdsbError, match="at most 64"):
        _call_by(y, X65, group_offsets(np.bincount(gid)), kw)
    with pytest.raises(ValueError, match="fast over is only available for lin_reg predictions"):
        _expr(p).over("g", fast=True)


# ---- 5. device entry, independence, reproducibility, chunking ----
@pytest.mark.parametrize("f32", [False, True])
def test_device_entry_matches_the_plugin(f32):
    p = 6
    sizes = [100, 6, 9000, 40]
    dt = np.float32 if f32 else np.float64
    y, X, gid = _groups(95, sizes, p, dt, "dup")
    offs = group_offsets(np.bincount(gid))
    beta, sv, status = dev.grouped_lin_reg_rcond(torch.tensor(X.T.copy(), device="cuda"), torch.tensor(y, device="cuda"),
                                                 torch.tensor(offs, device="cuda"), add_bias=True, rcond=-CUT)
    assert status.cpu().tolist() == [0, 1, 0, 0]
    b, s = beta.cpu().numpy(), sv.cpu().numpy()
    assert np.isnan(b[1]).all() and np.isnan(s[1]).all()
    assert np.all(np.diff(s[[0, 2, 3]], axis=1) <= 0)
    res = _call_by(y, X, offs, _expr(p, add_bias=True, rcond=CUT).kwargs, f32=f32)
    for g in (0, 2, 3):
        v = res[g].as_py()[0]
        assert np.array_equal(np.asarray(v["coeffs"], dt), b[g].astype(dt))
        assert np.array_equal(np.asarray(v["singular_values"], dt), s[g].astype(dt))


@pytest.mark.parametrize("f64", [True, False])
def test_independent_reproducible_and_chunk_invariant(f64):
    p = 8
    sizes = [129, 8193, 3000, 20000, 77]
    dt = np.float64 if f64 else np.float32
    y, X, gid = _groups(91, sizes, p, dt, "dup")
    offs = group_offsets(np.bincount(gid))
    kw = _expr(p, add_bias=True, rcond=CUT, l2_reg=0.0).kwargs
    f32 = not f64
    a = _call_by(y, X, offs, kw, f32=f32)
    assert a.equals(_call_by(y, X, offs, kw, f32=f32))
    assert a.equals(_call_by(y, X, offs, kw, chunks=7, f32=f32))
    y2, X2 = y.copy(), X.copy()
    lo, hi = offs[2], offs[3]
    y2[lo:hi] = y2[lo:hi][::-1] * dt(1.5)
    X2[lo:hi] = X2[lo:hi] + dt(0.25)
    d = _call_by(y2, X2, offs, kw, f32=f32)
    for g in range(len(sizes)):
        assert d[g].values.equals(a[g].values) == (g != 2), g


# ---- 6. a million groups ----
def test_million_groups(monkeypatch):
    n_groups, m, p = 1_000_000, 100, 3
    rng = np.random.default_rng(7)
    X = rng.standard_normal((n_groups * m, p)).astype(np.float32)
    y = (X @ np.array([0.5, -1.0, 0.25]) + 0.1 * rng.standard_normal(n_groups * m)).astype(np.float32)
    offs = np.arange(0, n_groups * m + 1, m, dtype=np.int64)
    kw = _expr(p, add_bias=True, rcond=1e-6).kwargs
    res = _call_by(y, X, offs, kw, f32=True)
    assert len(res) == n_groups and res.null_count == 0
    assert pa.types.is_large_list(res.type) and len(res.values) == n_groups
    monkeypatch.setattr(cfg, "LIN_REG_EXPR_F64", False)
    for g in (0, 1, 4242, 500_000, n_groups - 1):
        lo, hi = offs[g], offs[g + 1]
        got = _struct(res[g].as_py()[0])
        # alone, the group gives the same bits (independence), and the loop's fit to the parity rule
        one = _call_by(y[lo:hi], X[lo:hi], np.array([0, m], dtype=np.int64), kw, f32=True)
        assert one[0].values.equals(res[g].values), g
        sub = _frame(y[lo:hi], X[lo:hi], np.zeros(m, dtype=np.int64))
        floors = _check_margin(X[lo:hi], m, True, 0.0, 1e-6, True, f"group {g}")
        _check_group(monkeypatch, False, sub, lambda: _expr(p, add_bias=True, rcond=1e-6), got, floors, f"group {g}")
