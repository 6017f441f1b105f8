"""lin_reg(return_pred=True).over(key) on the device: pl_lr_pred_by fits every group with pl_lr_by's batched fit and runs
one segmented predict pass (K5 pass 3).  Checked against Polars' per-group loop (over(fast=False): one pl_lr_pred call
per group), against the oracle, and bit for bit against pdsb_dev_predict_* run group by group with pl_lr_by's
coefficients."""
import numpy as np
import pyarrow as pa
import pytest

import polars_ds_extension_b200 as pds
import polars_ds_extension_b200.config as cfg
from polars_ds_extension_b200 import Frame, _harness
from tests.backends import OracleBackend, _masked
from tests.parity_rule import accept_f32, accept_f64, rel

pytestmark = pytest.mark.gpu

ORC = OracleBackend()
F64 = [True, False]


def _cols(seed, sizes, p, dt, positive=False, shuffle=False):
    """Columns y, x0.. of groups of the given sizes, and each row's group id (rows in group order unless shuffled)."""
    rng = np.random.default_rng(seed)
    gid = np.repeat(np.arange(len(sizes)), sizes)
    if shuffle:
        gid = rng.permutation(gid)
    n = len(gid)
    X = np.abs(rng.standard_normal((n, p))) if positive else rng.standard_normal((n, p))
    beta = ((np.arange(p) % 7) - 3) / 4.0
    beta = np.abs(beta) if positive else beta
    y = X @ beta + 0.1 * rng.standard_normal(n) + 0.5 + 0.2 * np.sin(gid)
    return y.astype(dt), X.astype(dt), gid


def _frame(y, X, gid):
    return Frame({"y": y} | {f"x{i}": X[:, i] for i in range(X.shape[1])} | {"g": gid})


def _split(res):
    """struct {pred, resid} -> (pred, pred valid, resid, resid valid) as numpy."""
    (pv, pm), (rv, rm) = _masked(res.field("pred")), _masked(res.field("resid"))
    return pv, pm, rv, rm


def _kw(**over):
    kw = pds.lin_reg("x0", target="y", return_pred=True).kwargs
    kw.update(over)
    return kw


def _call_by(sym, y, X, offsets, kw, chunks=None):
    """pl_lr_pred_by / pl_lr_by straight through the ABI on columns already in group order."""
    ins = [pa.array(np.asarray(offsets, dtype=np.int64)), pa.array(y)] + [pa.array(X[:, i]) for i in range(X.shape[1])]
    names = ["__offsets__", "y"] + [f"x{i}" for i in range(X.shape[1])]
    return _harness.call_plugin(sym, ins, names, kw)


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint32 if a.dtype == np.float32 else np.uint64)


def _k4_group(y, X, lo, hi, coeffs, add_bias):
    """pdsb_dev_predict_* on device copies of rows [lo, hi) with the given coefficients."""
    import torch

    from polars_ds_extension_b200 import device as dev

    Xg = torch.tensor(np.ascontiguousarray(X[lo:hi].T), device="cuda")
    yg = torch.tensor(np.ascontiguousarray(y[lo:hi][None, :]), device="cuda")
    beta = torch.tensor(np.asarray(coeffs, dtype=np.float64)[None, :], device="cuda")
    st = torch.zeros(4, dtype=torch.int32, device="cuda")
    pr, rs = dev.predict(Xg, yg, beta, st, add_bias)
    torch.cuda.synchronize()
    return pr[0, :hi - lo].cpu().numpy(), rs[0, :hi - lo].cpu().numpy()


def _check_bits_against_k4(y, X, offsets, kw, sym_sfx):
    """pl_lr_pred_by == pdsb_dev_predict_* per group with pl_lr_by's coefficients, bit for bit; groups whose coefficients
    are null come out all null.  Returns the number of groups compared."""
    co = _call_by("pl_lr_by" + sym_sfx, y, X, offsets, kw)
    pv, pm, rv, rm = _split(_call_by("pl_lr_pred_by" + sym_sfx, y, X, offsets, kw))
    assert np.array_equal(pm, rm)
    seen = 0
    for g in range(len(offsets) - 1):
        lo, hi = int(offsets[g]), int(offsets[g + 1])
        c = co[g].as_py()
        if c is None:
            assert not pm[lo:hi].any(), f"group {g}: null coefficients but valid predictions"
            continue
        assert pm[lo:hi].all(), f"group {g}"
        if hi == lo:
            continue
        kp, kr = _k4_group(y, X, lo, hi, c, kw["bias"])
        assert np.array_equal(_bits(pv[lo:hi]), _bits(kp)), f"group {g}: pred differs from pdsb_dev_predict"
        assert np.array_equal(_bits(rv[lo:hi]), _bits(kr)), f"group {g}: resid differs from pdsb_dev_predict"
        seen += 1
    return seen


KINDS = {
    "ols": (5, dict(add_bias=True)),
    "ridge": (5, dict(add_bias=True, l2_reg=0.1)),
    "lasso": (5, dict(add_bias=True, l1_reg=0.01, tol=1e-9, max_iter=5000)),
    "enet": (5, dict(add_bias=False, l1_reg=0.01, l2_reg=0.02, tol=1e-9, max_iter=5000)),
    "nnls": (5, dict(add_bias=True, positive=True, tol=1e-10, max_iter=5000)),
    "positive_ridge": (5, dict(add_bias=False, positive=True, l2_reg=0.05, tol=1e-9, max_iter=5000)),
    "wide": (40, dict(add_bias=True, l2_reg=0.1)),
    "wide_nobias": (40, dict(add_bias=False)),
}


@pytest.mark.parametrize("f64", F64)
@pytest.mark.parametrize("kind", list(KINDS))
def test_agrees_with_polars_loop(monkeypatch, f64, kind):
    """over(fast=True) == over(fast=False) (one pl_lr_pred call per group, the path Polars takes).  The same arithmetic
    up to the moments' summation order: the coefficient tolerances of test_grouped_iterative_and_wide, carried through
    one row sum.  Rows are interleaved across groups, so the result must also come back in the frame's row order."""
    monkeypatch.setattr(cfg, "LIN_REG_EXPR_F64", f64)
    p, kw = KINDS[kind]
    positive = kw.get("positive", False)
    sizes = np.random.default_rng(78).integers(600, 1500, 16).tolist()
    y, X, gid = _cols(79, sizes, p, np.float64 if f64 else np.float32, positive=positive, shuffle=True)
    df = _frame(y, X, gid)
    xs = [f"x{i}" for i in range(p)]
    make = lambda: pds.lin_reg(*xs, target="y", return_pred=True, **kw)      # noqa: E731
    e = make()
    fast = _split(df.select(e.over("g", fast=True))[e.out_name])
    slow = _split(df.select(e.over("g"))[e.out_name])
    assert fast[1].all() and fast[3].all() and slow[1].all()
    tol = 1e-8 if f64 else 1e-4
    scale = float(np.max(np.abs(slow[0])))
    assert np.max(np.abs(fast[0] - slow[0])) / scale < tol, kind
    assert np.max(np.abs(fast[2] - slow[2])) / scale < tol, kind
    for g in (0, 7, 15):
        sub = df.filter(gid == g)
        monkeypatch.setattr(cfg, "LIN_REG_EXPR_F64", f64)
        o = ORC.eval(sub, make())
        got = fast[0][gid == g]
        if kind in ("ols", "ridge", "wide", "wide_nobias"):
            if f64:
                accept_f64(got, o["pred"][0], f"{kind} group {g}")
            else:
                monkeypatch.setattr(cfg, "LIN_REG_EXPR_F64", True)
                truth = ORC.eval(sub, make())
                accept_f32(got, o["pred"][0], truth["pred"][0], f"{kind} group {g}")
        else:   # iterative solvers: the optimiser's resolution, as in test_grouped_iterative_and_wide
            assert rel(got, o["pred"][0]) < (1e-6 if f64 else 2e-3), (kind, g)


@pytest.mark.parametrize("f64", F64)
@pytest.mark.parametrize("kind", ["ols", "lasso", "wide", "wide_nobias"])
def test_bit_exact_against_per_group_predict(f64, kind):
    """(NNLS is left out: in f32, pl_lr_pred_by runs pl_lr_pred_f32's 2000 sweeps and pl_lr_by_f32 pl_lr_f32's 200.)"""
    p, kw = KINDS[kind]
    sizes = np.random.default_rng(80).integers(1, 3000, 30).tolist() + [8192, 8193, 3]
    y, X, _ = _cols(81, sizes, p, np.float64 if f64 else np.float32, positive=kw.get("positive", False))
    offsets = np.concatenate([[0], np.cumsum(sizes)])
    k = pds.lin_reg("x0", target="y", return_pred=True, **kw).kwargs
    assert _check_bits_against_k4(y, X, offsets, k, "" if f64 else "_f32") >= 25


@pytest.mark.parametrize("f64", F64)
def test_edge_group_sizes(f64):
    """Sizes 0, 1, q-1 (null), q, around the 128-row item rounding and the 8192-row CHUNK: every row is written once,
    with the value pdsb_dev_predict_* gives on its group."""
    p = 3
    q = p + 1
    sizes = [0, 1, q - 1, q, 127, 128, 129, 0, 8191, 8192, 8193, 16385, 5]
    y, X, _ = _cols(82, sizes, p, np.float64 if f64 else np.float32)
    offsets = np.concatenate([[0], np.cumsum(sizes)])
    k = _kw(bias=True, singular_x_tol=0.0)
    assert _check_bits_against_k4(y, X, offsets, k, "" if f64 else "_f32") == 9
    pv, pm, _, _ = _split(_call_by("pl_lr_pred_by" + ("" if f64 else "_f32"), y, X, offsets, k))
    assert not pm[:1 + q - 1].any() and pm[1 + q - 1:].all()


@pytest.mark.parametrize("f64", F64)
@pytest.mark.parametrize("misaligned", [False, True])
def test_device_entry_writes_every_row_once(f64, misaligned):
    """pdsb_dev_grouped_predict_* into outputs filled with a sentinel: every row is overwritten, once, with K4's value
    for its group; also with a base address off the 16-byte grid (the one-row-per-lane kernel)."""
    import torch

    from polars_ds_extension_b200 import device as dev

    dt = torch.float64 if f64 else torch.float32
    p = 4
    sizes = [0, 1, 5, 127, 128, 129, 8191, 8192, 8193, 16385, 3, 300]
    y, X, _ = _cols(83, sizes, p, np.float64 if f64 else np.float32)
    n = len(y)
    off = 1 if misaligned else 0
    Z = torch.zeros((p + 1, (n + off + 3) // 4 * 4 + 4), dtype=dt, device="cuda")     # ld a multiple of 4
    Z[:p, off:off + n] = torch.tensor(np.ascontiguousarray(X.T), device="cuda")
    Z[p, off:off + n] = torch.tensor(y, device="cuda")
    Xd, yd = Z[:p, off:off + n], Z[p, off:off + n]
    offsets = torch.tensor(np.concatenate([[0], np.cumsum(sizes)]), dtype=torch.int64, device="cuda")
    beta, status = dev.grouped_lin_reg(Xd, yd, offsets, add_bias=True)
    pred = torch.full((n + 1,), 12345.0, dtype=dt, device="cuda")[off:]
    resid = torch.full((n + 1,), 12345.0, dtype=dt, device="cuda")[off:]
    valid = torch.full((n,), 7, dtype=torch.uint8, device="cuda")
    dev.grouped_predict(Xd, yd, offsets, beta, status, True, pred=pred, resid=resid, valid=valid)
    torch.cuda.synchronize()
    pv, rv, vv = pred[:n].cpu().numpy(), resid[:n].cpu().numpy(), valid.cpu().numpy()
    st, bh, oh = status.cpu().numpy(), beta.cpu().numpy(), offsets.cpu().numpy()
    assert set(vv.tolist()) <= {0, 1}
    for g in range(len(sizes)):
        lo, hi = int(oh[g]), int(oh[g + 1])
        if hi == lo:
            continue
        assert (vv[lo:hi] == (1 if st[g] == 0 else 0)).all(), g
        if st[g] != 0:
            continue
        kp, kr = _k4_group(y, X, lo, hi, bh[g], True)
        assert np.array_equal(_bits(pv[lo:hi]), _bits(kp)) and np.array_equal(_bits(rv[lo:hi]), _bits(kr)), g
    assert st[1] != 0 and st[2] == 0           # a single row < q coefficients: gated
    assert (pred[n:].cpu().numpy() == 12345.0).all()


@pytest.mark.parametrize("f64", F64)
def test_nulls_and_nan(monkeypatch, f64):
    monkeypatch.setattr(cfg, "LIN_REG_EXPR_F64", f64)
    dt = np.float64 if f64 else np.float32
    sizes = [400, 500, 300, 450]
    y, X, gid = _cols(84, sizes, 3, dt, shuffle=True)
    n = len(y)
    rng = np.random.default_rng(85)
    xnull = np.zeros(n, bool)
    xnull[rng.choice(n, 40, replace=False)] = True
    ynull = np.zeros(n, bool)
    ynull[rng.choice(n, 30, replace=False)] = True
    cols = {"y": pa.array(y, mask=ynull), "x0": pa.array(X[:, 0], mask=xnull), "x1": X[:, 1], "x2": X[:, 2], "g": gid}
    df = Frame(cols)
    e = pds.lin_reg("x0", "x1", "x2", target="y", add_bias=True, return_pred=True)
    fast = _split(df.select(e.over("g", fast=True))[e.out_name])
    slow = _split(df.select(e.over("g"))[e.out_name])
    null = xnull | ynull
    assert np.array_equal(fast[1], ~null) and np.array_equal(fast[3], ~null)
    assert np.array_equal(slow[1], ~null)
    scale = float(np.max(np.abs(slow[0][~null])))
    tol = 1e-8 if f64 else 1e-4
    assert np.max(np.abs(fast[0][~null] - slow[0][~null])) / scale < tol
    assert np.max(np.abs(fast[2][~null] - slow[2][~null])) / scale < tol

    # raise: the error of pl_lr_by
    er = pds.lin_reg("x0", "x1", "x2", target="y", add_bias=True, return_pred=True, null_policy="raise")
    with pytest.raises(pds.PdsbError, match="Nulls found in data"):
        df.select(er.over("g", fast=True))

    # a collinear group is all null; the other groups are bit for bit what they are with that group well posed
    X2 = X.copy()
    X2[gid == 2, 1] = 2 * X2[gid == 2, 0]
    base = Frame({"y": y, "x0": X[:, 0], "x1": X[:, 1], "x2": X[:, 2], "g": gid})
    coll = Frame({"y": y, "x0": X2[:, 0], "x1": X2[:, 1], "x2": X2[:, 2], "g": gid})
    a = _split(base.select(e.over("g", fast=True))[e.out_name])
    b = _split(coll.select(e.over("g", fast=True))[e.out_name])
    assert a[1].all() and not b[1][gid == 2].any() and not b[3][gid == 2].any() and b[1][gid != 2].all()
    assert np.array_equal(_bits(a[0][gid != 2]), _bits(b[0][gid != 2]))
    assert np.array_equal(_bits(a[2][gid != 2]), _bits(b[2][gid != 2]))

    # a genuine NaN value: NaN, not null; pl_lr_by leaves the row out of its group's fit
    X3 = X.copy()
    i = int(np.flatnonzero(gid == 1)[17])
    X3[i, 2] = np.nan
    nan_df = Frame({"y": y, "x0": X3[:, 0], "x1": X3[:, 1], "x2": X3[:, 2], "g": gid})
    c = _split(nan_df.select(e.over("g", fast=True))[e.out_name])
    assert c[1].all() and c[3].all()
    assert np.isnan(c[0][i]) and np.isnan(c[2][i])
    assert np.isfinite(c[0][np.arange(n) != i]).all()
    assert np.array_equal(_bits(c[0][gid != 1]), _bits(a[0][gid != 1]))


@pytest.mark.parametrize("f64", F64)
def test_config_group_count(monkeypatch, f64):
    """1e4 groups of 80..120 rows x 8 features (C3's group count at 1 % of its rows) against the oracle."""
    monkeypatch.setattr(cfg, "LIN_REG_EXPR_F64", f64)
    rng = np.random.default_rng(86)
    sizes = rng.integers(80, 121, 10_000).tolist()
    y, X, gid = _cols(87, sizes, 8, np.float64 if f64 else np.float32)
    df = _frame(y, X, gid)
    xs = [f"x{i}" for i in range(8)]
    make = lambda: pds.lin_reg(*xs, target="y", add_bias=True, return_pred=True)     # noqa: E731
    e = make()
    fast = _split(df.select(e.over("g", fast=True))[e.out_name])
    assert fast[1].all() and len(fast[0]) == len(y)
    offsets = np.concatenate([[0], np.cumsum(sizes)])
    for g in rng.integers(0, len(sizes), 60).tolist():
        lo, hi = offsets[g], offsets[g + 1]
        sub = df.slice(int(lo), int(hi - lo))
        monkeypatch.setattr(cfg, "LIN_REG_EXPR_F64", f64)
        o = ORC.eval(sub, make())
        if f64:
            accept_f64(fast[0][lo:hi], o["pred"][0], f"group {g}")
        else:
            monkeypatch.setattr(cfg, "LIN_REG_EXPR_F64", True)
            truth = ORC.eval(sub, make())
            accept_f32(fast[0][lo:hi], o["pred"][0], truth["pred"][0], f"group {g}")


@pytest.mark.parametrize("f64", F64)
def test_repeatable_and_chunked_inputs(f64):
    sfx = "" if f64 else "_f32"
    sizes = np.random.default_rng(88).integers(50, 5000, 40).tolist()
    y, X, _ = _cols(89, sizes, 6, np.float64 if f64 else np.float32)
    n = len(y)
    offsets = pa.array(np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64))
    kw = _kw(bias=True)
    names = ["__offsets__", "y"] + [f"x{i}" for i in range(6)]
    cols = [y] + [X[:, i] for i in range(6)]
    one = _harness.call_plugin("pl_lr_pred_by" + sfx, [offsets] + [pa.array(c) for c in cols], names, kw)
    again = _harness.call_plugin("pl_lr_pred_by" + sfx, [offsets] + [pa.array(c) for c in cols], names, kw)
    assert one.equals(again)
    cuts = [0, 1, 1000, 1001, n // 2 + 3, n]
    chunked = [pa.chunked_array([pa.array(c[a:b]) for a, b in zip(cuts[:-1], cuts[1:])]) for c in cols]
    assert _harness.call_plugin("pl_lr_pred_by" + sfx, [offsets] + chunked, names, kw).equals(one)
    sliced = [pa.array(np.concatenate([c[:13], c, c[:5]])).slice(13, n) for c in cols]
    assert _harness.call_plugin("pl_lr_pred_by" + sfx, [offsets] + sliced, names, kw).equals(one)


@pytest.mark.parametrize("f64", F64)
def test_offset_and_kwarg_errors_match_pl_lr_by(f64):
    sfx = "" if f64 else "_f32"
    y, X, _ = _cols(90, [10, 10, 10], 2, np.float64 if f64 else np.float32)
    kw = _kw(bias=True)
    bad = {
        "decreasing": ([0, 20, 10, 30], "non-decreasing"),
        "out of range": ([0, 40, 35, 30], "non-decreasing and within"),
        "last != n": ([0, 10, 20, 29], "bad group offsets"),
        "first != 0": ([1, 10, 20, 30], "bad group offsets"),
    }
    for what, (offs, msg) in bad.items():
        msgs = []
        for sym in ("pl_lr_by", "pl_lr_pred_by"):
            with pytest.raises(pds.PdsbError, match=msg) as ei:
                _call_by(sym + sfx, y, X, offs, kw)
            msgs.append(str(ei.value))
        assert msgs[0] == msgs[1], what
    for sym in ("pl_lr_by", "pl_lr_pred_by"):
        with pytest.raises(pds.PdsbError, match="weighted fits are not batched"):
            _call_by(sym + sfx, y, X, [0, 10, 20, 30], _kw(bias=True, weighted=True))
        with pytest.raises(pds.PdsbError, match="only null_policy='skip'"):
            ins = [pa.array(np.array([0, 10, 20, 30], dtype=np.int64)), pa.array(y, mask=np.arange(30) == 4),
                   pa.array(X[:, 0]), pa.array(X[:, 1])]
            _harness.call_plugin(sym + sfx, ins, ["__offsets__", "y", "x0", "x1"], _kw(bias=True, null_policy="zero"))


@pytest.mark.parametrize("p", [4, 14])
def test_predict_pass_reuses_the_fits_work_list(p):
    """pl_lr_pred_by's predict pass runs on the fit's work list: beyond pl_lr_by's launches it adds the predict kernel,
    and for p > 10 (where the fit's moments kernel needs no row ranges) the item -> rows map."""
    from polars_ds_extension_b200._lib import lib

    y, X, gid = _cols(31, [5, 9000, 3, 700], p, np.float64)
    offsets = np.concatenate([[0], np.cumsum(np.bincount(gid))])
    counts = {}
    for sym in ("pl_lr_by", "pl_lr_pred_by"):
        c0 = lib().pdsb_kernel_launch_count()
        _call_by(sym, y, X, offsets, _kw(bias=True))
        counts[sym] = lib().pdsb_kernel_launch_count() - c0
    assert counts["pl_lr_pred_by"] - counts["pl_lr_by"] == (1 if p <= 10 else 2)
