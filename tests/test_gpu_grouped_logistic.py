"""group_by(key).agg(logistic_reg) and logistic_reg(return_pred=True).over(key) on the device (K16): pl_logistic_by /
pl_logistic_pred_by fit every group in one launch sequence.  Checked against Polars' per-group loop (fast=False: one
pl_logistic_coeffs / pl_logistic_pred call per group), against the CPU oracle, bit for bit against pdsb_glm_predict
with the group's coefficients, for independence from the other groups, and for the device entry's status and
iteration count."""
import ctypes as C

import numpy as np
import pyarrow as pa
import pytest

import polars_ds_extension_b200 as pds
from polars_ds_extension_b200 import Frame, _harness
from polars_ds_extension_b200._lib import (GLM_BINOMIAL, LOGISTIC_CONVERGED, LOGISTIC_FAILED, LOGISTIC_MAX_ITER,
                                           Matrix, lib)
from tests.backends import OracleBackend, _masked
from tests.helpers import chunked, group_offsets

pytestmark = pytest.mark.gpu

ORC = OracleBackend()
PENALTIES = [(0.0, 0.0), (0.0, 1e-2), (1e-2, 0.0), (1e-2, 1e-2)]


def _sigmoid(z):
    return 0.5 * (1.0 + np.tanh(0.5 * z))


def _groups(seed, sizes, p, tie_below=0):
    """y, X and each row's group id, rows in group order.  Labels are Bernoulli draws around a mild signal.  A group of
    fewer than `tie_below` rows is pairs of one row with labels 1 and 0 (and, for an odd count, the first row again with
    label 0.5): it cannot be separated and its minimiser is beta = 0, where a small group of noisy labels would usually
    be separable, with no finite minimiser to compare."""
    rng = np.random.default_rng(seed)
    ys, Xs = [], []
    for g, m in enumerate(sizes):
        X = rng.standard_normal((m, p))
        if m < tie_below:
            half = X[: m // 2]
            X = np.concatenate([half, half, X[:1]])[:m]
            y = np.concatenate([np.ones(len(half)), np.zeros(len(half)), [0.5]])[:m]
        else:
            beta = 0.6 * np.cos(np.arange(p) + g) / np.sqrt(p)
            y = (rng.random(m) < _sigmoid(X @ beta + 0.2 * np.sin(g))).astype(np.float64)
        ys.append(y)
        Xs.append(X)
    gid = np.repeat(np.arange(len(sizes)), sizes)
    return np.concatenate(ys), np.concatenate(Xs), gid


def _frame(y, X, gid, **extra):
    return Frame({"y": y} | {f"x{i}": X[:, i] for i in range(X.shape[1])} | {"g": gid} | extra)


def _expr(p, **kw):
    return pds.logistic_reg(*[f"x{i}" for i in range(p)], target="y", **kw)


def _fast(df, e):
    res = df.group_by("g").agg(e, fast=True)[e.out_name]
    return [np.asarray(res[i].as_py()) for i in range(len(res))]


def _slow(df, e):
    res = df.group_by("g").agg(e, fast=False)[e.out_name]
    return [np.asarray(r[0].as_py()) for r in res]


def _call_by(sym, y, X, offsets, kw, chunks=1):
    """pl_logistic_by / pl_logistic_pred_by through the ABI on columns already in group order, each split in `chunks`."""
    ins = ([pa.array(np.asarray(offsets, dtype=np.int64)), chunked(y, chunks)]
           + [chunked(X[:, i], chunks) for i in range(X.shape[1])])
    names = ["__offsets__", "y"] + [f"x{i}" for i in range(X.shape[1])]
    return _harness.call_plugin(sym, ins, names, kw)


def _coeffs(res):
    return np.array([res[i].as_py() for i in range(len(res))])


def _cost(beta, X, y, bias, l1=0.0, l2=0.0):
    w = beta[: X.shape[1]]
    eta = X @ w + (beta[-1] if bias else 0.0)
    loss = np.mean(np.maximum(eta, 0) - y * eta + np.log1p(np.exp(-np.abs(eta))))
    return loss + 0.5 * l2 * w @ w + l1 * np.abs(w).sum()


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


def _glm_predict(X, beta, bias):
    """pdsb_glm_predict with the binomial family: K10's predict_strided, the rule of pl_logistic_pred."""
    Xm = np.ascontiguousarray(X, dtype=np.float64)
    xv = Matrix(Xm.ctypes.data, Xm.shape[0], Xm.shape[1], Xm.shape[1], 1)
    b = np.ascontiguousarray(beta, dtype=np.float64)
    out = np.empty(Xm.shape[0], dtype=np.float64)
    assert lib().pdsb_glm_predict(C.byref(xv), b.ctypes.data, len(b), int(bias), GLM_BINOMIAL, 0, out.ctypes.data) == 0
    return out


# ---- 1. fast group_by against the per-group loop ----
SIZES = [2, 3, 127, 128, 129, 1000, 8191, 8192, 8193, 16385, 20000]


@pytest.mark.parametrize("p", [1, 4, 8, 10, 11, 40, 64])
@pytest.mark.parametrize("bias", [True, False])
@pytest.mark.parametrize("l1,l2", PENALTIES)
def test_fast_group_by_matches_loop(p, bias, l1, l2):
    y, X, gid = _groups(100 + p, SIZES, p, tie_below=8 * (p + 1))
    df = _frame(y, X, gid)
    e = _expr(p, add_bias=bias, l1_reg=l1, l2_reg=l2, tol=1e-10, max_iter=200)
    fast, slow = _fast(df, e), _slow(df, e)
    bound = 1e-7 if l1 > 0 else 1e-9
    for g, (a, b) in enumerate(zip(fast, slow)):
        assert a.shape == b.shape == (p + int(bias),)
        assert np.all(np.isfinite(a)), g
        assert np.max(np.abs(a - b)) <= bound * max(1.0, np.max(np.abs(b))), (g, SIZES[g], np.max(np.abs(a - b)))


# ---- 2. each group against the CPU oracle ----
@pytest.mark.parametrize("bias", [True, False])
def test_each_group_matches_oracle(bias):
    sizes = [600, 2000, 9000, 4000]
    y, X, gid = _groups(7, sizes, 5)
    df = _frame(y, X, gid)
    e = _expr(5, add_bias=bias, tol=1e-8)
    fast = _fast(df, e)
    for g in range(len(sizes)):
        ref = ORC.eval(df.filter(gid == g), e)
        assert np.max(np.abs(fast[g] - ref)) < 1e-6, g


# ---- 3. per-row probabilities ----
@pytest.mark.parametrize("bias", [True, False])
def test_pred_rows_bit_for_bit(bias):
    sizes = [300, 8193, 1, 40, 5000]
    y, X, gid = _groups(11, sizes, 6, tie_below=20)
    rng = np.random.default_rng(5)
    drop = rng.random(len(y)) < 0.03
    drop[np.cumsum(sizes)[1]] = False                      # the one-row group keeps its row
    x2 = pa.array(X[:, 2], mask=drop)
    kw = _expr(6, add_bias=bias, tol=1e-9).kwargs
    offs = group_offsets(np.bincount(gid))
    ins_c = [pa.array(offs), pa.array(y)] + [x2 if i == 2 else pa.array(X[:, i]) for i in range(6)]
    names = ["__offsets__", "y"] + [f"x{i}" for i in range(6)]
    beta = _coeffs(_harness.call_plugin("pl_logistic_by", ins_c, names, kw))
    pred, valid = _masked(_harness.call_plugin("pl_logistic_pred_by", ins_c, names, kw))
    assert np.array_equal(valid, ~drop)
    Xz = np.where(drop[:, None], 0.0, X)                   # a dropped row's values do not matter; it is null
    for g in range(len(sizes)):
        lo, hi = offs[g], offs[g + 1]
        ref = _glm_predict(Xz[lo:hi], beta[g], bias)
        keep = ~drop[lo:hi]
        assert np.array_equal(_bits(pred[lo:hi][keep]), _bits(ref[keep])), g


def test_over_fast_matches_over_loop():
    sizes = [500, 3000, 64, 9000]
    y, X, gid = _groups(12, sizes, 4, tie_below=40)
    perm = np.random.default_rng(3).permutation(len(y))         # rows not in key order
    df = _frame(y[perm], X[perm], gid[perm])
    e = _expr(4, add_bias=True, tol=1e-10, return_pred=True)
    fa, fm = _masked(df.select(e.over("g", fast=True))[e.out_name])
    sa, sm = _masked(df.select(e.over("g", fast=False))[e.out_name])
    assert fm.all() and sm.all()
    assert np.max(np.abs(fa - sa)) < 1e-12


# ---- 4. edge groups ----
def test_all_ones_group():
    y, X, gid = _groups(13, [400, 300], 3)
    y[gid == 1] = 1.0
    df = _frame(y, X, gid)
    e = _expr(3, add_bias=True, tol=1e-10)
    fast, slow = _fast(df, e), _slow(df, e)
    for g in range(2):
        assert np.all(np.isfinite(fast[g])) and np.all(np.isfinite(slow[g]))
        sel = gid == g
        assert abs(_cost(fast[g], X[sel], y[sel], True) - _cost(slow[g], X[sel], y[sel], True)) < 1e-12


def test_nan_feature_fails_only_its_group():
    y, X, gid = _groups(14, [500, 700, 300], 4)
    e = _expr(4, add_bias=True, tol=1e-10)
    base = _fast(_frame(y, X, gid), e)
    Xn = X.copy()
    Xn[np.flatnonzero(gid == 1)[17], 2] = np.nan
    got = _fast(_frame(y, Xn, gid), e)
    assert np.all(np.isnan(got[1])) and np.all(np.isnan(_slow(_frame(y, Xn, gid), e)[1]))
    for g in (0, 2):
        assert np.array_equal(_bits(got[g]), _bits(base[g]))
    pred, valid = _masked(_call_by("pl_logistic_pred_by", y, Xn, group_offsets(np.bincount(gid)),
                                   _expr(4, return_pred=True).kwargs))
    assert valid.all() and np.all(np.isnan(pred[gid == 1])) and np.all(np.isfinite(pred[gid != 1]))


def test_fewer_rows_than_coefficients():
    y, X, gid = _groups(15, [6, 500], 8)
    df = _frame(y, X, gid)
    e = _expr(8, add_bias=True, tol=1e-10, max_iter=60)
    fast, slow = _fast(df, e), _slow(df, e)
    sel = gid == 0
    assert np.all(np.isfinite(fast[0])) and np.all(np.isfinite(slow[0]))
    assert abs(_cost(fast[0], X[sel], y[sel], True) - _cost(slow[0], X[sel], y[sel], True)) < 1e-12
    assert np.max(np.abs(fast[1] - slow[1])) < 1e-9 * max(1.0, np.max(np.abs(slow[1])))


def test_one_row_group():
    y, X, gid = _groups(16, [1, 800, 1], 3)
    df = _frame(y, X, gid)
    for bias in (True, False):
        e = _expr(3, add_bias=bias, l2_reg=1e-2, tol=1e-10)
        fast, slow = _fast(df, e), _slow(df, e)
        for g in range(3):
            assert np.max(np.abs(fast[g] - slow[g])) < 1e-9 * max(1.0, np.max(np.abs(slow[g]))), (bias, g)


def test_group_with_every_row_null_is_empty_data():
    y, X, gid = _groups(17, [50, 20, 50], 2)
    df = _frame(y, X, gid)
    df.columns["x1"] = pa.chunked_array([pa.array(X[:, 1], mask=gid == 1)])
    e = _expr(2, add_bias=True)
    for fast in (True, False):
        with pytest.raises(pds.PdsbError, match="Empty data"):
            df.group_by("g").agg(e, fast=fast)
    with pytest.raises(pds.PdsbError, match="Empty data"):
        df.select(_expr(2, return_pred=True).over("g", fast=True))


@pytest.mark.parametrize("policy", ["raise", "zero", "one", "0.5", "skip"])
def test_null_policies_match_loop(policy):
    y, X, gid = _groups(18, [400, 900, 300], 3)
    rng = np.random.default_rng(19)
    xmask, ymask = rng.random(len(y)) < 0.04, rng.random(len(y)) < 0.03
    df = _frame(y, X, gid)
    df.columns["x0"] = pa.chunked_array([pa.array(X[:, 0], mask=xmask)])
    df.columns["y"] = pa.chunked_array([pa.array(y, mask=ymask)])
    e = _expr(3, add_bias=True, tol=1e-10, null_policy=policy)
    if policy == "raise":
        for fast in (True, False):
            with pytest.raises(pds.PdsbError, match="Nulls found in data"):
                df.group_by("g").agg(e, fast=fast)
        return
    fast, slow = _fast(df, e), _slow(df, e)
    for g in range(3):
        assert np.max(np.abs(fast[g] - slow[g])) < 1e-9 * max(1.0, np.max(np.abs(slow[g]))), (policy, g)
    ep = _expr(3, add_bias=True, tol=1e-10, null_policy=policy, return_pred=True)
    fa, fm = _masked(df.select(ep.over("g", fast=True))[ep.out_name])
    sa, sm = _masked(df.select(ep.over("g", fast=False))[ep.out_name])
    assert np.array_equal(fm, sm)
    assert np.max(np.abs(fa[fm] - sa[sm])) < 1e-12


@pytest.mark.parametrize("max_iter", [1, 2, 3])
@pytest.mark.parametrize("l1", [0.0, 1e-2])
def test_max_iter_matches_loop(max_iter, l1):
    y, X, gid = _groups(20, [300, 5000, 9000], 5)
    df = _frame(y, X, gid)
    e = _expr(5, add_bias=True, l1_reg=l1, tol=1e-10, max_iter=max_iter)
    fast, slow = _fast(df, e), _slow(df, e)
    for g in range(3):
        assert np.max(np.abs(fast[g] - slow[g])) < 1e-9 * max(1.0, np.max(np.abs(slow[g]))), g


# ---- 5. independence and reproducibility ----
def test_group_independent_of_the_others():
    rng = np.random.default_rng(21)
    sizes = rng.integers(20, 300, 10_000)
    sizes[:3] = [9000, 8193, 129]
    y, X, gid = _groups(22, sizes, 4, tie_below=12)
    offs = group_offsets(np.bincount(gid))
    kw = _expr(4, add_bias=True, l2_reg=1e-3, tol=1e-10).kwargs
    everything = _coeffs(_call_by("pl_logistic_by", y, X, offs, kw))
    again = _coeffs(_call_by("pl_logistic_by", y, X, offs, kw))
    assert np.array_equal(_bits(everything), _bits(again))
    for g in (0, 1, 2, 5000):
        lo, hi = offs[g], offs[g + 1]
        alone = _coeffs(_call_by("pl_logistic_by", y[lo:hi], X[lo:hi], [0, hi - lo], kw))
        assert np.array_equal(_bits(alone[0]), _bits(everything[g])), g
    cut = offs[3]                                     # the first three groups only, then the rest with one group added
    head = _coeffs(_call_by("pl_logistic_by", y[:cut], X[:cut], offs[:4], kw))
    assert np.array_equal(_bits(head), _bits(everything[:3]))
    ye, Xe = np.concatenate([y, y[:50]]), np.concatenate([X, X[:50]])
    more = _coeffs(_call_by("pl_logistic_by", ye, Xe, np.append(offs, offs[-1] + 50), kw))
    assert np.array_equal(_bits(more[:-1]), _bits(everything))


def test_chunked_and_sliced_inputs():
    y, X, gid = _groups(23, [700, 9000, 50, 3000], 3)
    offs = group_offsets(np.bincount(gid))
    kw = _expr(3, add_bias=True, tol=1e-10).kwargs
    kwp = _expr(3, add_bias=True, tol=1e-10, return_pred=True).kwargs
    base = _coeffs(_call_by("pl_logistic_by", y, X, offs, kw))
    pbase = _call_by("pl_logistic_pred_by", y, X, offs, kwp).to_numpy(zero_copy_only=False)
    assert np.array_equal(_bits(_coeffs(_call_by("pl_logistic_by", y, X, offs, kw, chunks=5))), _bits(base))
    assert np.array_equal(_bits(_call_by("pl_logistic_pred_by", y, X, offs, kwp, chunks=3).to_numpy(zero_copy_only=False)),
                          _bits(pbase))
    pad = 37                                          # the same rows as slices of longer arrays
    yy, XX = np.concatenate([np.zeros(pad), y]), np.concatenate([np.zeros((pad, 3)), X])
    ins = [pa.array(offs), pa.array(yy).slice(pad)] + [pa.array(XX[:, i]).slice(pad) for i in range(3)]
    names = ["__offsets__", "y", "x0", "x1", "x2"]
    assert np.array_equal(_bits(_coeffs(_harness.call_plugin("pl_logistic_by", ins, names, kw))), _bits(base))


# ---- 6. scale and errors ----
def test_ten_thousand_groups_sample_against_loop():
    rng = np.random.default_rng(24)
    sizes = rng.integers(800, 1200, 10_000)
    y, X, gid = _groups(25, sizes, 8)
    df = _frame(y, X, gid)
    e = _expr(8, add_bias=True, tol=1e-10)
    fast = _fast(df, e)
    assert len(fast) == 10_000
    for g in rng.choice(10_000, 200, replace=False):
        ref = _slow(df.filter(gid == g), e)[0]
        assert np.max(np.abs(fast[g] - ref)) < 1e-9 * max(1.0, np.max(np.abs(ref))), g


def test_offset_and_feature_errors():
    y, X, gid = _groups(26, [30, 40], 2)
    kw = _expr(2).kwargs
    for sym, lr_sym in (("pl_logistic_by", "pl_lr_by"), ("pl_logistic_pred_by", "pl_lr_pred_by")):
        for offs in ([0, 30, 71], [0, 50, 30, 70], [5, 30, 70]):
            with pytest.raises(pds.PdsbError) as a:
                _call_by(sym, y, X, offs, kw)
            with pytest.raises(pds.PdsbError) as b:
                _call_by(lr_sym, y, X, offs, pds.lin_reg("x0", target="y").kwargs)
            assert str(a.value) == str(b.value)
    Xw = np.random.default_rng(0).standard_normal((70, 65))
    with pytest.raises(pds.PdsbError) as a:
        _call_by("pl_logistic_by", y, Xw, [0, 30, 70], kw)
    with pytest.raises(pds.PdsbError) as b:
        _harness.call_plugin("pl_logistic_coeffs", [pa.array(y)] + [pa.array(Xw[:, i]) for i in range(65)],
                             ["y"] + [f"x{i}" for i in range(65)], kw)
    assert str(a.value) == str(b.value)


def test_device_entry_status_and_iterations():
    import torch

    from polars_ds_extension_b200 import device as dev

    y, X, gid = _groups(27, [600, 900, 800], 3)
    X[np.flatnonzero(gid == 2)[5], 1] = np.inf
    offs = group_offsets(np.bincount(gid))
    Xd = torch.tensor(np.ascontiguousarray(X.T), device="cuda")
    yd = torch.tensor(y, device="cuda")
    od = torch.tensor(offs, device="cuda")
    beta, status, n_iter = dev.grouped_logistic(Xd, yd, od, add_bias=True, tol=1e-10, max_iter=100)
    st = status.cpu().numpy()
    assert st[0] == st[1] == LOGISTIC_CONVERGED and st[2] == LOGISTIC_FAILED
    assert np.all(np.isnan(beta[2].cpu().numpy()))
    # the loop's own iteration counts: the call runs as long as its slowest group
    runs = []
    for g in range(2):
        lo, hi = offs[g], offs[g + 1]
        for k in range(1, 100):
            b, s, it = dev.grouped_logistic(Xd[:, lo:hi].contiguous(), yd[lo:hi].contiguous(),
                                            torch.tensor([0, hi - lo], device="cuda"), add_bias=True, tol=1e-10,
                                            max_iter=k)
            if s.item() == LOGISTIC_CONVERGED:
                runs.append(k)
                break
            assert s.item() == LOGISTIC_MAX_ITER and it == k
    assert n_iter == max(runs)
    beta2, status2, n2 = dev.grouped_logistic(Xd, yd, od, add_bias=True, tol=1e-10, max_iter=2)
    assert n2 == 2 and np.all(status2.cpu().numpy()[:2] == LOGISTIC_MAX_ITER)
    # the coefficients of the loop on the same rows
    e = _expr(3, add_bias=True, tol=1e-10, max_iter=100)
    slow = _slow(_frame(y, X, gid), e)
    for g in range(2):
        assert np.max(np.abs(beta[g].cpu().numpy() - slow[g])) < 1e-9 * max(1.0, np.max(np.abs(slow[g])))


@pytest.mark.parametrize("p", [4, 14])
def test_device_entry_launch_count(p):
    """One work list per call (count, scan, item -> rows and group), the state's init, then per iteration pass A and
    the step (no item sum: every group here is one item)."""
    import torch

    from polars_ds_extension_b200 import device as dev

    y, X, gid = _groups(41, [300, 5000, 40], p)
    od = torch.tensor(group_offsets(np.bincount(gid)), device="cuda")
    Xd = torch.tensor(np.ascontiguousarray(X.T), device="cuda")
    yd = torch.tensor(y, device="cuda")
    c0 = lib().pdsb_kernel_launch_count()
    _, _, n_iter = dev.grouped_logistic(Xd, yd, od, add_bias=True, l2_reg=0.01, max_iter=50)
    assert lib().pdsb_kernel_launch_count() - c0 == 4 + 2 * n_iter
