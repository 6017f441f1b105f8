"""Parity tests proper: the CUDA path, called through the plugin C ABI exactly like Polars would call it
(pickled kwargs + Arrow C data -> `_polars_plugin_pl_lr*` in _polars_ds_b200.so), checked against

  (a) the reference's own known-answer tests (tests/cases.py: same seeds, external checkers, tolerances), and
  (b) the CPU oracle on the same seeded inputs (oracle/lin_reg_oracle.py), element by element.

Tolerances (north_star): 1e-6 relative for f64, 1e-4 relative for f32.
"""
import numpy as np
import pytest

import polars_ds_extension_b200 as pds
import polars_ds_extension_b200.config as cfg
from polars_ds_extension_b200 import Frame
from tests import cases
from tests.backends import OracleBackend, PluginBackend

pytestmark = pytest.mark.gpu

GPU = PluginBackend()
ORC = OracleBackend()


@pytest.mark.parametrize("case", cases.ALL_CASES, ids=lambda f: f.__name__)
def test_reference_cases_f64(case, monkeypatch):
    monkeypatch.setattr(cfg, "LIN_REG_EXPR_F64", True)
    case(GPU)


@pytest.mark.parametrize("case", cases.ALL_CASES, ids=lambda f: f.__name__)
def test_reference_cases_f32(case, monkeypatch):
    monkeypatch.setattr(cfg, "LIN_REG_EXPR_F64", False)
    case(GPU)


from tests.parity_rule import accept_f32, accept_f64, rel as _rel  # noqa: E402


def _frame(seed, n, p, dtype=np.float64, noise=0.1):
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((n, p))
    beta = ((np.arange(p) % 7) - 3) / 4.0
    y = X @ beta + noise * rng.standard_normal(n) + 0.5
    d = {f"x{i}": X[:, i].astype(dtype) for i in range(p)}
    d["y"] = y.astype(dtype)
    return Frame(d), [f"x{i}" for i in range(p)]


def _three(monkeypatch, f64, df, make):
    """(gpu, oracle in the same precision, f64 oracle on the same inputs) of the expression `make()` builds."""
    monkeypatch.setattr(cfg, "LIN_REG_EXPR_F64", f64)
    e = make()
    g, o = GPU.eval(df, e), ORC.eval(df, e)
    if f64:
        return g, o, o
    monkeypatch.setattr(cfg, "LIN_REG_EXPR_F64", True)
    truth = ORC.eval(df, make())
    monkeypatch.setattr(cfg, "LIN_REG_EXPR_F64", False)
    return g, o, truth


def _accept(f64, g, o, truth, what=""):
    if f64:
        accept_f64(g, o, what)
    else:
        accept_f32(g, o, truth, what)


@pytest.mark.parametrize("f64", [True, False])
@pytest.mark.parametrize("n,p,bias", [(100_000, 4, True), (20_000, 32, False), (3_000, 64, True), (257, 1, True),
                                      (8_192, 64, False), (300_000, 64, True), (1_000_000, 32, False)])
def test_lin_reg_vs_oracle(monkeypatch, f64, n, p, bias):
    """config[0] at full size (100k x 4 f64, bias), config[1] / config[4] shapes up to 1e6 rows through the plugin ABI —
    8 192 x 64, 300 000 x 64 and 1e6 x 32 run on the wgmma kernel, 100 000 x 4 on the register-moments kernel."""
    df, xs = _frame(20 + p, n, p, np.float64 if f64 else np.float32)
    g, o, truth = _three(monkeypatch, f64, df, lambda: pds.lin_reg(*xs, target="y", add_bias=bias))
    _accept(f64, g, o, truth, "coeffs")
    if not f64 and n >= 4096:
        from polars_ds_extension_b200._lib import lib
        # the tensor-core kernel did this fit — or, for few features on many rows, the register-moments kernel (path 3)
        assert lib().pdsb_last_moments_path() == (3 if (p <= 10 and n >= 65536) else 1)
    g, o, truth = _three(monkeypatch, f64, df, lambda: pds.lin_reg(*xs, target="y", add_bias=bias, return_pred=True))
    _accept(f64, g["pred"][0], o["pred"][0], truth["pred"][0], "pred")
    # residuals are differences of O(1) numbers: same absolute scale as the predictions
    scale = np.abs(truth["pred"][0]).max()
    er_g = np.max(np.abs(g["resid"][0] - truth["resid"][0])) / scale
    er_o = np.max(np.abs(o["resid"][0] - truth["resid"][0])) / scale
    assert er_g <= (1e-6 if f64 else max(er_o, 2e-6))


@pytest.mark.parametrize("f64", [True, False])
def test_solvers_and_ridge_vs_oracle(monkeypatch, f64):
    df, xs = _frame(31, 5000, 8, np.float64 if f64 else np.float32)
    for solver in ["qr", "svd", "choleskey", "cholesky"]:
        for l2 in [0.0, 0.5]:
            g, o, truth = _three(monkeypatch, f64, df, lambda: pds.lin_reg(*xs, target="y", add_bias=True, solver=solver, l2_reg=l2))
            _accept(f64, g, o, truth, f"{solver} l2={l2}")


@pytest.mark.parametrize("f64", [True, False])
def test_report_vs_oracle(monkeypatch, f64):
    df, xs = _frame(32, 4000, 5, np.float64 if f64 else np.float32)
    for se in ["se", "hc0", "hc1", "hc2", "hc3"]:
        g, o, truth = _three(monkeypatch, f64, df, lambda: pds.lin_reg_report(*xs, target="y", add_bias=True, std_err=se))
        assert g["features"] == o["features"]
        for k in o:
            if k == "features":
                continue
            if k == "p>|t|":
                # p-values span many decades: element-wise relative comparison on ln p (a vector-relative rule would only
                # test the largest one)
                lg, lo, lt = (np.log(np.maximum(np.asarray(v[k], np.float64), 1e-300)) for v in (g, o, truth))
                eg, eo = np.max(np.abs(lg - lt) / np.abs(lt)), np.max(np.abs(lo - lt) / np.abs(lt))
                assert eg <= (1e-6 if f64 else max(eo, 2e-6)), (se, k, eg, eo)
            else:
                _accept(f64, g[k], o[k], truth[k], f"{se}:{k}")


@pytest.mark.parametrize("f64", [True, False])
@pytest.mark.parametrize("window,p,bias,l2,n", [(1024, 8, False, 0.0, 0), (37, 3, True, 0.1, 0), (2, 1, False, 0.0, 0),
                                                (5000, 4, True, 0.0, 0), (1024, 8, False, 0.0, 1_000_000),
                                                (1024, 8, True, 0.0, 0), (100, 11, True, 0.0, 0), (64, 14, True, 0.05, 0),
                                                (300, 30, False, 0.0, 0)])
def test_rolling_vs_definition(monkeypatch, f64, window, p, bias, l2, n):
    """config[3] (window 1024, 8 features) up to 1e6 rows through the plugin ABI: every checked row == OLS on its window
    (the identity the reference's tests assert, test_linear_exprs.py:814-854), >= 1000 rows checked at 1e6.  Coefficient
    counts 1..9 take the packed f32 kernel (f32) / the lane-per-moment kernel (f64), 10..12 the lane-per-moment kernel,
    above 12 the generic shared-memory path (the reference has no limit, lr_online_solvers.rs:148-301)."""
    monkeypatch.setattr(cfg, "LIN_REG_EXPR_F64", f64)
    n = n or max(3 * window + 77, 4000)
    df, xs = _frame(40 + p, n, p, np.float64 if f64 else np.float32)
    r = GPU.eval(df, pds.rolling_lin_reg(*xs, target="y", window_size=window, add_bias=bias, l2_reg=l2))
    X = np.column_stack([df[c].to_numpy().astype(np.float64) for c in xs] + ([np.ones(n)] if bias else []))
    y = df["y"].to_numpy().astype(np.float64)
    assert all(c is None for c in r["coeffs"][: window - 1])
    from oracle.lin_reg_oracle import window_ols

    rng = np.random.default_rng(1)
    e32 = None
    if not f64:
        # the f32 reference restatement: the oracle's sequential Woodbury walk in f32 (faer_rolling_lr).  On long frames it
        # is run on segments (a fresh window fit at the segment start, like the reference's own start), which also keeps
        # its drift — the reference's f32 error grows with the rows walked — to a segment's length.
        seg = max(2 * window, 1500)
        starts = [0] if n <= 20_000 else sorted(set(rng.integers(0, n - seg, 10).tolist()))
        e32 = {}
        for s0 in starts:
            m = n if n <= 20_000 else seg
            o = ORC.eval(df.slice(s0, m), pds.rolling_lin_reg(*xs, target="y", window_size=window, add_bias=bias, l2_reg=l2))
            for i in range(window - 1, m):
                e32.setdefault(s0 + i, o["coeffs"][i])
        pool = np.array(sorted(e32))
        rows = set(pool[rng.integers(0, len(pool), 1500 if n >= 1_000_000 else 60)].tolist()) | ({window - 1, min(n - 1, 2 * window)} & set(e32))
    else:
        rows = set(rng.integers(window - 1, n, 60).tolist()) | {window - 1, n - 1, window, min(n - 1, 2 * window)}
    for j in sorted(rows):
        truth = window_ols(X, y, j - window + 1, j + 1, lam=l2, add_bias=bias)
        if f64:
            accept_f64(r["coeffs"][j], truth, f"row {j}")
            assert abs(r["pred"][0][j] - X[j] @ truth) <= 1e-6 * max(1.0, abs(X[j] @ truth))
        else:
            eg, eo, _ = accept_f32(r["coeffs"][j], e32[j], truth, f"row {j}")
            assert abs(r["pred"][0][j] - X[j] @ truth) <= max(1e-4, 2 * eo) * max(1.0, np.abs(X[j]) @ np.abs(truth))
    if not f64 and n >= 1_000_000:
        assert len(rows) >= 1000
    assert r["pred"][1][window - 1:].all() and not r["pred"][1][: window - 1].any()


@pytest.mark.parametrize("f64", [True, False])
def test_recursive_vs_definition(monkeypatch, f64):
    monkeypatch.setattr(cfg, "LIN_REG_EXPR_F64", f64)
    n, p = 6000, 4
    df, xs = _frame(50, n, p, np.float64 if f64 else np.float32)
    r = GPU.eval(df, pds.recursive_lin_reg(*xs, target="y", start_with=10, add_bias=True, l2_reg=0.01))
    X = np.column_stack([df[c].to_numpy().astype(np.float64) for c in xs] + [np.ones(n)])
    y = df["y"].to_numpy().astype(np.float64)
    from oracle.lin_reg_oracle import window_ols

    o32 = None if f64 else ORC.eval(df, pds.recursive_lin_reg(*xs, target="y", start_with=10, add_bias=True, l2_reg=0.01))
    for j in [9, 10, 50, 1023, 1024, 1025, 3000, n - 1]:
        truth = window_ols(X, y, 0, j + 1, lam=0.01, add_bias=True)
        if f64:
            accept_f64(r["coeffs"][j], truth, f"row {j}")
        else:
            accept_f32(r["coeffs"][j], o32["coeffs"][j], truth, f"row {j}")
    assert r["coeffs"][8] is None
    # and against the oracle's sequential Woodbury restatement on a short prefix (f64 only: f32 Woodbury drifts)
    if f64:
        o = ORC.eval(df.limit(300), pds.recursive_lin_reg(*xs, target="y", start_with=10, add_bias=True, l2_reg=0.01))
        for j in range(9, 300, 17):
            assert _rel(r["coeffs"][j], o["coeffs"][j]) < 1e-6


@pytest.mark.parametrize("f64", [True, False])
@pytest.mark.parametrize("big", [False, True])
def test_grouped_config_shape(monkeypatch, f64, big):
    """config[2]: ragged contiguous groups x 8 features through the batched symbol == per-group oracle; `big` = 1e4 groups
    of 80..120 rows (the config's group COUNT at 1 % of its rows)."""
    rng = np.random.default_rng(60)
    sizes = rng.integers(80, 121, 10_000).tolist() if big else rng.integers(800, 1200, 40).tolist() + [9000, 20000, 9]
    gid = np.repeat(np.arange(len(sizes)), sizes)
    n = len(gid)
    df, xs = _frame(61, n, 8, np.float64 if f64 else np.float32)
    df = df.with_columns(g=gid)
    monkeypatch.setattr(cfg, "LIN_REG_EXPR_F64", f64)
    fast = GPU.group_eval(df, "g", pds.lin_reg(*xs, target="y", add_bias=True), fast=True)
    assert len(fast) == len(sizes)
    check = rng.integers(0, len(sizes), 200).tolist() if big else [0, 1, 17, 40, 41, 42]
    for g in check:
        sub = df.filter(gid == g)
        monkeypatch.setattr(cfg, "LIN_REG_EXPR_F64", f64)
        o = ORC.eval(sub, pds.lin_reg(*xs, target="y", add_bias=True))
        if f64:
            accept_f64(fast[g], o, f"group {g}")
        else:
            monkeypatch.setattr(cfg, "LIN_REG_EXPR_F64", True)
            truth = ORC.eval(sub, pds.lin_reg(*xs, target="y", add_bias=True))
            accept_f32(fast[g], o, truth, f"group {g}")


def test_bit_reproducible(monkeypatch):
    monkeypatch.setattr(cfg, "LIN_REG_EXPR_F64", False)
    df, xs = _frame(70, 50_000, 16, np.float32)
    e = pds.lin_reg(*xs, target="y", add_bias=True, return_pred=True)
    a, b = GPU.eval(df, e), GPU.eval(df, e)
    assert np.array_equal(a["pred"][0], b["pred"][0])


def test_pageable_inputs_take_the_staged_route_and_match_pinned(monkeypatch):
    """Polars hands a plugin pageable buffers: columns >= 1 MiB go through the pinned staging ring (h2d.cc); the result is
    bit-identical to the same call on page-locked inputs (same bytes reach the same kernels)."""
    import pyarrow as pa
    import torch

    from polars_ds_extension_b200 import _harness
    from polars_ds_extension_b200._lib import lib

    n, p = 3_000_000, 6
    rng = np.random.default_rng(5)
    cols = [rng.standard_normal(n, dtype=np.float32) for _ in range(p + 1)]
    kw = {"bias": True, "null_policy": "skip", "l1_reg": 0.0, "l2_reg": 0.0, "solver": "qr", "tol": 1e-5, "max_iter": 200,
          "weighted": False, "positive": False, "singular_x_tol": 1e-6}
    names = ["y"] + [f"x{i}" for i in range(p)]
    a = _harness.call_plugin("pl_lr_pred_f32", [pa.array(c) for c in cols], names, kw)
    assert lib().pdsb_last_staged_bytes() == (p + 1) * n * 4
    pinned = [torch.from_numpy(c).pin_memory().numpy() for c in cols]
    b = _harness.call_plugin("pl_lr_pred_f32", [pa.array(c) for c in pinned], names, kw)
    assert lib().pdsb_last_staged_bytes() == 0
    assert a.field("pred").equals(b.field("pred")) and a.field("resid").equals(b.field("resid"))


@pytest.mark.parametrize("f64", [True, False])
@pytest.mark.parametrize("kind", ["lasso", "enet", "nnls", "positive_ridge", "wide"])
def test_grouped_iterative_and_wide(monkeypatch, f64, kind):
    """The batched group_by entry beyond OLS / ridge: lasso, elastic net, NNLS and positive ridge per group on the reduced
    Grams (one launch sequence instead of one ABI call per group), and p > 33 features per group.  Checked against the
    same expression evaluated group by group through the standard symbol (the path Polars itself takes) and against the
    oracle."""
    monkeypatch.setattr(cfg, "LIN_REG_EXPR_F64", f64)
    rng = np.random.default_rng(77)
    p = 40 if kind == "wide" else 5
    sizes = rng.integers(600, 1500, 24).tolist()
    gid = np.repeat(np.arange(len(sizes)), sizes)
    n = len(gid)
    X = np.abs(rng.standard_normal((n, p))) if kind in ("nnls", "positive_ridge") else rng.standard_normal((n, p))
    beta = np.abs(((np.arange(p) % 7) - 3) / 4.0) if kind in ("nnls", "positive_ridge") else ((np.arange(p) % 7) - 3) / 4.0
    y = X @ beta + 0.1 * rng.standard_normal(n) + 0.5
    dt = np.float64 if f64 else np.float32
    df = Frame({f"x{i}": X[:, i].astype(dt) for i in range(p)} | {"y": y.astype(dt)}).with_columns(g=gid)
    xs = [f"x{i}" for i in range(p)]
    make = {
        "lasso": lambda: pds.lin_reg(*xs, target="y", add_bias=True, l1_reg=0.01, tol=1e-9, max_iter=5000),
        "enet": lambda: pds.lin_reg(*xs, target="y", add_bias=False, l1_reg=0.01, l2_reg=0.02, tol=1e-9, max_iter=5000),
        "nnls": lambda: pds.lin_reg(*xs, target="y", add_bias=True, positive=True, tol=1e-10, max_iter=5000),
        "positive_ridge": lambda: pds.lin_reg(*xs, target="y", add_bias=False, positive=True, l2_reg=0.05, tol=1e-9, max_iter=5000),
        "wide": lambda: pds.lin_reg(*xs, target="y", add_bias=True, l2_reg=0.1),
    }[kind]
    e = make()
    fast = GPU.group_eval(df, "g", e, fast=True)
    slow = GPU.group_eval(df, "g", e, fast=False)
    assert len(fast) == len(sizes)
    for g in range(len(sizes)):
        # same arithmetic (f64 iterations on the f64-accumulated Gram): only the moments' summation order differs
        assert _rel(fast[g], slow[g]) < (1e-9 if f64 else 2e-5), (kind, g)
    for g in (0, 7, 23):
        sub = df.filter(gid == g)
        monkeypatch.setattr(cfg, "LIN_REG_EXPR_F64", f64)
        o = ORC.eval(sub, make())
        tol = 1e-6 if f64 else (1e-4 if kind == "wide" else 2e-3)     # f32 twin: 200 / 2000 fixed sweeps, optimiser resolution
        assert _rel(fast[g], o) < tol, (kind, g)
