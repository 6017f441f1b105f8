"""Rolling and recursive lin_reg (K6/K7, `k6_online.cu`) on every pass-C kernel, checked row by row against the window
definition, with and without nulls.

Pass C has three kernels.  `pdsb_last_online_path()` says which one ran, and every case asserts the one it is meant to
cover (D = p + bias coefficients):

  1  packed f32 row pairs   f32, D <= 9: recursive, or rolling with window >= 64 that does not skip nulls
  2  lane-per-moment        f64 with D <= 12; f32 with D = 10..12, with window < 64, or rolling with skip
  3  generic shared memory  D >= 13, either dtype

The truth is the definition in float64, not the oracle's sequential Woodbury walk (which drifts in f32): row r uses the
finite rows of [r-w+1, r] (rolling) or [0, r] (recursive); G = sum z z' + lambda I with lambda on every diagonal entry,
the bias one included (DESIGN.md §5, deviation 4); b = sum z y; beta = G^-1 b.  The window sums are differences of
long-double prefix sums of exact products, so the truth carries no error of its own at these tolerances.

Expected `valid`: rolling r >= w-1, and with skip also count >= min_valid_rows; recursive with skip: row r is finite and
count >= start_with; recursive without skip: r >= start_with - 1.  Invalid rows hold zero coefficients and pred 0.

Acceptance per row (max-norm vector-relative, like tests/parity_rule.py):
  f64  rel(gpu, truth) <= 1e-9 (every window well conditioned: at least 3 D rows, or lambda > 0)
  f32  rel(gpu, truth) <= max(C32 * rel(m32, truth), eps32 * cond(G), 2e-6).  m32 is a float32 Cholesky solve of the
       float32-rounded exact window Gram and X'y: the rounding the kernels cannot avoid.  The packed kernel also rounds a
       64-term f32 scan per step, hence C32 > 1.  m32 is one sample of that rounding and lands much closer to the truth
       than usual on some rows; eps32 * cond(G), the first-order bound of any stable float32 solve of a float32-rounded
       G, keeps such a row from tightening the bound below what the arithmetic allows.
  pred == x_r . beta_r of the returned coefficients to the dtype's rounding: NaN when a feature of row r is null,
       finite when only y is (the reference forms pred from the raw row, NaN for nulls).
"""
import numpy as np
import pytest

# f32 acceptance factor, from an H100 80GB HBM3 at 400 W.  Over every f32 case in this file, the worst
# rel(gpu, truth) / rel(m32, truth) on a row above 2e-6 was 6.99: the packed kernel, recursive, D = 8, start_with 8.  The
# lane-per-moment kernel at window 2 reached 9.8 and 11.4 on rows with cond(G) 98 and 73.  On those rows m32 happened to
# land close to the truth, and the GPU error was within eps32 * cond(G).  No row needs C32 once that term is in the
# bound.
C32 = 8.0
EPS32 = float(np.finfo(np.float32).eps)
F64_TOL = 1e-9
FLOOR = 2e-6
PACKED, LANE, GENERIC = 1, 2, 3
ROUTE_NAME = {PACKED: "packed", LANE: "lane", GENERIC: "generic"}


def _route(f64, D, window, skip=False):
    if D >= 13:
        return GENERIC
    if not f64 and D <= 9 and (window == 0 or (window >= 64 and not skip)):
        return PACKED
    return LANE


def _ridge(D, rows):
    """lambda for windows that can hold fewer than 3 D rows (their Gram may be near singular), 0 otherwise"""
    return 0.0 if rows >= 3 * D else 0.25


# ---------------------------------------------------------------------------------------------------------------------
# data and the definition
# ---------------------------------------------------------------------------------------------------------------------
def _data(seed, n, p, f64, nulls=None, window=0, min_rows=0):
    """X (n, p) and y (n,) as float64 arrays holding values of the data dtype; NaN placed as `nulls` says:
    "x" about 5 % of rows with one null feature, "y" about 5 % null targets, "burst" a run of rows with a null feature
    longer than window - min_rows (rolling: the windows after it fall below min_rows and recover) or rows 50..349
    (recursive: the first valid row moves behind it)."""
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((n, p))
    beta = ((np.arange(p) % 7) - 3) / 4.0
    y = X @ beta + 0.1 * rng.standard_normal(n) + 0.5
    if nulls == "x":
        rows = np.flatnonzero(rng.random(n) < 0.05)
        X[rows, rng.integers(0, p, rows.size)] = np.nan
    elif nulls == "y":
        y[rng.random(n) < 0.05] = np.nan
    elif nulls == "burst":
        a, b = (1500, 1500 + window - min_rows + 7) if window else (50, 350)
        X[a:b, 0] = np.nan
    dt = np.float64 if f64 else np.float32
    return X.astype(dt).astype(np.float64), y.astype(dt).astype(np.float64)


def _design(X, bias):
    return np.column_stack([X, np.ones(len(X))]) if bias else X


def _moments(Z, y):
    """per-row [z z' (D*D), z y (D), 1] of the finite rows, zero for the others (exact products for f32 data)"""
    fin = np.isfinite(Z).all(1) & np.isfinite(y)
    Z = np.where(fin[:, None], Z, 0.0)
    yz = np.where(fin, y, 0.0)
    n, D = Z.shape
    return np.concatenate([(Z[:, :, None] * Z[:, None, :]).reshape(n, D * D), Z * yz[:, None], fin[:, None]], axis=1)


def _prefix_base(Z, y, end, block=1 << 16):
    """long-double sum of the moments of rows [0, end)"""
    acc = np.zeros(Z.shape[1] * (Z.shape[1] + 1) + 1, np.longdouble)
    for a in range(0, end, block):
        acc += _moments(Z[a:min(a + block, end)], y[a:min(a + block, end)]).sum(0, dtype=np.longdouble)
    return acc


def _expect(Z, y, window, min_rows, skip, lam, f64, first=0, base=None, drop=None, bias_lambda=True):
    """Expected valid flags, coefficients (f64 truth, and the f32 model m32) and Grams for every row of Z (design rows
    first .. first + len(Z) - 1 of the frame).  Rolling: Z must start window - 1 rows before the first row whose window
    is complete.  Recursive: `base` = moments of the rows before `first`.  `drop` = a row (index into Z) to leave out
    and `bias_lambda=False` leaves lambda off the last diagonal entry: the perturbations of the sensitivity check."""
    n, D = Z.shape
    M = _moments(Z, y)
    if drop is not None:
        M[drop] = 0.0
    P = np.zeros((n + 1, M.shape[1]), np.longdouble)
    np.cumsum(M, axis=0, dtype=np.longdouble, out=P[1:])
    hi = np.arange(1, n + 1)
    S = P[hi] - P[np.maximum(hi - window, 0)] if window else P[hi] + (0 if base is None else base)
    cnt = S[:, -1].astype(np.float64)
    r = first + np.arange(n)
    fin = np.isfinite(Z).all(1) & np.isfinite(y)
    if window:
        valid = (r >= window - 1) & ((cnt >= min_rows) if skip else True)
        if first > 0:
            valid &= np.arange(n) >= window - 1                 # windows that start before Z: not solved (not checked)
    elif skip:
        valid = fin & (cnt >= min_rows)
    else:
        valid = r >= min_rows - 1
    lam_diag = np.full(D, lam)
    if not bias_lambda:
        lam_diag[-1] = 0.0
    G = S[:, :D * D].astype(np.float64).reshape(n, D, D) + np.diag(lam_diag)
    b = S[:, D * D:D * D + D].astype(np.float64)
    truth = np.full((n, D), np.nan)
    m32 = np.full((n, D), np.nan)
    v = np.flatnonzero(valid)
    if v.size:
        truth[v] = np.linalg.solve(G[v], b[v][..., None])[..., 0]
        if not f64:
            G32 = S[v, :D * D].astype(np.float32).reshape(-1, D, D) + np.diag(lam_diag.astype(np.float32))
            L = np.linalg.cholesky(G32)
            u = np.linalg.solve(L, S[v, D * D:D * D + D].astype(np.float32)[..., None])
            m32[v] = np.linalg.solve(np.swapaxes(L, 1, 2), u)[..., 0]
    return valid, truth, m32, G


def _rel_rows(a, t):
    return np.abs(a - t).max(1) / np.maximum(np.abs(t).max(1), 1e-300)


def _coeffs_ok(f64, got, truth, m32, G, c32=C32):
    """per-row acceptance of coefficients `got` against the truth; returns (ok, rel(got), bound, floor of the bound)"""
    eg = _rel_rows(np.asarray(got, np.float64), truth)
    if f64:
        return eg <= F64_TOL, eg, np.full(eg.shape, F64_TOL), np.full(eg.shape, F64_TOL)
    floor = np.maximum(EPS32 * np.linalg.cond(G), FLOOR)
    bound = np.maximum(c32 * _rel_rows(m32, truth), floor)
    return eg <= bound, eg, bound, floor


def _compare(what, f64, Z, exp, coeffs, pred, valid, rows=None, c32=C32):
    """Assert the device outputs against `_expect`'s on `rows` (indices into Z, default all).  Returns the worst f32
    ratio rel(gpu, truth) / rel(m32, truth) over rows above the floor (the C32 this case needs)."""
    ev, truth, m32, G = exp
    rows = np.arange(len(Z)) if rows is None else np.asarray(rows)
    ev, truth, m32, G, Z = ev[rows], truth[rows], m32[rows], G[rows], Z[rows]
    coeffs, pred, valid = np.asarray(coeffs, np.float64)[rows], np.asarray(pred, np.float64)[rows], np.asarray(valid)[rows]
    D = Z.shape[1]
    got_valid = valid.astype(bool)
    bad = np.flatnonzero(got_valid != ev)
    assert bad.size == 0, (f"{what}: valid differs at {bad.size} rows, first {rows[bad[:8]].tolist()}: "
                           f"got {got_valid[bad[:8]].astype(int).tolist()}")
    inv = ~ev
    assert not coeffs[inv].any() and not pred[inv].any(), f"{what}: an invalid row has nonzero coefficients or pred"
    v = np.flatnonzero(ev)
    assert v.size > 0, f"{what}: no valid row checked"
    ok, eg, bound, floor = _coeffs_ok(f64, coeffs[v], truth[v], m32[v], G[v], c32)
    if not ok.all():
        i = int(np.argmax(eg / bound))
        raise AssertionError(f"{what}: row {rows[v[i]]}: rel(gpu, truth) {eg[i]:.3e} > bound {bound[i]:.3e} "
                             f"({int((~ok).sum())} rows fail), cond(G) {np.linalg.cond(G[v[i]]):.3e}")
    ratio = 0.0
    if not f64:
        em = _rel_rows(m32[v], truth[v])
        above = eg > floor
        if above.any():
            ratio = float(np.max(eg[above] / np.maximum(em[above], 1e-300)))
    # pred: x_r . beta_r of the returned coefficients, NaN exactly where a feature of the row is null
    xnan = np.isnan(Z[v]).any(1)
    pnan = np.isnan(pred[v])
    bad = np.flatnonzero(xnan != pnan)
    assert bad.size == 0, (f"{what}: pred NaN pattern differs at {bad.size} valid rows, first {rows[v[bad[:8]]].tolist()}: "
                           f"pred {pred[v[bad[:8]]].tolist()}")
    f = v[~xnan]
    xb = (Z[f] * coeffs[f]).sum(1)
    eps = np.finfo(np.float64 if f64 else np.float32).eps
    tol = 2 * D * eps * (np.abs(Z[f]) * np.abs(coeffs[f])).sum(1) + 1e-30
    err = np.abs(pred[f] - xb)
    if not (err <= tol).all():
        i = int(np.argmax(err / tol))
        raise AssertionError(f"{what}: row {rows[f[i]]}: pred {pred[f[i]]!r} != x . beta {xb[i]!r}")
    return ratio


# ---------------------------------------------------------------------------------------------------------------------
# the device call
# ---------------------------------------------------------------------------------------------------------------------
def _gpu(X, y, f64, bias, window, min_rows, skip, lam):
    """device.online_lin_reg on (X, y) -> (coeffs, pred, valid) as numpy, and the pass-C kernel that ran"""
    import torch

    from polars_ds_extension_b200 import device as dev
    from polars_ds_extension_b200._lib import lib

    dt = torch.float64 if f64 else torch.float32
    Xt = torch.from_numpy(np.ascontiguousarray(X.T)).to(device="cuda", dtype=dt)
    yt = torch.from_numpy(y).to(device="cuda", dtype=dt)
    co, pr, va = dev.online_lin_reg(Xt, yt, window=window, min_rows=min_rows, add_bias=bias, l2_reg=lam, skip=skip)
    route = int(lib().pdsb_last_online_path())
    return co.cpu().numpy(), pr.cpu().numpy(), va.cpu().numpy(), route


def _run(record_property, f64, D, bias, window, start, n, nulls=None, min_rows=None, seed=0):
    """One case on all rows: rolling when window > 0 (skip with min_rows when `nulls`), else recursive from `start`."""
    p = D - int(bias)
    skip = nulls is not None
    if window:
        mr = min_rows if skip else window
        lam = _ridge(D, mr if skip else window)
    else:
        mr = start
        lam = _ridge(D, start)
    X, y = _data(seed, n, p, f64, nulls, window, mr)
    Z = _design(X, bias)
    co, pr, va, route = _gpu(X, y, f64, bias, window, mr, skip, lam)
    what = (f"{'f64' if f64 else 'f32'} D={D} bias={bias} {'w=' + str(window) if window else 'start=' + str(start)} "
            f"n={n} nulls={nulls} min_rows={mr} lambda={lam}")
    want = _route(f64, D, window, skip)
    assert route == want, f"{what}: pass C ran the {ROUTE_NAME.get(route, route)} kernel, not the {ROUTE_NAME[want]} one"
    ratio = _compare(what, f64, Z, _expect(Z, y, window, mr, skip, lam, f64), co, pr, va)
    if not f64:
        record_property("f32_ratio", ratio)


# ---------------------------------------------------------------------------------------------------------------------
# cases: every (route, D) rolling and recursive in each dtype the route serves
# ---------------------------------------------------------------------------------------------------------------------
PACKED_W = [64, 65, 127, 1024, 1025, 3000]
LANE32_W = [2, 33, 63]
F64_W = [2, 63, 64, 700, 1024, 1025]         # under half a chain, the lane kernel sums its head rows directly
# odd and not a multiple of 64; a multiple of 1024; under 1024 + 64 rows (the packed kernel gets no interior chain)
NS = [5003, 4096, 1077, 2989]


def _starts(D):
    return [1, D, 1500]


def _plain_cases():
    out = []

    def add(f64, D, window, start, i):
        bias = D > 1 and (D % 2 == 0) == (window > 0)
        n = NS[i % len(NS)]
        if n < max(window, start) + 100:
            n = 2 * max(window, start) + 1001
        if D >= 20:
            n = min(n, 3001)
        route = ROUTE_NAME[_route(f64, D, window)]
        kind = f"w{window}" if window else f"start{start}"
        out.append(pytest.param(f64, D, bias, window, start, n,
                                id=f"{route}-{'f64' if f64 else 'f32'}-D{D}-{'bias' if bias else 'nobias'}-{kind}-n{n}"))

    for D in range(1, 10):                                           # packed, f32
        add(False, D, PACKED_W[(D - 1) % len(PACKED_W)], 0, D)
        add(False, D, 0, _starts(D)[(D - 1) % 3], D + 1)
    for D in range(1, 13):                                           # lane-per-moment, f32: short windows; D = 10..12
        add(False, D, LANE32_W[(D - 1) % len(LANE32_W)], 0, D + 2)
    for D in (10, 11, 12):
        add(False, D, 0, _starts(D)[D % 3], D)
    for D in range(1, 13):                                           # lane-per-moment, f64
        add(True, D, F64_W[(D - 1) % len(F64_W)], 0, D + 3)
        add(True, D, 0, _starts(D)[D % 3], D)
    for j, D in enumerate((13, 20, 40)):                             # generic, both dtypes
        for f64 in (False, True):
            add(f64, D, (63, 1025, 127)[j], 0, j + f64)
            add(f64, D, 0, _starts(D)[(j + f64) % 3], j)
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("f64,D,bias,window,start,n", _plain_cases())
def test_online_vs_definition(record_property, f64, D, bias, window, start, n):
    _run(record_property, f64, D, bias, window, start, n, seed=1000 + 97 * D + window + start)


# (dtype, D, bias, window or 0, start, nulls, min_rows as "D" / "half" of the window / a number)
_NULL_CASES = [
    # f32, D <= 9, window >= 64: rolling with skip runs on the lane-per-moment kernel, recursive on the packed one
    (False, 8, True, 64, 0, "x", "D"),
    (False, 9, False, 1024, 0, "y", "half"),
    (False, 5, True, 127, 0, "burst", "D"),
    (False, 3, False, 65, 0, "burst", "half"),
    (False, 8, True, 0, 8, "x", None),
    (False, 9, False, 0, 1500, "y", None),
    (False, 4, True, 0, 200, "burst", None),
    # lane-per-moment, f32 (window < 64, or D = 10..12)
    (False, 5, True, 33, 0, "x", "D"),
    (False, 7, False, 63, 0, "y", "half"),
    (False, 11, True, 1024, 0, "burst", "D"),
    (False, 7, True, 600, 0, "x", "half"),
    (False, 10, False, 0, 10, "x", None),
    (False, 11, True, 0, 1500, "y", None),
    (False, 12, False, 0, 200, "burst", None),
    # lane-per-moment, f64
    (True, 8, True, 64, 0, "x", "D"),
    (True, 9, False, 1025, 0, "y", "half"),
    (True, 5, True, 63, 0, "burst", "D"),
    (True, 12, False, 0, 12, "x", None),
    (True, 8, True, 0, 1500, "y", None),
    (True, 5, False, 0, 200, "burst", None),
    # generic
    (False, 13, True, 127, 0, "x", "D"),
    (True, 13, False, 127, 0, "y", "half"),
    (True, 20, True, 200, 0, "burst", "D"),
    (False, 20, False, 200, 0, "burst", "half"),
    (False, 13, True, 0, 13, "x", None),
    (True, 13, False, 0, 1500, "y", None),
    (False, 20, True, 0, 200, "burst", None),
    (True, 20, False, 0, 20, "x", None),
]


def _null_params():
    out = []
    for f64, D, bias, window, start, nulls, mr in _NULL_CASES:
        min_rows = None if not window else (D if mr == "D" else window // 2)
        route = ROUTE_NAME[_route(f64, D, window, True)]
        kind = f"w{window}-min{min_rows}" if window else f"start{start}"
        out.append(pytest.param(f64, D, bias, window, start, nulls, min_rows,
                                id=f"{route}-{'f64' if f64 else 'f32'}-D{D}-{kind}-{nulls}"))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("f64,D,bias,window,start,nulls,min_rows", _null_params())
def test_online_skip_nulls_vs_definition(record_property, f64, D, bias, window, start, nulls, min_rows):
    """null_policy="skip": null rows leave the windows, windows below min_valid_rows are invalid, and the prediction of
    a valid row is formed from its raw values (NaN for a null feature, finite when only y is null)."""
    n = 4096 if (D + window) % 3 == 0 else 5003
    _run(record_property, f64, D, bias, window, start, n, nulls=nulls, min_rows=min_rows,
         seed=2000 + 31 * D + window + start)


# ---------------------------------------------------------------------------------------------------------------------
# size: pass B carries between blocks of 1024 chains
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("window", [1024, 0], ids=["rolling1024", "recursive"])
@pytest.mark.parametrize("f64", [False, True], ids=["f32", "f64"])
def test_three_scan_blocks(record_property, f64, window):
    """2 200 001 rows = 2149 chains of 1024 rows: the chain scan runs over three 1024-chain blocks and carries between
    them.  Every row of chains 1023..1025 and 2047..2049 and the last row are checked."""
    n, D, start = 2_200_001, 8, 1500
    X, y = _data(3000 + window, n, D, f64)
    co, pr, va, route = _gpu(X, y, f64, False, window, window or start, False, 0.0)
    want = _route(f64, D, window)
    assert route == want, f"pass C ran the {ROUTE_NAME.get(route, route)} kernel, not the {ROUTE_NAME[want]} one"
    ratio = 0.0
    base, done = np.zeros(D * D + D + 1, np.longdouble), 0
    for a, b in [(1023 * 1024, 1026 * 1024), (2047 * 1024, 2050 * 1024), (n - 1, n)]:
        what = f"{'f64' if f64 else 'f32'} n={n} {'w=' + str(window) if window else 'start=' + str(start)} rows {a}..{b - 1}"
        if window:
            s0 = a - window + 1
            exp = _expect(X[s0:b], y[s0:b], window, window, False, 0.0, f64, first=s0)
        else:
            s0 = a
            base += _prefix_base(X[done:a], y[done:a], a - done)
            done = a
            exp = _expect(X[s0:b], y[s0:b], 0, start, False, 0.0, f64, first=s0, base=base)
        ratio = max(ratio, _compare(what, f64, X[s0:b], exp, co[s0:b], pr[s0:b], va[s0:b], rows=np.arange(a - s0, b - s0)))
    if not f64:
        record_property("f32_ratio", ratio)


# ---------------------------------------------------------------------------------------------------------------------
# fill policies through the plugin ABI
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("where", ["x", "y"])
@pytest.mark.parametrize("rolling", [True, False], ids=["rolling", "recursive"])
@pytest.mark.parametrize("f64", [False, True], ids=["f32", "f64"])
def test_fill_policy_through_the_plugin(monkeypatch, record_property, f64, rolling, where):
    """null_policy="0.5" through `pl_rolling_lr[_f32]` / `pl_recursive_lr[_f32]`: null features are filled with 0.5; a null
    target drops its row (rolling: the window skips it; recursive: the row is invalid and, as the oracle restates
    DESIGN.md §5 deviation 2, every kept row pairs with its own coefficients).  Checked against the definition on the
    filled data and against the f64 oracle."""
    import polars_ds_extension_b200 as pds
    import polars_ds_extension_b200.config as cfg
    from polars_ds_extension_b200 import Frame
    from polars_ds_extension_b200._lib import lib
    from tests.backends import OracleBackend, PluginBackend

    n, p, bias, lam = 3001, 4, True, 0.1
    D = p + 1
    window, min_rows, start = 128, 64, 20
    X, y = _data(4000 + 2 * rolling + (where == "y"), n, p, f64, where)
    cols = {f"x{j}": [None if np.isnan(v) else float(v) for v in X[:, j]] for j in range(p)}
    cols["y"] = [None if np.isnan(v) else float(v) for v in y]
    df = Frame(cols)
    xs = [f"x{j}" for j in range(p)]

    def make():
        if rolling:
            return pds.rolling_lin_reg(*xs, target="y", window_size=window, add_bias=bias, l2_reg=lam,
                                       min_valid_rows=min_rows, null_policy="0.5")
        return pds.recursive_lin_reg(*xs, target="y", start_with=start, add_bias=bias, l2_reg=lam, null_policy="0.5")

    monkeypatch.setattr(cfg, "LIN_REG_EXPR_F64", f64)
    g = PluginBackend().eval(df, make())
    route = int(lib().pdsb_last_online_path())
    want = _route(f64, D, window if rolling else 0, where == "y")
    assert route == want, f"pass C ran the {ROUTE_NAME.get(route, route)} kernel, not the {ROUTE_NAME[want]} one"
    monkeypatch.setattr(cfg, "LIN_REG_EXPR_F64", True)
    o = OracleBackend().eval(df, make())

    Xf = np.where(np.isnan(X), 0.5, X)
    if not f64:
        Xf = Xf.astype(np.float32).astype(np.float64)
    Z = _design(Xf, bias)
    skip = where == "y"
    exp = _expect(Z, y, window if rolling else 0, min_rows if rolling else start, skip, lam, f64)
    valid = np.array([c is not None for c in g["coeffs"]])
    co = np.array([c if c is not None else np.zeros(D) for c in g["coeffs"]], np.float64)
    pred = np.where(g["pred"][1], g["pred"][0], 0.0)
    what = f"{'f64' if f64 else 'f32'} {'rolling' if rolling else 'recursive'} nulls in {where}"
    ratio = _compare(what, f64, Z, exp, co, pred, valid)
    if not f64:
        record_property("f32_ratio", ratio)
    # against the f64 oracle (its sequential Woodbury walk drifts a little even in f64)
    ovalid = np.array([c is not None for c in o["coeffs"]])
    assert np.array_equal(valid, ovalid), f"{what}: valid differs from the oracle"
    oco = np.array([c if c is not None else np.zeros(D) for c in o["coeffs"]], np.float64)
    v = np.flatnonzero(valid)
    e = _rel_rows(co[v], oco[v])
    assert e.max() <= (1e-6 if f64 else 1e-4), f"{what}: row {v[np.argmax(e)]}: rel(gpu, oracle f64) {e.max():.3e}"
    ep = np.abs(pred[v] - o["pred"][0][v]) / np.maximum(np.abs(o["pred"][0][v]), 1.0)
    assert ep.max() <= (1e-6 if f64 else 1e-4), f"{what}: row {v[np.argmax(ep)]}: pred differs from the oracle by {ep.max():.3e}"


# ---------------------------------------------------------------------------------------------------------------------
# the tolerances can see the errors this file exists to catch (CPU)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("f64", [False, True], ids=["f32", "f64"])
def test_acceptance_rejects_plausible_kernel_errors(f64):
    """On the seeded data of a rolling skip case (D = 8 with bias, window 1024, null targets, lambda > 0), each of
    these moves the coefficients past the acceptance bound on the checked rows: a window one row longer or shorter; one
    chain-boundary row dropped; lambda left off the bias diagonal; one null row counted (its y taken as 0)."""
    n, D, window, min_rows, lam = 4096, 8, 1024, 512, 0.25
    X, y = _data(2000 + 31 * D + window, n, D - 1, f64, "y", window, min_rows)
    Z = _design(X, True)
    ev, truth, m32, G = _expect(Z, y, window, min_rows, True, lam, f64)
    dt = np.float64 if f64 else np.float32

    def rejected(what, other):
        ov, ot = other[0], other[1]
        both = np.flatnonzero(ev & ov)
        assert both.size > 0
        got = ot[both].astype(dt)                      # what a kernel would return
        ok = _coeffs_ok(f64, got, truth[both], m32[both], G[both])[0]
        assert not ok.all(), f"{what}: every checked row still passes"
        return int((~ok).sum())

    # the unperturbed definition, rounded to the dtype, passes
    ok = _coeffs_ok(f64, truth[ev].astype(dt), truth[ev], m32[ev], G[ev])[0]
    assert ok.all()
    for w in (window - 1, window + 1):
        rejected(f"window {w}", _expect(Z, y, w, min_rows, True, lam, f64))
    r1 = 1024 + int(np.flatnonzero(np.isfinite(y[1024:]))[0])          # the first finite row of chain 1
    assert rejected(f"row {r1} dropped", _expect(Z, y, window, min_rows, True, lam, f64, drop=r1)) >= 500
    rejected("lambda off the bias diagonal", _expect(Z, y, window, min_rows, True, lam, f64, bias_lambda=False))
    r0 = int(np.flatnonzero(np.isnan(y[window:]))[0]) + window
    y0 = y.copy()
    y0[r0] = 0.0
    rejected(f"null row {r0} counted", _expect(Z, y0, window, min_rows, True, lam, f64))
