"""CPU oracles for isotonic_regression (test infrastructure only).

* ``reference_pava``: the reference's loop (src/num_ext/isotonic_regression.rs, itself scipy's PAVA) restated in Python,
  with the symbol's n <= 1 passthrough, its checks and error strings, and the reversal for ``increasing=False``.
* ``pava_ld``: the same loop in ``np.longdouble`` (for n up to ~2e5).
* ``blocks_ld``: scipy's block boundaries with every block mean recomputed in long double (``np.add.reduceat``), for
  larger n.
* ``exact_pava``: PAVA in exact rational arithmetic, for integer data; ``exact_f64`` rounds it correctly to f64.
"""
from __future__ import annotations

from fractions import Fraction

import numpy as np


class IsotonicError(ValueError):
    pass


def _pava(x, w):
    """scipy's PAVA (_pava_pybind.cpp), as the reference ports it: x and w are overwritten by the block means and
    weights, r[b] is where block b starts."""
    n = len(x)
    r = [0] * (n + 1)
    r[1] = 1
    b = 0
    xb_pre, wb_pre = x[0], w[0]
    i = 1
    while i < n:
        b += 1
        xb, wb = x[i], w[i]
        if xb_pre >= xb:
            b -= 1
            sb = wb_pre * xb_pre + wb * xb
            wb += wb_pre
            xb = sb / wb
            while i + 1 < n and xb >= x[i + 1]:
                i += 1
                sb += w[i] * x[i]
                wb += w[i]
                xb = sb / wb
            while b > 0 and x[b - 1] >= xb:
                b -= 1
                sb += w[b] * x[b]
                wb += w[b]
                xb = sb / wb
        xb_pre = xb
        x[b] = xb
        wb_pre = wb
        w[b] = wb
        r[b + 1] = i + 1
        i += 1
    f = n - 1
    for k in range(b, -1, -1):
        t = r[k]
        for j in range(t, f + 1):
            x[j] = x[k]
        if k == 0:
            break
        f = t - 1
    return x


def reference_pava(y, weights=None, increasing=True):
    """pl_isotonic_regression on Python lists / arrays (None = null), f64 arithmetic, the reference's checks in order."""
    y = list(y)
    if len(y) <= 1:
        return y
    if any(v is None for v in y):
        raise IsotonicError("Input should not contain nulls.")
    if weights is not None:
        weights = list(weights)
        if len(weights) != len(y):
            raise IsotonicError("Weights should not contain nulls and must be the same length as y.")
        if any(v is None for v in weights):
            raise IsotonicError("Weight should not contain nulls.")
        if any(float(v) <= 0.0 for v in weights):
            raise IsotonicError("Weight should not contain negative values.")
        w = [np.float64(v) for v in weights]
    else:
        w = [np.float64(1.0)] * len(y)
    x = [np.float64(v) for v in y]
    if not increasing:
        x.reverse()
        w.reverse()
    with np.errstate(invalid="ignore", over="ignore"):
        out = np.array(_pava(x, w), dtype=np.float64)
    return out if increasing else out[::-1].copy()


def pava_ld(y, weights=None, increasing=True):
    """The same loop in long double; returns f64 values of the long-double solution."""
    y = np.asarray(y, dtype=np.float64)
    x = [np.longdouble(v) for v in (y if increasing else y[::-1])]
    wa = np.ones(len(y)) if weights is None else np.asarray(weights, dtype=np.float64)
    w = [np.longdouble(v) for v in (wa if increasing else wa[::-1])]
    out = np.array(_pava(x, w), dtype=np.longdouble)
    return out if increasing else out[::-1].copy()


def blocks_ld(y, weights=None, increasing=True):
    """scipy's blocks, each mean recomputed as sum(w y) / sum(w) in long double (for n where pava_ld is too slow)."""
    from scipy.optimize import isotonic_regression

    y = np.asarray(y, dtype=np.float64)
    res = isotonic_regression(y, weights=weights, increasing=increasing)
    starts = np.asarray(res.blocks[:-1], dtype=np.int64)
    yl = y.astype(np.longdouble)
    wl = np.ones(len(y), dtype=np.longdouble) if weights is None else np.asarray(weights).astype(np.longdouble)
    means = np.add.reduceat(wl * yl, starts) / np.add.reduceat(wl, starts)
    return np.repeat(means, np.diff(np.asarray(res.blocks, dtype=np.int64)))


def exact_pava(y, weights=None, increasing=True):
    """PAVA in exact rationals (integer y and w); a list of Fractions."""
    ys = [Fraction(int(v)) for v in y]
    ws = [Fraction(1)] * len(ys) if weights is None else [Fraction(int(v)) for v in weights]
    if not increasing:
        ys = [-v for v in ys]
    S, W, E = [], [], []
    for i, (v, wv) in enumerate(zip(ys, ws)):
        s, ww = v * wv, wv
        while S and S[-1] / W[-1] >= s / ww:
            s += S.pop()
            ww += W.pop()
            E.pop()
        S.append(s)
        W.append(ww)
        E.append(i + 1)
    out, lo = [], 0
    for s, ww, e in zip(S, W, E):
        out.extend([s / ww] * (e - lo))
        lo = e
    return out if increasing else [-v for v in out]


def exact_f64(y, weights=None, increasing=True):
    """The exact solution correctly rounded to f64."""
    return np.array([float(v) for v in exact_pava(y, weights, increasing)], dtype=np.float64)


def rel_err(g, ref, y):
    """max |g - ref| / max |y| (ref may be long double)."""
    d = np.abs(np.asarray(g, dtype=np.longdouble) - np.asarray(ref, dtype=np.longdouble))
    return float(np.max(d) / max(np.max(np.abs(np.asarray(y, dtype=np.float64))), 1e-300))


def shape(kind, n, seed):
    """Test columns: random walk, noisy upward trend, strictly increasing, strictly decreasing, increasing with a final
    huge drop (every block pooled), sawtooth (one violation per 32 rows), long constant runs."""
    rng = np.random.default_rng(seed)
    i = np.arange(n, dtype=np.float64)
    if kind == "walk":
        return np.cumsum(rng.standard_normal(n))
    if kind == "trend":
        return i * (4.0 / n) + rng.standard_normal(n)
    if kind == "increasing":
        return i + rng.uniform(0.0, 0.5, n)
    if kind == "decreasing":
        return -i - rng.uniform(0.0, 0.5, n)
    if kind == "drop":
        y = i + rng.uniform(0.0, 0.5, n)
        y[-1] = -float(n) * n                      # below minus the sum of the rest: one block
        return y
    if kind == "sawtooth":
        return (i % 32) + 16.0 * (i // 32) + 0.05 * rng.standard_normal(n)
    if kind == "runs":
        return np.repeat(rng.integers(-3, 4, n // 1000 + 1), 1000)[:n].astype(np.float64)
    raise ValueError(kind)


SHAPES = ["walk", "trend", "increasing", "decreasing", "drop", "sawtooth", "runs"]
