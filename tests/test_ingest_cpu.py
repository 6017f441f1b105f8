"""The oracle's frame builder pinned to the reference's ingest rules (no GPU needed):

  * f32 FILL casts every feature straight to Float32 and fills with the f32-parsed literal (linear_regression_f32.rs:
    148-152, :169-173, :256-258); f64 FILL casts to Float64 and fills with the f64 literal (linear_regression.rs:211-213);
  * the policy parser rounds the fill literal once to the compute dtype (src/linear/mod.rs:56, `str::parse::<T>`);
  * the plain-numpy expected frame of tests/test_gpu_ingest.py and the oracle's series_to_mat_for_lr /
    series_to_mat_for_multi_lr agree on the same generated inputs, so the two statements of the rule cannot drift.
"""
from fractions import Fraction

import numpy as np
import pytest

from oracle import lin_reg_oracle as orc
from tests import test_gpu_ingest as ingest

BIG = np.array(ingest.DOUBLE_ROUNDING + [-v for v in ingest.DOUBLE_ROUNDING] + [3, -7], dtype=np.int64)
UBIG = np.array(ingest.DOUBLE_ROUNDING + [2**63 + 2**39 + 1, 2**64 - 1, 5], dtype=np.uint64)


def _f32_exact(text: str) -> np.float32:
    """The f32 nearest to the decimal `text` (ties to even), by exact comparison with every f32 near it."""
    x = Fraction(text)
    # every finite f32 is m * 2^e with |m| < 2^24 and e >= -149; +-2^128 stands for +-inf
    e = max(-149, (abs(x).numerator.bit_length() - abs(x).denominator.bit_length()) - 24) if x else -149
    best = None
    for k in range(e - 2, e + 3):
        q = Fraction(2) ** k
        for m in (int(x / q) - 1, int(x / q), int(x / q) + 1):
            v = m * q
            if abs(m) >= 2**24 and abs(v) != 2**128:
                continue
            key = (abs(v - x), m & 1 if abs(v) < 2**128 else 0)
            if best is None or key < best[0]:
                best = (key, v)
    v = best[1]
    return np.float32(np.inf if v >= 2**128 else -np.inf if v <= -(2**128) else float(v))


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint32 if a.dtype == np.float32 else np.uint64)


@pytest.mark.parametrize("vals", [BIG, UBIG], ids=["i64", "u64"])
def test_f32_fill_casts_integers_straight_to_f32(vals):
    valid = np.ones(len(vals), bool)
    valid[-1] = False
    y = orc.Col("y", np.arange(len(vals), dtype=np.float64))
    _, X, mask = orc.series_to_mat_for_lr([y, orc.Col("x", vals, valid)], False, orc.parse_null_policy("one"),
                                          np.float32)
    want = vals.astype(np.float32)
    want[-1] = 1.0
    assert mask is None
    assert np.array_equal(_bits(X[:, 0]), _bits(want))
    assert not np.array_equal(_bits(X[:-1, 0]), _bits(vals[:-1].astype(np.float64).astype(np.float32)))


@pytest.mark.parametrize("vals", [BIG, UBIG], ids=["i64", "u64"])
def test_f64_fill_keeps_the_cast_through_f64(vals):
    valid = np.ones(len(vals), bool)
    valid[0] = False
    y = orc.Col("y", np.arange(len(vals), dtype=np.float64))
    _, X, _ = orc.series_to_mat_for_lr([y, orc.Col("x", vals, valid)], False, orc.parse_null_policy("-2.5"), np.float64)
    want = vals.astype(np.float64)
    want[0] = -2.5
    assert np.array_equal(_bits(X[:, 0]), _bits(want))


PARSE_CASES = [ingest.MIDPOINT, "0.1", "-2.5", "1e-46", "7e-46", "-1.4e-45", "3.4028235677973366e38",
               "3.40282357e38", "1e39", "16777217", "16777219", "0.333333333333333333333333", "1.00000017881393432617187",
               "-0.0", "1E2"]


@pytest.mark.parametrize("text", PARSE_CASES)
def test_policy_parser_rounds_the_fill_once(text):
    kind, fill = orc.parse_null_policy(text)
    assert kind == "fill"
    got32 = orc.fill_value(fill, np.float32)
    want32 = ingest.round_fill(text, np.float32)
    assert np.array_equal(_bits(np.float32(got32)), _bits(_f32_exact(text))), (text, got32)
    assert np.array_equal(_bits(np.float32(want32)), _bits(_f32_exact(text))), (text, want32)
    assert orc.fill_value(fill, np.float64) == float(text)


def test_midpoint_fill_differs_from_rounding_through_double():
    """The string whose f32 rounding through double ties to 1.0: correct rounding gives 1 + 2^-23."""
    assert np.float32(float(ingest.MIDPOINT)) == np.float32(1.0)
    assert _f32_exact(ingest.MIDPOINT) == np.float32(1 + 2**-23)
    assert orc.fill_value(orc.parse_null_policy(ingest.MIDPOINT)[1], np.float32) == np.float32(1 + 2**-23)


def test_multi_target_fill_uses_the_f32_literal():
    n = 12
    x = orc.Col("x", BIG[:n] if len(BIG) >= n else np.resize(BIG, n), np.arange(n) % 4 != 0)
    ys = [orc.Col("a", np.ones(n)), orc.Col("b", np.zeros(n))]
    _, X = orc.series_to_mat_for_multi_lr(ys + [x], 2, False, orc.parse_null_policy(ingest.MIDPOINT), np.float32)
    want = x.values.astype(np.float32)
    want[~x.valid] = np.float32(1 + 2**-23)
    assert np.array_equal(_bits(X[:, 0]), _bits(want))


def test_invalid_policy_string():
    with pytest.raises(orc.OracleError, match="Invalid NullPolicy."):
        orc.parse_null_policy("not_a_policy")


# ---------------------------------------------------------------------------------------------------------------
# the expected frame of the GPU test == the oracle's frame builder
# ---------------------------------------------------------------------------------------------------------------
def _oracle_frame(cols, n_targets, text, dt, multi, online):
    """The oracle's frame in build_frame's shape: (Z [n_cols, n], row mask or None); rows the oracle filters out are
    all-zero rows with mask 0 here.  OracleError -> ingest.Expected."""
    inputs = [orc.Col(f"c{i}", v, None if m is None else m) for i, (v, m) in enumerate(cols)]
    n = len(cols[0][0])
    try:
        kind, fill = orc.parse_null_policy(text)
        if multi:
            Y, X = orc.series_to_mat_for_multi_lr(inputs, n_targets, False, (kind, fill), dt)
            return np.vstack([Y.T, X.T]), None
        if online:     # pl_rolling_lr's renaming (linear_regression.rs:1214-1219), then no row is ever dropped
            kind = {"skip": "skip_window", "fill": "fill_window"}.get(kind, kind)
        y, X, mask = orc.series_to_mat_for_lr(inputs, False, (kind, fill), dt)
    except orc.OracleError as e:
        raise ingest.Expected(str(e))
    Zk = np.vstack([y[None, :], X.T])
    if not isinstance(mask, np.ndarray):
        return Zk, None
    Z = np.zeros((Zk.shape[0], n), dt)
    Z[:, mask] = Zk
    return Z, mask.astype(dt)


def _assert_same(a, b, what):
    a, b = np.asarray(a), np.asarray(b, dtype=np.asarray(a).dtype)
    assert a.shape == b.shape, what
    an, bn = np.isnan(a), np.isnan(b)
    assert np.array_equal(an, bn), what
    assert np.array_equal(_bits(np.where(an, 0, a)), _bits(np.where(bn, 0, b))), what


@pytest.mark.parametrize("dt", [np.float32, np.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("src", list(ingest.SOURCES))
def test_expected_frame_agrees_with_the_oracle(src, dt):
    n = 61
    rng = np.random.default_rng(len(src) * 7 + (dt == np.float32))
    x = ingest.source_values(src, n, rng)
    y = rng.standard_normal(n)
    x2 = rng.integers(-1000, 1000, n).astype(np.int32)
    placements = {"none": (None, None), "feature": (None, rng.random(n) > 0.2), "target": (rng.random(n) > 0.2, None),
                  "both": (rng.random(n) > 0.2, rng.random(n) > 0.2), "column": (None, np.zeros(n, bool))}
    for place, (yv, xv) in placements.items():
        for multi, online, nt in ((False, False, 1), (False, True, 1), (True, False, 2)):
            cols = [(y, yv), (x, xv), (x2, None)]
            if multi:
                cols = [(y, None), (x2.astype(np.float64), yv), (x, xv)]
            for text in ingest.POLICIES:
                what = f"{src} {place} multi={multi} online={online} {text!r}"
                try:
                    Z, mask, _ = ingest.expected_frame(cols, nt, text, dt, multi=multi, online=online)
                except ingest.Expected as e:
                    with pytest.raises(ingest.Expected) as ei:
                        _oracle_frame(cols, nt, text, dt, multi, online)
                    assert str(ei.value) == str(e), what
                    continue
                try:
                    oZ, omask = _oracle_frame(cols, nt, text, dt, multi, online)
                except ingest.Expected as e:
                    # the oracle's frame builder also holds the fits' row-count check; the frame itself is all-masked
                    assert str(e).startswith("#Data < #features") and mask is not None and mask.sum() < len(cols) - nt
                    continue
                _assert_same(Z, oZ, what)
                assert (mask is None) == (omask is None), what
                if mask is not None:
                    _assert_same(mask, omask, what)
