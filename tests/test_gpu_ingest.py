"""The Arrow ingest path, bit for bit: ``build_frame`` (csrc/host/lr_host.cc) with the K1 kernels (k1_pack.cu) and the
staging ring (h2d.cc), for every source dtype, slice offset, chunk split, null placement and null policy, against a
frame written out below in plain numpy; then the fits that start from it, end to end through the plugin symbols.

The expected frame states the reference's rule (paths relative to the polars_ds sources):

  * every value is cast once to the compute dtype dt: ``series_to_slice_inner`` (src/utils/mod.rs:140-144) and the
    fill branches' ``cast(Float64)`` / ``cast(Float32)`` (src/num_ext/linear_regression.rs:211-213,
    linear_regression_f32.rs:148-152) convert the source value straight to dt, one rounding;
  * the fill literal is ``str::parse::<T>`` of the policy string (src/linear/mod.rs:43-60): NullPolicy<f64> for the f64
    symbols, NullPolicy<f32> for the _f32 twins, rounded once to dt;
  * ``skip`` drops every row with a null in any column (linear_regression.rs:199-206): here the row is kept, all-zero,
    with mask 0; ``zero`` / ``one`` / a number fill the features and a null target drops the row (:207-231); ``ignore``
    keeps nulls as NaN (:194-197); ``raise`` is "Nulls found in data" (:198);
  * multi-target (series_to_mat_for_multi_lr, :301-332): raise, any other policy than a fill, and a null target are
    errors; a fill fills the features;
  * rolling / recursive (online): no row is dropped, nulls stay NaN or take the fill, no mask;
  * weights: nulls become NaN and take no part in the row mask.

Rows n..ld of the device frame are padding and are not compared.
"""
from fractions import Fraction

import numpy as np
import pyarrow as pa
import pytest

pytestmark = pytest.mark.gpu

MIDPOINT = "1.000000059604644775390625000000001"        # 1 + 2^-24 (the f32 midpoint above 1) plus a little
POLICIES = ["skip", "zero", "one", "0.1", "-2.5", MIDPOINT, "ignore", "raise", "not_a_policy"]
FILLS = ["zero", "one", "0.1", "-2.5", MIDPOINT]

SOURCES = {
    "i8": (np.int8, pa.int8()), "u8": (np.uint8, pa.uint8()), "i16": (np.int16, pa.int16()),
    "u16": (np.uint16, pa.uint16()), "i32": (np.int32, pa.int32()), "u32": (np.uint32, pa.uint32()),
    "i64": (np.int64, pa.int64()), "u64": (np.uint64, pa.uint64()), "bool": (np.bool_, pa.bool_()),
    "f32": (np.float32, pa.float32()), "f64": (np.float64, pa.float64()),
}

# integers whose conversion to f32 through f64 rounds twice (2^60 + 2^36 + 1 -> 1.1529215e18 instead of 1.1529216e18)
DOUBLE_ROUNDING = [2**60 + 2**36 + 1, 2**62 + 2**38 + 1]
EXTREMES = {
    "i64": [np.iinfo(np.int64).min, np.iinfo(np.int64).max, 0, -1, 1, 2**53 + 1, -(2**53 + 1)]
    + DOUBLE_ROUNDING + [-v for v in DOUBLE_ROUNDING],
    "u64": [0, np.iinfo(np.uint64).max, 2**63 + 2**39 + 1, 2**53 + 1] + DOUBLE_ROUNDING,
    "f32": [np.inf, -np.inf, -0.0, np.nan, 1e-45, 3.4028235e38, -1.1754942e-38],
    # 1 + 2^-24 ties to 1.0 in f32, one bit above it rounds up; 1e300 overflows f32; -1e-310 is an f64 subnormal
    "f64": [1 + 2**-24, 1 + 2**-24 + 2**-52, 1e300, -1e300, -1e-310, np.nan, -0.0, np.inf, 2**-149 * 1.5],
}
N_EXTREMES = 12          # rows that never get a null, so every extreme value reaches the kernel


class Expected(Exception):
    """The error the reference raises for this input (its message is compared with the library's)."""


# ---------------------------------------------------------------------------------------------------------------
# Inputs
# ---------------------------------------------------------------------------------------------------------------
def source_values(kind: str, n: int, rng) -> np.ndarray:
    """n values of the source dtype over its whole range, with the kind's extremes in the first rows."""
    npt = SOURCES[kind][0]
    if kind == "bool":
        v = rng.random(n) < 0.5
        v[:4] = [True, False, True, True]
        return v
    if kind in ("f32", "f64"):
        v = (rng.standard_normal(n) * np.exp(rng.uniform(-20, 20, n))).astype(npt)
    else:
        info = np.iinfo(npt)
        v = rng.integers(info.min, info.max, n, dtype=npt, endpoint=True)
        v[:2] = [info.min, info.max]
    ext = EXTREMES.get(kind, [])
    v[:len(ext)] = np.array(ext, dtype=npt)
    return v


def make_column(values: np.ndarray, arrow_type, valid=None, cuts=(), offset: int = 0, bitmap: bool = False,
                seed: int = 0) -> pa.ChunkedArray:
    """A chunked Arrow column holding `values` (nulls where `valid` is False): one array with `offset` leading junk rows
    taken off with ``.slice(offset)`` (so ArrowArray.offset = offset), cut into chunks at the row indices `cuts`
    (repeated cuts give empty chunks).  bitmap: a validity buffer even when `valid` is None (a null in the junk head;
    needs offset >= 1)."""
    rng = np.random.default_rng(seed)
    n = len(values)
    head = values[rng.integers(0, max(n, 1), offset)] if n else np.zeros(offset, values.dtype)
    full = np.concatenate([head, values])
    full_valid = np.concatenate([rng.random(offset) < 0.5, np.ones(n, bool) if valid is None else valid])
    if valid is None and not bitmap:
        full_valid[:offset] = True
    if bitmap and offset:
        full_valid[0] = False
    arr = pa.array(full, type=arrow_type, mask=None if full_valid.all() else ~full_valid).slice(offset)
    edges = [0, *cuts, n]
    return pa.chunked_array([arr.slice(a, b - a) for a, b in zip(edges[:-1], edges[1:])], type=arrow_type)


# ---------------------------------------------------------------------------------------------------------------
# The expected frame
# ---------------------------------------------------------------------------------------------------------------
def round_fill(text: str, dt):
    """str::parse::<T> (src/linear/mod.rs:56): the decimal `text` rounded once, to nearest-even, to dt.  The exact value is
    a Fraction; of the nearest dt value to the double's rounding and its two neighbours, the closest wins."""
    x = Fraction(text)
    if dt == np.float64:
        return np.float64(float(x))                 # int / int true division: correctly rounded
    with np.errstate(over="ignore"):
        c = np.float32(float(x))
    cands = [c, np.nextafter(c, np.float32(-np.inf)), np.nextafter(c, np.float32(np.inf))]
    return min(cands, key=lambda v: (abs(_exact_f32(v) - x), int(np.array(v).view(np.uint32)) & 1))


def _exact_f32(v) -> Fraction:
    """The value of an f32 as a Fraction, +-inf standing at +-2^128 (where round-to-nearest puts the overflow)."""
    return Fraction(float(v)) if np.isfinite(v) else Fraction(2**128) * (1 if v > 0 else -1)


def parse_policy(text: str, dt):
    t = text.lower()
    if t in ("raise", "skip", "ignore", "skip_window"):
        return t, None
    if t in ("zero", "one"):
        return "fill", dt(t == "one")
    try:
        return "fill", round_fill(text, dt)
    except ValueError:
        raise Expected("Invalid NullPolicy.")


def expected_frame(cols, n_targets: int, text: str, dt, multi: bool = False, online: bool = False, weights=None):
    """cols: [(values, valid or None)] targets first.  -> (Z [n_cols, n] dt, mask [n] dt or None, w [n] dt or None), or
    raises Expected with the reference's message."""
    kind, fill = parse_policy(text, dt)
    n = len(cols[0][0])
    null = [np.zeros(n, bool) if v is None else ~np.asarray(v, bool) for _, v in cols]
    y_null = any(null[c].any() for c in range(n_targets))
    x_null = any(null[c].any() for c in range(n_targets, len(cols)))
    Z = [np.asarray(v).astype(dt) for v, _ in cols]            # one rounding from the source value
    mask = None
    if y_null or x_null:
        if multi:
            if kind == "raise":
                raise Expected("Nulls found in data")
            if kind != "fill":
                raise Expected("The null policy is not supported by multi-target linear regression.")
            if y_null:
                raise Expected("Filling null doesn't work for multi-target lstsq when there are nulls in any of the "
                               "targets.")
        elif kind == "raise":
            raise Expected("Nulls found in data")
        if kind == "skip" and not online:
            mask = ~np.any(null, axis=0)
        else:
            for c in range(len(cols)):
                # a fill fills the features; everything else keeps the null as NaN (ignore, online skip, a null target)
                Z[c][null[c]] = fill if kind == "fill" and c >= n_targets else np.nan
            if kind == "fill" and y_null and not online and not multi:
                mask = ~null[0]
    if mask is not None:
        for c in range(len(cols)):
            Z[c][~mask] = 0
        mask = mask.astype(dt)
    w = None
    if weights is not None:
        w = np.asarray(weights[0]).astype(dt)
        if weights[1] is not None:
            w[~np.asarray(weights[1], bool)] = np.nan
    return np.stack(Z), mask, w


def assert_bits(got, exp, what: str):
    """Bit-for-bit equality (NaN positions equal, NaN payloads not compared); prints the differing bit patterns."""
    got = np.ascontiguousarray(got)
    exp = np.ascontiguousarray(exp, dtype=got.dtype)
    assert got.shape == exp.shape, (what, got.shape, exp.shape)
    ui = np.uint32 if got.dtype == np.float32 else np.uint64
    gn, en = np.isnan(got), np.isnan(exp)
    bad = (gn != en) | (~gn & ~en & (got.view(ui) != exp.view(ui)))
    if bad.any():
        w = 2 * got.itemsize
        lines = [f"  {i}: got {got[i]!r} (0x{int(got.view(ui)[i]):0{w}x}), expected {exp[i]!r} (0x{int(exp.view(ui)[i]):0{w}x})"
                 for i in (tuple(int(k) for k in r) for r in np.argwhere(bad)[:8])]
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.size} entries differ\n" + "\n".join(lines))


def device_frame(arrays, n_targets: int, text: str, dt, **kw):
    import torch

    from polars_ds_extension_b200 import device
    from polars_ds_extension_b200._lib import PdsbError

    tdt = torch.float32 if dt == np.float32 else torch.float64
    try:
        n, Z, mask, w = device.build_frame(arrays, n_targets, text, tdt, **kw)
    except PdsbError as e:
        return str(e)
    torch.cuda.synchronize()
    return (Z[:, :n].cpu().numpy(), None if mask is None else mask[:n].cpu().numpy(),
            None if w is None else w[:n].cpu().numpy())


def check_frame(arrays, cols, n_targets, text, dt, what, multi=False, online=False, weights=None, **kw):
    """build_frame on `arrays` vs expected_frame on `cols` (the same data as numpy)."""
    got = device_frame(arrays, n_targets, text, dt, multi=multi, online=online,
                       weights=None if weights is None else weights[0], **kw)
    try:
        Z, mask, w = expected_frame(cols, n_targets, text, dt, multi=multi, online=online,
                                    weights=None if weights is None else weights[1])
    except Expected as e:
        assert got == str(e), f"{what}: expected the error {str(e)!r}, got {got if isinstance(got, str) else 'a frame'}"
        return
    assert not isinstance(got, str), f"{what}: unexpected error {got!r}"
    gZ, gmask, gw = got
    assert_bits(gZ, Z, f"{what} Z")
    assert (gmask is None) == (mask is None), f"{what}: row mask {'missing' if mask is not None else 'unexpected'}"
    if mask is not None:
        assert_bits(gmask, mask, f"{what} mask")
    if w is not None:
        assert_bits(gw, w, f"{what} w")


# ---------------------------------------------------------------------------------------------------------------
# build_frame, bit for bit
# ---------------------------------------------------------------------------------------------------------------
PLACEMENTS = ["none", "bitmap", "feature", "target", "both", "column"]


def _null_rows(rng, n, rate=0.2):
    v = rng.random(n) >= rate
    v[:N_EXTREMES] = True
    return v


@pytest.mark.parametrize("dt", [np.float32, np.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("src", list(SOURCES))
def test_build_frame_casts_each_source_dtype_once(src, dt):
    """[y f64 | x src | x2 i32] at slice offsets 0..9 (bit offsets 0..7 and a byte-crossing head), x cut into chunks at
    rows that are not multiples of 8 with an empty and a 1-row chunk, nulls nowhere / in x / in y / in both / a whole x
    column, under every policy; odd offsets give x's null count as unknown (-1, recounted from the bitmaps)."""
    n = 203
    rng = np.random.default_rng(abs(hash(src)) % 2**32)
    x = source_values(src, n, rng)
    y = rng.standard_normal(n)
    x2 = rng.integers(-2**31, 2**31 - 1, n, dtype=np.int32)
    for off in range(10):
        for place in PLACEMENTS:
            if place == "bitmap" and off == 0:
                continue
            xv = _null_rows(rng, n) if place in ("feature", "both") else None
            if place == "column":
                xv = np.zeros(n, bool)
            yv = _null_rows(rng, n, 0.1) if place in ("target", "both") else None
            x2v = _null_rows(rng, n, 0.05) if place == "both" else None
            arrays = [make_column(y, pa.float64(), yv, (64,), (off + 3) % 10, place == "bitmap", seed=off),
                      make_column(x, SOURCES[src][1], xv, (13 + off, 13 + off, 14 + off, 101), off, place == "bitmap",
                                  seed=off + 1),
                      make_column(x2, pa.int32(), x2v, (), 9 - off, seed=off + 2)]
            cols = [(y, yv), (x, xv), (x2, x2v)]
            ncs = [None, -1 if off % 2 else None, None]
            for pol in POLICIES:
                check_frame(arrays, cols, 1, pol, dt, f"{src} off={off} {place} {pol!r}", null_counts=ncs)


def test_int64_and_uint64_to_f32_round_once():
    """The three double-rounding integers and their negatives, alone: the direct conversion (cvt.rn.f32.s64 / .u64)."""
    i = np.array(DOUBLE_ROUNDING + [2**63 - 2**39 - 1] + [-v for v in DOUBLE_ROUNDING], dtype=np.int64)
    u = np.array(DOUBLE_ROUNDING + [2**63 + 2**39 + 1, 2**64 - 2**39 - 1], dtype=np.uint64)
    for vals, t in ((i, pa.int64()), (u, pa.uint64())):
        y = np.arange(len(vals), dtype=np.float32)
        got = device_frame([pa.chunked_array([pa.array(y)]), pa.chunked_array([pa.array(vals, type=t)])], 1, "skip",
                           np.float32)
        assert_bits(got[0][1], vals.astype(np.float32), f"{t} -> f32")
        assert not np.array_equal(vals.astype(np.float32), vals.astype(np.float64).astype(np.float32))


@pytest.mark.parametrize("dt", [np.float32, np.float64], ids=["f32", "f64"])
def test_fill_literal_rounds_once(dt):
    """The fill string parsed as NullPolicy<T>: the midpoint string is 1 + 2^-23 in f32 (strtod then a cast to float
    lands on the midpoint and ties to 1.0)."""
    n = 40
    x = np.arange(n, dtype=np.int16)
    xv = np.arange(n) % 3 != 1
    y = np.ones(n)
    arrays = [pa.chunked_array([pa.array(y)]), make_column(x, pa.int16(), xv, (), 5)]
    got = device_frame(arrays, 1, MIDPOINT, dt)
    want = np.float32(1 + 2**-23) if dt == np.float32 else np.float64(1.0000000596046448)
    assert_bits(got[0][1][~xv], np.full((~xv).sum(), want, dt), f"fill {MIDPOINT}")


@pytest.mark.parametrize("dt", [np.float32, np.float64], ids=["f32", "f64"])
def test_build_frame_multi_target(dt):
    """multi=True: the three error texts of series_to_mat_for_multi_lr and FILL on the features (two targets)."""
    n = 150
    rng = np.random.default_rng(3)
    y1, y2 = rng.standard_normal(n), rng.standard_normal(n).astype(np.float32)
    x1, x2 = source_values("i64", n, rng), source_values("u16", n, rng)
    for off in (0, 3, 7):
        for place in ("none", "feature", "target", "both"):
            x1v = _null_rows(rng, n) if place in ("feature", "both") else None
            y2v = _null_rows(rng, n) if place in ("target", "both") else None
            arrays = [make_column(y1, pa.float64(), None, (), off), make_column(y2, pa.float32(), y2v, (77,), off + 1),
                      make_column(x1, pa.int64(), x1v, (9, 9, 10), off + 2), make_column(x2, pa.uint16(), None, (), off)]
            cols = [(y1, None), (y2, y2v), (x1, x1v), (x2, None)]
            for pol in POLICIES:
                check_frame(arrays, cols, 2, pol, dt, f"multi off={off} {place} {pol!r}", multi=True)


@pytest.mark.parametrize("dt", [np.float32, np.float64], ids=["f32", "f64"])
def test_build_frame_online(dt):
    """online=True (rolling / recursive): nulls stay NaN or take the fill, and no row mask."""
    n = 97
    rng = np.random.default_rng(4)
    y = rng.standard_normal(n).astype(np.float32)
    x1, x2 = source_values("i16", n, rng), source_values("u32", n, rng)
    for off in (1, 6):
        for place in ("feature", "target", "both"):
            x1v = _null_rows(rng, n) if place in ("feature", "both") else None
            yv = _null_rows(rng, n) if place in ("target", "both") else None
            arrays = [make_column(y, pa.float32(), yv, (50,), off), make_column(x1, pa.int16(), x1v, (3,), off + 2),
                      make_column(x2, pa.uint32(), None, (), off)]
            cols = [(y, yv), (x1, x1v), (x2, None)]
            for pol in ("skip", "ignore", "raise") + tuple(FILLS):
                check_frame(arrays, cols, 1, pol, dt, f"online off={off} {place} {pol!r}", online=True)


@pytest.mark.parametrize("dt", [np.float32, np.float64], ids=["f32", "f64"])
def test_build_frame_weights(dt):
    """Weights: cast once, nulls NaN, not part of the row mask (which comes from the data alone)."""
    n = 130
    rng = np.random.default_rng(5)
    y, x = rng.standard_normal(n), source_values("u8", n, rng)
    xv = _null_rows(rng, n)
    for wsrc in ("f32", "f64", "i32"):
        wv_ = source_values(wsrc, n, rng) if wsrc == "i32" else rng.uniform(0.1, 2.0, n).astype(SOURCES[wsrc][0])
        wvalid = _null_rows(rng, n, 0.1)
        warr = make_column(wv_, SOURCES[wsrc][1], wvalid, (33,), 5)
        arrays = [make_column(y, pa.float64(), None, (), 2), make_column(x, pa.uint8(), xv, (8, 17), 3)]
        for pol in ("skip", "zero", "ignore"):
            check_frame(arrays, [(y, None), (x, xv)], 1, pol, dt, f"weights {wsrc} {pol}", weights=(warr, (wv_, wvalid)))


def test_build_frame_shape_errors():
    a = pa.chunked_array([pa.array(np.ones(5))])
    assert device_frame([a], 1, "skip", np.float64) == "Data is empty"
    assert device_frame([a, pa.chunked_array([pa.array(np.ones(4))])], 1, "skip", np.float64) == \
        "Seires don't have the same length."
    e = pa.chunked_array([pa.array(np.ones(0))])
    assert device_frame([e, e], 1, "skip", np.float64) == "Empty data"


def test_staged_ingest_matches_expected_and_pinned():
    """Raw (non-matching dtype) columns of >= 1 MiB from pageable memory go through the pinned staging ring and then
    pack_kernel: a 3 000 017-row int32 feature and a u8 feature with nulls at bit offset 3.  The frame is the expected
    frame bit for bit, and a pl_lr_pred_f32 call on them is bit-identical to the same call on page-locked copies."""
    import torch

    from polars_ds_extension_b200 import _harness
    from polars_ds_extension_b200._lib import lib

    n = 3_000_017
    rng = np.random.default_rng(11)
    xi = rng.integers(-1000, 1000, n, dtype=np.int32)
    xu = rng.integers(0, 256, n, dtype=np.uint8)
    xuv = rng.random(n) >= 0.01
    y = (0.002 * xi - 0.01 * xu + rng.standard_normal(n)).astype(np.float32)
    arrays = [make_column(y, pa.float32()), make_column(xi, pa.int32(), offset=6),
              make_column(xu, pa.uint8(), xuv, offset=3)]
    assert arrays[2].chunks[0].offset == 3
    cols = [(y, None), (xi, None), (xu, xuv)]
    for pinned in (False, True):
        got = device_frame(arrays, 1, "skip", np.float32, pinned=pinned)
        staged = lib().pdsb_last_staged_bytes()
        assert staged == (0 if pinned else n * (4 + 4 + 1)), (pinned, staged)
        Z, mask, _ = expected_frame(cols, 1, "skip", np.float32)
        assert_bits(got[0], Z, f"staged Z (pinned={pinned})")
        assert_bits(got[1], mask, f"staged mask (pinned={pinned})")
    kw = {"bias": True, "null_policy": "skip", "l1_reg": 0.0, "l2_reg": 0.0, "solver": "qr", "tol": 1e-5, "max_iter": 200,
          "weighted": False, "positive": False, "singular_x_tol": 1e-6}
    names = ["y", "xi", "xu"]
    a = _harness.call_plugin("pl_lr_pred_f32", arrays, names, kw)
    assert lib().pdsb_last_staged_bytes() == n * (4 + 4 + 1)

    def pinned_copy(ch):
        page_locked = lambda b: torch.from_numpy(np.frombuffer(b, np.uint8).copy()).pin_memory().numpy()  # noqa: E731
        bufs = [None if b is None else pa.py_buffer(page_locked(b)) for b in ch.buffers()]
        return pa.Array.from_buffers(ch.type, len(ch), bufs, null_count=ch.null_count, offset=ch.offset)

    pinned = [pa.chunked_array([pinned_copy(c) for c in a_.chunks]) for a_ in arrays]
    b = _harness.call_plugin("pl_lr_pred_f32", pinned, names, kw)
    assert lib().pdsb_last_staged_bytes() == 0
    assert a.field("pred").equals(b.field("pred")) and a.field("resid").equals(b.field("resid"))
    assert a.field("pred").null_count == int((~xuv).sum())


# ---------------------------------------------------------------------------------------------------------------
# End to end through the plugin symbols
# ---------------------------------------------------------------------------------------------------------------
ORDER = list(SOURCES)
SMALL = {"i8": (-3, 4), "u8": (0, 6), "i16": (-4, 5), "u16": (0, 8), "i32": (-3, 4), "u32": (0, 6), "i64": (-4, 5),
         "u64": (0, 8)}           # unit-scale integers: X'X stays well conditioned in f32


def e2e_frame(seed: int, n: int, p: int, x_nulls: bool = True, y_nulls: bool = True, kinds=None, y_kind=None):
    """Frame of p features of mixed source dtypes (ORDER cycled, or `kinds`), every one at its own slice offset and chunk
    split, nulls (1 %) in every third feature and in y; values exactly representable in f32 so that the f64 oracle on the
    same frame is the truth of the f32 problem.  -> (Frame, feature names, y validity or None, row-valid of the features)"""
    from polars_ds_extension_b200 import Frame

    rng = np.random.default_rng(seed)
    kinds = kinds or [ORDER[j % len(ORDER)] for j in range(p)]
    cols, X, fvalid = {}, np.zeros((n, p)), np.ones(n, bool)
    for j, k in enumerate(kinds):
        npt, at = SOURCES[k]
        if k == "bool":
            v = rng.random(n) < 0.1
        elif k in ("f32", "f64"):
            v = rng.standard_normal(n).astype(np.float32).astype(npt)
        else:
            v = rng.integers(*SMALL[k], n).astype(npt)
            if k[0] == "u":             # sparse: a small mean against the spread
                v[rng.random(n) >= 0.2] = 0
        valid = (rng.random(n) >= 0.01) if (x_nulls and j % 3 == 0) else None
        if valid is not None:
            fvalid &= valid
        cuts = (n // 3 + j % 7, n // 3 + j % 7, 2 * n // 3 + 1) if j % 2 else (n // 2 - j % 5,)
        cols[f"x{j}"] = make_column(v, at, valid, cuts, (j * 3) % 10, seed=seed + j)
        X[:, j] = v.astype(np.float64)
    beta = ((np.arange(p) % 7) - 3) / 4.0 / np.maximum(np.abs(X).max(axis=0), 1)
    y = (X @ beta + 0.5 + 0.01 * rng.standard_normal(n)).astype(np.float32)
    yvalid = (rng.random(n) >= 0.01) if y_nulls else None
    if y_kind is not None:
        y = (y > np.median(y)).astype(np.float32)
    cols["y"] = make_column(y, pa.float32(), yvalid, (n // 5,), 4, seed=seed + 99)
    return Frame(cols), [f"x{j}" for j in range(p)], yvalid, fvalid


def _three(monkeypatch, f64, df, make):
    """(gpu, oracle in the same precision, f64 oracle on the same inputs) of the expression `make()` builds."""
    import polars_ds_extension_b200.config as cfg
    from tests.backends import OracleBackend, PluginBackend

    monkeypatch.setattr(cfg, "LIN_REG_EXPR_F64", f64)
    e = make()
    g, o = PluginBackend().eval(df, e), OracleBackend().eval(df, e)
    if f64:
        return g, o, o
    monkeypatch.setattr(cfg, "LIN_REG_EXPR_F64", True)
    truth = OracleBackend().eval(df, make())
    monkeypatch.setattr(cfg, "LIN_REG_EXPR_F64", False)
    return g, o, truth


def _accept(f64, g, o, truth, what):
    from tests.parity_rule import accept_f32, accept_f64

    assert g is not None and o is not None, what
    if f64:
        accept_f64(g, o, what)
    else:
        accept_f32(g, o, truth, what)


def _check_pred(f64, g, o, truth, what, kept=None):
    """pred / resid of pl_lr_pred: the valid bitmap is the oracle's exactly, no kept row is NaN, values by the rule."""
    for part in ("pred", "resid"):
        (gv, gval), (ov, oval), (tv, _) = g[part], o[part], truth[part]
        assert np.array_equal(gval, oval), f"{what} {part}: valid bitmap differs from the oracle's"
        if kept is not None:
            assert np.array_equal(gval, kept), f"{what} {part}: kept rows"
        assert np.isfinite(gv[gval]).all(), f"{what} {part}: a kept row is NaN"
        if part == "pred":
            _accept(f64, gv[gval], ov[oval], tv[oval], f"{what} {part}")


def _lr(xs, target="y", **kw):
    """lin_reg with a bias and without the rank gate (the mixed features are checked, not the gate)."""
    import polars_ds_extension_b200 as pds

    return pds.lin_reg(*xs, target=target, add_bias=True, singular_x_tol=0.0, **kw)


def _route():
    from polars_ds_extension_b200._lib import lib

    return lib().pdsb_last_moments_path()


@pytest.mark.parametrize("f64", [False, True], ids=["f32", "f64"])
@pytest.mark.parametrize("n,p", [(20_011, 3), (20_011, 17), (20_011, 64), (300_007, 3), (300_007, 17), (300_007, 64)])
def test_masked_lin_reg_on_mixed_inputs(monkeypatch, f64, n, p):
    """pl_lr / pl_lr_pred with "skip" and nulls in features and target: the masked wgmma kernel (path 1) in f32, the
    masked DMMA kernels in f64; pred's valid bitmap is the oracle's and masked rows are never NaN-poisoned."""
    import polars_ds_extension_b200 as pds

    df, xs, _, _ = e2e_frame(100 + p + n % 7, n, p)
    g, o, truth = _three(monkeypatch, f64, df, lambda: _lr(xs))
    _accept(f64, g, o, truth, f"lin_reg {n}x{p}")
    if not f64:
        assert _route() == 1, _route()
    if n < 100_000:
        g, o, truth = _three(monkeypatch, f64, df, lambda: _lr(xs, return_pred=True))
        _check_pred(f64, g, o, truth, f"lin_reg pred {n}x{p}")
        if not f64:
            assert _route() == 1, _route()


@pytest.mark.parametrize("f64", [False, True], ids=["f32", "f64"])
def test_fill_with_null_target_keeps_target_valid_rows(monkeypatch, f64):
    """FILL ("-2.5") with nulls in features and target: the features are filled and the kept rows are exactly the rows
    whose target is valid."""
    import polars_ds_extension_b200 as pds

    df, xs, yvalid, _ = e2e_frame(7, 20_011, 11)
    for pol in ("-2.5", "one"):
        g, o, truth = _three(monkeypatch, f64, df, lambda: _lr(xs, null_policy=pol))
        _accept(f64, g, o, truth, f"lin_reg {pol}")
        g, o, truth = _three(monkeypatch, f64, df,
                             lambda: _lr(xs, null_policy=pol, return_pred=True))
        _check_pred(f64, g, o, truth, f"lin_reg pred {pol}", kept=yvalid)


def test_int_features_without_nulls_take_the_register_kernel(monkeypatch):
    """No nulls, integer features of every width at offsets and chunk splits, n >= 65 536 and p <= 10: the register
    moments kernel (path 3) in f32."""
    import polars_ds_extension_b200 as pds

    df, xs, _, _ = e2e_frame(8, 70_001, 8, x_nulls=False, y_nulls=False,
                             kinds=["i8", "u8", "i16", "u16", "i32", "u32", "i64", "u64"])
    g, o, truth = _three(monkeypatch, False, df, lambda: _lr(xs))
    _accept(False, g, o, truth, "lin_reg int features")
    assert _route() == 3, _route()


@pytest.mark.parametrize("f64", [False, True], ids=["f32", "f64"])
def test_weighted_lin_reg_on_mixed_inputs(monkeypatch, f64):
    """Weighted pl_lr on mixed, sliced, chunked inputs (f32: the widened DMMA kernels).  With nulls, "skip" drops rows
    and the weights no longer match the data: the reference's error (linear_regression.rs:441-446), on both sides."""
    import polars_ds_extension_b200 as pds
    import polars_ds_extension_b200.config as cfg
    from polars_ds_extension_b200._lib import PdsbError
    from tests.backends import OracleBackend, PluginBackend

    from oracle.lin_reg_oracle import OracleError

    w = np.random.default_rng(9).uniform(0.2, 2.0, 20_011).astype(np.float32)
    wcol = make_column(w, pa.float32(), None, (1001,), 5)
    make = lambda: _lr(xs, weights="w")  # noqa: E731
    df, xs, _, _ = e2e_frame(9, 20_011, 6, x_nulls=False, y_nulls=False)
    g, o, truth = _three(monkeypatch, f64, df.with_columns(w=wcol), make)
    _accept(f64, g, o, truth, "weighted lin_reg")
    if not f64:
        assert _route() == 0, _route()
    df, xs, _, _ = e2e_frame(9, 20_011, 6)
    df = df.with_columns(w=wcol)
    monkeypatch.setattr(cfg, "LIN_REG_EXPR_F64", f64)
    with pytest.raises(PdsbError, match="Shape of weights is not the same as the data."):
        PluginBackend().eval(df, make())
    with pytest.raises(OracleError, match="Shape of weights is not the same as the data."):
        OracleBackend().eval(df, make())


@pytest.mark.parametrize("f64", [False, True], ids=["f32", "f64"])
@pytest.mark.parametrize("p", [5, 70])
def test_small_fits_on_mixed_inputs(monkeypatch, f64, p):
    """n < 4096 (no tensor-core kernel in f32; p = 70 takes the tile kernel): pl_lr and pl_lr_pred with "skip"."""
    import polars_ds_extension_b200 as pds

    df, xs, _, _ = e2e_frame(10 + p, 3_001, p)
    g, o, truth = _three(monkeypatch, f64, df, lambda: _lr(xs))
    _accept(f64, g, o, truth, f"small lin_reg p={p}")
    if not f64:
        assert _route() == 0, _route()
    g, o, truth = _three(monkeypatch, f64, df, lambda: _lr(xs, return_pred=True))
    _check_pred(f64, g, o, truth, f"small lin_reg pred p={p}")


@pytest.mark.parametrize("f64", [False, True], ids=["f32", "f64"])
@pytest.mark.parametrize("pol", ["-2.5", MIDPOINT])
def test_multi_target_fill(monkeypatch, f64, pol):
    """pl_lr_multi / pl_lr_multi_pred with a fill policy and nulls in the features."""
    import polars_ds_extension_b200 as pds

    df, xs, _, _ = e2e_frame(12, 5_003, 6, y_nulls=False)
    y2 = np.random.default_rng(12).standard_normal(5_003).astype(np.float32)
    df = df.with_columns(y2=make_column(y2, pa.float32(), None, (17,), 3))
    g, o, truth = _three(monkeypatch, f64, df, lambda: _lr(xs, target=["y", "y2"],
                                                                   null_policy=pol))
    for k in o:
        _accept(f64, g[k], o[k], truth[k], f"multi {k}")
    g, o, truth = _three(monkeypatch, f64, df, lambda: _lr(xs, target=["y", "y2"],
                                                                   null_policy=pol, return_pred=True))
    for k in o:
        (gv, gval), (ov, oval), (tv, _) = g[k], o[k], truth[k]
        assert np.array_equal(gval, oval), k
        _accept(f64, gv[gval], ov[oval], tv[oval], f"multi pred {k}")


@pytest.mark.parametrize("f64", [False, True], ids=["f32", "f64"])
@pytest.mark.parametrize("weighted", [False, True])
def test_reports_skip(monkeypatch, f64, weighted):
    """lin_reg_report and the WLS report with "skip" on mixed, sliced inputs; nulls in features and target for the OLS
    report only (the reference's WLS report keeps every weight while "skip" drops rows, so it has no answer there)."""
    import polars_ds_extension_b200 as pds

    df, xs, _, _ = e2e_frame(13, 5_003, 5, x_nulls=not weighted, y_nulls=not weighted)
    w = np.random.default_rng(13).uniform(0.2, 2.0, 5_003).astype(np.float32)
    df = df.with_columns(w=make_column(w, pa.float32(), None, (), 2))
    g, o, truth = _three(monkeypatch, f64, df, lambda: pds.lin_reg_report(
        *xs, target="y", add_bias=True, null_policy="skip", weights="w" if weighted else None))
    for k in ("beta", "std_err", "t", "p>|t|"):
        if k in o:
            _accept(f64, g[k], o[k], truth[k], f"report {k}")
    assert g["features"] == o["features"]


@pytest.mark.parametrize("pol", ["skip", "zero"])
def test_logistic_on_mixed_inputs(monkeypatch, pol):
    """logistic_reg (float64 only) with "skip" and "zero" on mixed, sliced, null-bearing features and target."""
    import polars_ds_extension_b200 as pds
    from tests.backends import OracleBackend, PluginBackend
    from tests.parity_rule import rel

    df, xs, _, _ = e2e_frame(14, 5_003, 6, y_kind="binary")
    e = pds.logistic_reg(*xs, target="y", add_bias=True, null_policy=pol, tol=1e-10, max_iter=400)
    g, o = PluginBackend().eval(df, e), OracleBackend().eval(df, e)
    assert rel(g, o) < 1e-5, (pol, rel(g, o))
    e = pds.logistic_reg(*xs, target="y", add_bias=True, null_policy=pol, tol=1e-10, max_iter=400, return_pred=True)
    (gv, gval), (ov, oval) = PluginBackend().eval(df, e), OracleBackend().eval(df, e)
    assert np.array_equal(gval, oval)
    assert rel(gv[gval], ov[oval]) < 1e-5


@pytest.mark.parametrize("f64", [False, True], ids=["f32", "f64"])
@pytest.mark.parametrize("pol", ["skip", "one"])
@pytest.mark.parametrize("rolling", [True, False], ids=["rolling", "recursive"])
def test_online_fits_on_mixed_inputs(monkeypatch, f64, pol, rolling):
    """rolling_lin_reg / recursive_lin_reg with "skip" and "one": one int16 and one u32 feature, nulls, offset slices."""
    import polars_ds_extension_b200 as pds
    from tests.parity_rule import rel

    df, xs, _, _ = e2e_frame(15, 2_001, 3, kinds=["i16", "u32", "f64"])
    make = (lambda: pds.rolling_lin_reg(*xs, target="y", window_size=60, add_bias=True, null_policy=pol)) if rolling \
        else (lambda: pds.recursive_lin_reg(*xs, target="y", start_with=30, add_bias=True, null_policy=pol))
    g, o, truth = _three(monkeypatch, f64, df, make)
    assert [c is None for c in g["coeffs"]] == [c is None for c in o["coeffs"]]
    assert np.array_equal(g["pred"][1], o["pred"][1])
    rows = [i for i, c in enumerate(o["coeffs"]) if c is not None]
    assert rows
    gc, oc = np.array([g["coeffs"][i] for i in rows]), np.array([o["coeffs"][i] for i in rows])
    tc = np.array([truth["coeffs"][i] for i in rows])
    tol = 1e-6 if f64 else 1e-3
    worst = max(rel(gc[k], oc[k]) for k in range(len(rows)))
    assert worst < tol or (not f64 and max(rel(gc[k], tc[k]) for k in range(len(rows))) < tol), worst
