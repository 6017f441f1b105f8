"""CPU-side checks of rolling_lin_reg over groups: the device and host entries are exported and declared in pdsb.h, their
argument errors (window < 1, bad offsets, the single call's checks) come before any device work, and a well-formed call
fails loudly without a GPU."""
import ctypes as C
from pathlib import Path

import numpy as np
import pyarrow as pa
import pytest

from polars_ds_extension_b200 import device as dev
from polars_ds_extension_b200._lib import Column, HostResult, LrKwargs, PdsbError, check, lib
from tests.helpers import has_gpu

ROOT = Path(__file__).resolve().parent.parent
ENTRIES = ["pdsb_host_grouped_rolling", "pdsb_dev_grouped_rolling_lin_reg_f32", "pdsb_dev_grouped_rolling_lin_reg_f64"]


@pytest.mark.parametrize("fn", ENTRIES)
def test_entry_exported_and_declared(fn):
    assert hasattr(lib(), fn), fn
    assert f"int {fn}(" in (ROOT / "include" / "pdsb.h").read_text(), fn


def _host(offsets, window=3, n=10, policy="raise", f32=True):
    keep: list = []
    rng = np.random.default_rng(0)
    arrs = [pa.array(rng.standard_normal(n).astype(np.float32 if f32 else np.float64)) for _ in range(3)]
    cols = (Column * 3)(*[dev._column(a, None, False, keep) for a in arrs])
    kw = LrKwargs(bias=1, null_policy=policy.encode(), n=window, lambda_=0.0, min_size=0)
    off = (C.c_int64 * len(offsets))(*offsets)
    r = HostResult()
    try:
        check(lib().pdsb_host_grouped_rolling(cols, 3, off, len(offsets) - 1, C.byref(kw), int(f32), C.byref(r)))
    finally:
        lib().pdsb_host_result_free(C.byref(r))


@pytest.mark.parametrize("offsets,msg", [([0, 5, 9], "grouped rolling_lin_reg: bad group offsets"),
                                         ([1, 5, 10], "grouped rolling_lin_reg: bad group offsets"),
                                         ([0, 6, 5, 10], "grouped rolling_lin_reg: group offsets must be non-decreasing")])
def test_bad_offsets_are_refused_before_device_work(offsets, msg):
    with pytest.raises(PdsbError, match=msg):
        _host(offsets)


@pytest.mark.parametrize("window,sizes,msg", [(0, [5, 5], "window / start_with must be >= 1"),
                                              (6, [6, 4], "#Data < window size"),
                                              (3, [5, 2, 3], "#Data < #features"),
                                              (3, [5, 0, 5], "Empty data")])
def test_the_single_calls_checks_come_before_device_work(window, sizes, msg):
    with pytest.raises(PdsbError, match=msg):
        _host([0] + np.cumsum(sizes).tolist(), window=window, n=sum(sizes))


def test_policy_name_is_checked():
    with pytest.raises(PdsbError):
        _host([0, 5, 10], policy="nonsense")


@pytest.mark.parametrize("sfx", ["f32", "f64"])
@pytest.mark.parametrize("window", [0, -3])
def test_device_entry_refuses_window_below_one(sfx, window):
    fn = getattr(lib(), f"pdsb_dev_grouped_rolling_lin_reg_{sfx}")
    with pytest.raises(PdsbError, match=f"grouped rolling_lin_reg: window must be >= 1 \\(got {window}\\)"):
        check(fn(None, 10, None, 10, 2, 1, window, 0, 0.0, None, 2, None, None, None, None, None))


@pytest.mark.skipif(has_gpu(), reason="checks the loud failure on a box without a GPU")
@pytest.mark.parametrize("f32", [True, False])
def test_well_formed_call_fails_loudly_without_gpu(f32):
    with pytest.raises(PdsbError, match="no CPU fallback"):
        _host([0, 5, 10], f32=f32)
    fn = getattr(lib(), f"pdsb_dev_grouped_rolling_lin_reg_{'f32' if f32 else 'f64'}")
    with pytest.raises(PdsbError, match="no CPU fallback"):
        check(fn(None, 10, None, 10, 2, 1, 3, 0, 0.0, None, 2, None, None, None, None, None))
