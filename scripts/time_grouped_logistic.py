"""Time group_by(key).agg(logistic_reg) on the device (K16): the batched fit on device-resident data with CUDA events,
the plugin call end to end, and Polars' per-group loop for scale.

    python scripts/time_grouped_logistic.py [--repeats R] [--scale S]

Cases (median and range over R timed runs after one warm-up, one JSON line each), f64 [X | y] column-major, 8 features
plus a bias, labels drawn from a logistic model:
  * 1e4 groups of 1e4 rows;
  * 1e6 groups of 100 rows;
  * one 5e7-row group followed by 1e5 groups of 500 rows;
  each with the iterations the call ran, its algorithmic bytes (the sum over iterations of the rows of the groups still
  running times (p + 1) * 8: pass A reads X and y once per iteration, w and z never reach memory) and the share of the
  3.35 TB/s data-sheet HBM3 bandwidth those bytes imply.  The running groups per iteration come from extra calls with
  max_iter = 1, 2, ... outside the timed runs;
  * the pl_logistic_by plugin call on 1e7 host rows in 1e4 groups (host clock after a synchronise: upload, fit, copy
    back);
  * for scale, group_by().agg(fast=False) (one pl_logistic_coeffs call per group, Polars' loop) and fast=True on the
    first 1 % of the rows in key order.
The device name and power limit are read in the same run.  Writes nothing to disk.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from scripts.timing import device_info, event_times, host_times, line  # noqa: E402

P = 8
S = 8          # bytes per f64 value
TOL = 1e-8


def device_case(torch, L, sizes, label, repeats):
    from polars_ds_extension_b200._lib import LOGISTIC_MAX_ITER, check

    n, ng = int(sum(sizes)), len(sizes)
    ld = (n + 1) // 2 * 2
    gen = torch.Generator(device="cuda").manual_seed(5)
    X = torch.randn((P, ld), dtype=torch.float64, device="cuda", generator=gen)
    w = torch.linspace(-1.0, 1.0, P, dtype=torch.float64, device="cuda")
    y = (torch.rand(ld, dtype=torch.float64, device="cuda", generator=gen) < torch.sigmoid(w @ X + 0.3)).double()
    size_t = torch.tensor(sizes, dtype=torch.int64, device="cuda")
    offsets = torch.cat([torch.zeros(1, dtype=torch.int64, device="cuda"), torch.cumsum(size_t, 0)])
    beta = torch.empty((ng, P + 1), dtype=torch.float64, device="cuda")
    status = torch.empty(ng, dtype=torch.int32, device="cuda")
    n_iter = C.c_int64(0)
    ptr = lambda t: C.c_void_p(t.data_ptr())     # noqa: E731

    def fit(max_iter=200):
        check(L.pdsb_dev_grouped_logistic_f64(ptr(X), ld, ptr(y), None, ptr(offsets), ng, n, P, 1, 0.0, 0.0, TOL,
                                              max_iter, ptr(beta), ptr(status), C.byref(n_iter), None))

    ts = event_times(torch, fit, repeats)
    iters = int(n_iter.value)
    # rows read per iteration: every group's rows at iteration 1, then those of the groups still running
    running_rows = [n]
    for k in range(1, iters):
        fit(k)
        running_rows.append(int(size_t[status == LOGISTIC_MAX_ITER].sum()))
    fit()
    nbytes = sum(running_rows) * (P + 1) * S
    line(f"{label}: grouped logistic fit", n, ng, ts, nbytes, iterations=iters,
         ms_per_iteration=float(np.median(ts)) * 1e3 / iters, running_rows_per_iteration=running_rows,
         converged=int((status == 0).sum()))
    del X, y
    torch.cuda.empty_cache()


def main():
    import pyarrow as pa
    import torch

    import polars_ds_extension_b200 as pds
    from polars_ds_extension_b200 import _harness

    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--scale", type=float, default=1.0, help="fraction of the default row counts")
    args = ap.parse_args()
    print(json.dumps(device_info(torch)), flush=True)
    L = pds.lib()
    rng = np.random.default_rng(4)
    n = int(1e8 * args.scale)
    k = max(1, int(1e4 * args.scale))
    device_case(torch, L, [n // k] * k, "1e4 groups of 1e4 rows", args.repeats)
    device_case(torch, L, [100] * (n // 100), "1e6 groups of 100 rows", args.repeats)
    device_case(torch, L, [n // 2] + [500] * (n // 2 // 500), "one 5e7-row group + 1e5 groups of 500 rows", args.repeats)

    # the plugin end to end on host columns
    nh = int(1e7 * args.scale)
    ngh = max(1, int(1e4 * args.scale))
    gid = np.sort(rng.integers(0, ngh, nh))
    Xh = rng.standard_normal((nh, P))
    yh = (rng.random(nh) < 1.0 / (1.0 + np.exp(-(Xh @ (np.arange(P) / P - 0.5) + 0.3)))).astype(np.float64)
    counts = np.bincount(gid, minlength=ngh)
    offs = pa.array(np.concatenate([[0], np.cumsum(counts)]).astype(np.int64))
    xs = [f"x{i}" for i in range(P)]
    e = pds.logistic_reg(*xs, target="y", add_bias=True, tol=TOL)
    ins = [offs, pa.array(yh)] + [pa.array(np.ascontiguousarray(Xh[:, i])) for i in range(P)]
    names = ["__offsets__", "y"] + xs

    line("pl_logistic_by plugin call (host columns in key order)", nh, ngh,
         host_times(torch, lambda: _harness.call_plugin("pl_logistic_by", ins, names, e.kwargs), args.repeats))
    cut = nh // 100          # the first 1 % of the rows in key order: ~1 % of the groups, whole
    sl = pds.Frame({"y": yh[:cut]} | {x: Xh[:cut, i] for i, x in enumerate(xs)} | {"g": gid[:cut]})
    ngs = len(np.unique(gid[:cut]))
    line("1 % slice: group_by('g').agg(fast=False), one pl_logistic_coeffs call per group", cut, ngs,
         host_times(torch, lambda: sl.group_by("g").agg(e), 1))
    line("1 % slice: group_by('g').agg(fast=True)", cut, ngs,
         host_times(torch, lambda: sl.group_by("g").agg(e, fast=True), args.repeats))


if __name__ == "__main__":
    main()
