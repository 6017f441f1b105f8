"""Time rolling_lin_reg over groups on the device with CUDA events, through the host entry, and the per-group loop.

    python scripts/time_grouped_rolling.py [--repeats R] [--scale S] [--loop-groups K]

Cases (median and range over R timed runs after one warm-up, one JSON line each):
  * pdsb_dev_grouped_rolling_lin_reg_* on resident data, min_rows = 0:
      - 1e4 groups x 1e4 rows x 8 f32 features with a bias, window 1024 (packed pass C), next to
        pdsb_dev_online_lin_reg_f32 on the same 1e8 rows as one rolling column;
      - 1e6 x 100, 8 f32 features with a bias, window 20 (lane-per-moment pass C, direct head);
      - 1 x 1e8, 8 f32 features with a bias, window 20: the grouped lane-per-moment instance on the chains of one
        column, next to pdsb_dev_online_lin_reg_f32 on the same rows (the single-column instance, same chains);
      - 1e3 x 1e4, 8 f64 features with a bias, window 256 (lane-per-moment);
      - 1e3 x 1e4, 8 f32 features with a bias, window 256, every other group skipping nulls: two plans in one call
        (packed pass C for the groups without skip, lane-per-moment with the direct head for the others);
      - 1e3 x 1e3, 13 f32 features with a bias, window 256 (14 coefficients: generic pass C).
    Each is reported against the 3.35 TB/s data-sheet HBM3 bandwidth from the minimum bytes per row: read x and y, write
    the coefficients, pred and the validity byte;
  * pdsb_host_grouped_rolling (f32) on 1e3 groups x 1e4 host rows x 8 f32 features with a bias, window 1024 (host clock
    after a synchronise; includes the upload and the copy back);
  * the loop of pl_rolling_lr_f32 once per group (what Polars' over does) on the first K of those groups, scaled up to
    1e3 groups.
The device name and power limit are read in the same run.  Writes nothing to disk.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from scripts.timing import device_info, event_times, host_times, line  # noqa: E402


def main():
    import pyarrow as pa
    import torch

    import polars_ds_extension_b200 as pds
    from polars_ds_extension_b200 import _harness
    from polars_ds_extension_b200 import device as dev
    from polars_ds_extension_b200._lib import Column, HostResult, LrKwargs, check

    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--scale", type=float, default=1.0, help="fraction of the default group counts")
    ap.add_argument("--loop-groups", type=int, default=50, help="groups the per-group loop is timed on")
    args = ap.parse_args()
    print(json.dumps(device_info(torch)), flush=True)
    L = pds.lib()
    gen = torch.Generator(device="cuda").manual_seed(1)
    # (name, groups, rows per group, features, dtype, window, every other group skips)
    cases = [("1e4 x 1e4, w 1024", 10_000, 10_000, 8, torch.float32, 1024, False),
             ("1e6 x 100, w 20", 1_000_000, 100, 8, torch.float32, 20, False),
             ("1 x 1e8, w 20", 1, 100_000_000, 8, torch.float32, 20, False),
             ("1e3 x 1e4 f64, w 256", 1_000, 10_000, 8, torch.float64, 256, False),
             ("1e3 x 1e4, w 256, half the groups skip", 1_000, 10_000, 8, torch.float32, 256, True),
             ("1e3 x 1e3, 14 coefficients, w 256", 1_000, 1_000, 13, torch.float32, 256, False)]
    for name, G, s, p, dt, w, half in cases:
        G, s = (1, max(1024, int(s * args.scale))) if G == 1 else (max(2, int(G * args.scale)), s)
        n = G * s
        sfx = "f32" if dt == torch.float32 else "f64"
        esz = 4 if dt == torch.float32 else 8
        q = p + 1
        X = torch.randn((p, n), dtype=dt, device="cuda", generator=gen)
        y = X.sum(0) * 0.25 + 0.1 * torch.randn(n, dtype=dt, device="cuda", generator=gen)
        offsets = torch.arange(0, n + 1, s, dtype=torch.int64, device="cuda")
        skip = (torch.arange(G, device="cuda") % 2).to(torch.uint8) if half else None
        co = torch.empty((n, q), dtype=dt, device="cuda")
        pr = torch.empty(n, dtype=dt, device="cuda")
        va = torch.empty(n, dtype=torch.uint8, device="cuda")
        fn = getattr(L, f"pdsb_dev_grouped_rolling_lin_reg_{sfx}")
        sp = None if skip is None else skip.data_ptr()
        ts = event_times(torch, lambda: check(fn(X.data_ptr(), n, y.data_ptr(), n, p, 1, w, 0, 0.0, offsets.data_ptr(),
                                                 G, sp, co.data_ptr(), pr.data_ptr(), va.data_ptr(), None)),
                         args.repeats)
        path = int(L.pdsb_last_online_path())
        assert int(va.sum()) == G * (s - w + 1)
        nbytes = n * ((p + 1) * esz + q * esz + esz + 1)
        line(f"pdsb_dev_grouped_rolling_lin_reg_{sfx}", n, G, ts, nbytes, shape=name, features=p, bias=True, window=w,
             pass_c=path)
        if name.startswith("1e4 x 1e4") or name.startswith("1 x 1e8"):
            one = getattr(L, f"pdsb_dev_online_lin_reg_{sfx}")
            ts = event_times(torch, lambda: check(one(X.data_ptr(), n, y.data_ptr(), n, p, 1, w, 0, 0, 0.0,
                                                      co.data_ptr(), pr.data_ptr(), va.data_ptr(), None)), args.repeats)
            line(f"pdsb_dev_online_lin_reg_{sfx} on the same rows as one rolling column", n, 1, ts, nbytes, window=w,
                 pass_c=int(L.pdsb_last_online_path()))
        del X, y, offsets, skip, co, pr, va
        torch.cuda.empty_cache()

    G, s, p, w = max(2, int(1000 * args.scale)), 10_000, 8, 1024
    rng = np.random.default_rng(2)
    X = rng.standard_normal((G * s, p)).astype(np.float32)
    y = (X.sum(1) * 0.25 + 0.1 * rng.standard_normal(G * s)).astype(np.float32)
    cols = [pa.chunked_array([pa.array(y)])] + [pa.chunked_array([pa.array(X[:, j])]) for j in range(p)]
    keep: list = []
    ccols = (Column * len(cols))(*[dev._column(c, None, False, keep) for c in cols])
    off = (C.c_int64 * (G + 1))(*(np.arange(G + 1, dtype=np.int64) * s).tolist())
    kw = LrKwargs(bias=1, null_policy=b"raise", n=w, lambda_=0.0, min_size=0)

    def fast():
        r = HostResult()
        check(L.pdsb_host_grouped_rolling(ccols, len(cols), off, G, C.byref(kw), 1, C.byref(r)))
        L.pdsb_host_result_free(C.byref(r))

    line("pdsb_host_grouped_rolling f32 e2e (host columns)", G * s, G, host_times(torch, fast, args.repeats),
         features=p, window=w)
    names = ["y"] + [f"x{j}" for j in range(p)]
    pkw = {"null_policy": "raise", "n": w, "bias": True, "lambda": 0.0, "min_size": 0}
    K = min(args.loop_groups, G)
    parts = [[c.slice(g * s, s) for c in cols] for g in range(K)]
    _harness.call_plugin("pl_rolling_lr_f32", parts[0], names, pkw)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for part in parts:
        _harness.call_plugin("pl_rolling_lr_f32", part, names, pkw)
    t = time.perf_counter() - t0
    print(json.dumps({"case": "per-group loop: pl_rolling_lr_f32 once per group", "groups_timed": K,
                      "rows_per_group": s, "ms_timed": t * 1e3, "ms_scaled_to_groups": t * 1e3 * G / K,
                      "groups": G}), flush=True)


if __name__ == "__main__":
    main()
