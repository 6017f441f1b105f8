"""Time recursive_lin_reg(...).over(key) on the device with CUDA events, through the plugin, and Polars' loop.

    python scripts/time_grouped_recursive.py [--repeats R] [--scale S] [--loop-groups K]

Cases (median and range over R timed runs after one warm-up, one JSON line each):
  * pdsb_dev_grouped_recursive_lin_reg_* on resident data, start_with = 16:
      - 1e4 groups x 1e4 rows x 8 f32 features with a bias (packed pass C), next to pdsb_dev_online_lin_reg_f32 on the
        same 1e8 rows as one recursive column;
      - 5e3 x 2.5e3 and 1e6 x 100, 8 f32 features with a bias (packed);
      - 1e3 x 1e4, 8 f64 features with a bias (lane-per-moment pass C);
      - 1e3 x 1e3, 13 f32 features with a bias (14 coefficients: generic pass C).
    Each is reported against the 3.35 TB/s data-sheet HBM3 bandwidth from the minimum bytes per row: read x and y, write
    the coefficients, pred and the validity byte;
  * pl_recursive_lr_by_f32 through the plugin C ABI on 1e3 groups x 1e4 host rows x 8 f32 features with a bias (host
    clock after a synchronise; includes the upload and the copy back);
  * Polars' loop (one pl_recursive_lr_f32 call per group) on the first K of those groups, scaled up to 1e3 groups.
The device name and power limit are read in the same run.  Writes nothing to disk.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from scripts.timing import PEAK, device_info, event_times, host_times  # noqa: E402

START = 16


def main():
    import pyarrow as pa
    import torch

    import polars_ds_extension_b200 as pds
    from polars_ds_extension_b200 import _harness
    from polars_ds_extension_b200._lib import check

    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--scale", type=float, default=1.0, help="fraction of the default group counts")
    ap.add_argument("--loop-groups", type=int, default=50, help="groups the per-group loop is timed on")
    args = ap.parse_args()
    print(json.dumps(device_info(torch)), flush=True)
    L = pds.lib()
    gen = torch.Generator(device="cuda").manual_seed(1)
    cases = [("1e4 x 1e4", 10_000, 10_000, 8, torch.float32), ("5e3 x 2.5e3", 5_000, 2_500, 8, torch.float32),
             ("1e6 x 100", 1_000_000, 100, 8, torch.float32), ("1e3 x 1e4 f64", 1_000, 10_000, 8, torch.float64),
             ("1e3 x 1e3, 14 coefficients", 1_000, 1_000, 13, torch.float32)]
    for name, G, s, p, dt in cases:
        G = max(1, int(G * args.scale))
        n = G * s
        sfx = "f32" if dt == torch.float32 else "f64"
        esz = 4 if dt == torch.float32 else 8
        q = p + 1
        X = torch.randn((p, n), dtype=dt, device="cuda", generator=gen)
        y = X.sum(0) * 0.25 + 0.1 * torch.randn(n, dtype=dt, device="cuda", generator=gen)
        offsets = torch.arange(0, n + 1, s, dtype=torch.int64, device="cuda")
        co = torch.empty((n, q), dtype=dt, device="cuda")
        pr = torch.empty(n, dtype=dt, device="cuda")
        va = torch.empty(n, dtype=torch.uint8, device="cuda")
        fn = getattr(L, f"pdsb_dev_grouped_recursive_lin_reg_{sfx}")
        ts = event_times(torch, lambda: check(fn(X.data_ptr(), n, y.data_ptr(), n, p, 1, START, 0.0, offsets.data_ptr(),
                                                 G, None, co.data_ptr(), pr.data_ptr(), va.data_ptr(), None)),
                         args.repeats)
        m, lo, hi = float(np.median(ts)), min(ts), max(ts)
        path = int(L.pdsb_last_online_path())
        assert int(va.sum()) == G * (s - START + 1)
        nbytes = n * ((p + 1) * esz + q * esz + esz + 1)
        print(json.dumps({"case": f"pdsb_dev_grouped_recursive_lin_reg_{sfx}", "shape": name, "groups": G, "rows": n,
                          "features": p, "bias": True, "pass_c": path, "ms_median": m * 1e3, "ms_min": lo * 1e3,
                          "ms_max": hi * 1e3, "hbm_fraction_min_bytes": nbytes / m / PEAK}), flush=True)
        if name == "1e4 x 1e4":
            one = getattr(L, f"pdsb_dev_online_lin_reg_{sfx}")
            ts = event_times(torch, lambda: check(one(X.data_ptr(), n, y.data_ptr(), n, p, 1, 0, START, 0, 0.0,
                                                      co.data_ptr(), pr.data_ptr(), va.data_ptr(), None)), args.repeats)
            m, lo, hi = float(np.median(ts)), min(ts), max(ts)
            print(json.dumps({"case": f"pdsb_dev_online_lin_reg_{sfx} on the same rows as one recursive column",
                              "rows": n, "pass_c": int(L.pdsb_last_online_path()), "ms_median": m * 1e3,
                              "ms_min": lo * 1e3, "ms_max": hi * 1e3, "hbm_fraction_min_bytes": nbytes / m / PEAK}),
                  flush=True)
        del X, y, offsets, co, pr, va
        torch.cuda.empty_cache()

    G, s, p = max(1, int(1000 * args.scale)), 10_000, 8
    rng = np.random.default_rng(2)
    X = rng.standard_normal((G * s, p)).astype(np.float32)
    y = (X.sum(1) * 0.25 + 0.1 * rng.standard_normal(G * s)).astype(np.float32)
    cols = [pa.chunked_array([pa.array(y)])] + [pa.chunked_array([pa.array(X[:, j])]) for j in range(p)]
    names = ["y"] + [f"x{j}" for j in range(p)]
    offsets = pa.chunked_array([pa.array(np.arange(G + 1, dtype=np.int64) * s)])
    kw = {"null_policy": "raise", "n": START, "bias": True, "lambda": 0.0, "min_size": 0}

    def fast():
        return _harness.call_plugin("pl_recursive_lr_by_f32", [offsets] + cols, ["__offsets__"] + names, kw)

    ts = host_times(torch, fast, args.repeats)
    print(json.dumps({"case": "pl_recursive_lr_by_f32 e2e (plugin, host columns)", "groups": G, "rows": G * s,
                      "features": p, "ms_median": float(np.median(ts)) * 1e3, "ms_min": min(ts) * 1e3,
                      "ms_max": max(ts) * 1e3}), flush=True)
    K = min(args.loop_groups, G)
    parts = [[c.slice(g * s, s) for c in cols] for g in range(K)]
    _harness.call_plugin("pl_recursive_lr_f32", parts[0], names, kw)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for part in parts:
        _harness.call_plugin("pl_recursive_lr_f32", part, names, kw)
    t = time.perf_counter() - t0
    print(json.dumps({"case": "Polars' loop: pl_recursive_lr_f32 once per group", "groups_timed": K,
                      "rows_per_group": s, "ms_timed": t * 1e3, "ms_scaled_to_groups": t * 1e3 * G / K,
                      "groups": G}), flush=True)


if __name__ == "__main__":
    main()
