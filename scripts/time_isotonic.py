"""Time isotonic_regression on device-resident data with CUDA events, one end-to-end plugin call, and SciPy.

    python scripts/time_isotonic.py [--repeats R] [--scale S]

Cases (median and range over R timed runs after one warm-up, one JSON line each):
  * pdsb_dev_isotonic_f64 on 1e8 resident f64 rows, unweighted and weighted, on six shapes: random walk, noisy upward
    trend, strictly increasing (no pooling), strictly decreasing (one block), increasing with a final huge drop (every
    block pooled across every partition and level) and a sawtooth (one violation per 32 rows).  Reported against the
    3.35 TB/s data-sheet HBM3 bandwidth from the minimum 16 B/row (read y, write the fit; 24 B/row with weights) and from
    the design's own upper bound (the leaf pass also writes 25 B per stack block, at most one block per row, and the
    final pass rewrites at most every row);
  * the worst shape's time over the random walk's, per weighting (no path is serial when it stays small);
  * pds.isotonic_regression through the plugin C ABI on 1e7 f64 host rows (host clock after a synchronise; includes the
    upload of the pageable Arrow buffers and the copy back);
  * for scale, scipy.optimize.isotonic_regression (one CPU core) at 1e7 rows.
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

SHAPES = ["walk", "trend", "increasing", "decreasing", "drop", "sawtooth"]


def make(torch, kind, n, gen):
    i = torch.arange(n, dtype=torch.float64, device="cuda")
    if kind == "walk":
        return torch.cumsum(torch.randn(n, dtype=torch.float64, device="cuda", generator=gen), 0)
    if kind == "trend":
        return i * (4.0 / n) + torch.randn(n, dtype=torch.float64, device="cuda", generator=gen)
    u = 0.5 * torch.rand(n, dtype=torch.float64, device="cuda", generator=gen)
    if kind == "increasing":
        return i + u
    if kind == "decreasing":
        return -i - u
    if kind == "drop":
        y = i + u
        y[-1] = -float(n) * n          # below minus the sum of the rest: everything pools into one block
        return y
    if kind == "sawtooth":
        return torch.remainder(i, 32.0) + 16.0 * torch.floor(i / 32.0) + 0.05 * (u - 0.25)
    raise ValueError(kind)


def main():
    import torch

    import polars_ds_extension_b200 as pds
    from polars_ds_extension_b200._lib import check

    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--scale", type=float, default=1.0, help="fraction of the default row counts")
    args = ap.parse_args()
    print(json.dumps(device_info(torch)), flush=True)
    L = pds.lib()
    n = int(1e8 * args.scale)
    st = torch.empty(1, dtype=torch.int32, device="cuda")
    out = torch.empty(n, dtype=torch.float64, device="cuda")
    gen = torch.Generator(device="cuda").manual_seed(1)
    w = 0.5 + 1.5 * torch.rand(n, dtype=torch.float64, device="cuda", generator=gen)
    med = {}
    for kind in SHAPES:
        y = make(torch, kind, n, gen)
        for weighted in (False, True):
            wp = w.data_ptr() if weighted else None
            ts = event_times(torch, lambda: check(L.pdsb_dev_isotonic_f64(y.data_ptr(), wp, n, 1, out.data_ptr(),
                                                                          st.data_ptr(), None)), args.repeats)
            assert st.item() == 0
            m, lo, hi = float(np.median(ts)), min(ts), max(ts)
            med[(kind, weighted)] = m
            least = 24.0 if weighted else 16.0
            design = least + 25.0 + 8.0
            print(json.dumps({"case": "pdsb_dev_isotonic_f64", "shape": kind, "weighted": weighted, "rows": n,
                              "ms_median": m * 1e3, "ms_min": lo * 1e3, "ms_max": hi * 1e3,
                              f"hbm_fraction_{int(least)}B": least * n / m / PEAK,
                              "design_bytes_per_row_max": design, "hbm_fraction_design_max": design * n / m / PEAK}),
                  flush=True)
        del y
    for weighted in (False, True):
        worst = max(SHAPES, key=lambda k: med[(k, weighted)])
        print(json.dumps({"case": "worst shape / random walk", "weighted": weighted, "worst": worst,
                          "ratio": med[(worst, weighted)] / med[("walk", weighted)]}), flush=True)
    del out, w
    torch.cuda.empty_cache()
    n = int(1e7 * args.scale)
    rng = np.random.default_rng(2)
    yh = np.cumsum(rng.standard_normal(n))
    df = pds.Frame({"y": yh})
    e = pds.isotonic_regression("y")
    ts = host_times(torch, lambda: df.select(e), args.repeats)
    print(json.dumps({"case": "isotonic_regression e2e (plugin, host columns, random walk)", "rows": n,
                      "ms_median": float(np.median(ts)) * 1e3, "ms_min": min(ts) * 1e3, "ms_max": max(ts) * 1e3}),
          flush=True)
    from scipy.optimize import isotonic_regression

    i = np.arange(n, dtype=np.float64)
    for kind, yc in (("walk", yh), ("trend", i * (4.0 / n) + rng.standard_normal(n))):
        ts = []
        for _ in range(3):
            t0 = time.perf_counter()
            isotonic_regression(yc)
            ts.append(time.perf_counter() - t0)
        print(json.dumps({"case": "scipy.optimize.isotonic_regression (CPU, one core)", "shape": kind, "rows": n,
                          "ms_median": float(np.median(ts)) * 1e3, "ms_min": min(ts) * 1e3, "ms_max": max(ts) * 1e3}),
              flush=True)


if __name__ == "__main__":
    main()
