"""Time isotonic_regression(...).over(key) on the device with CUDA events, through the plugin, and Polars' loop.

    python scripts/time_grouped_isotonic.py [--repeats R] [--scale S] [--loop-groups K]

Cases (median and range over R timed runs after one warm-up, one JSON line each):
  * pdsb_dev_grouped_isotonic_f64 on resident f64 random walks (one walk per group), unweighted:
    1e4 groups x 1e4 rows, 1e6 x 100, 1e7 x 10, and 1e6 x 100 plus one 1e7-row group; with pdsb_dev_isotonic_f64 on the
    same 1e8 rows as one column for comparison.  Reported against the 3.35 TB/s data-sheet HBM3 bandwidth from the
    minimum 16 B/row (read y, write the fit);
  * pl_isotonic_regression_by through the plugin C ABI on 1e3 groups x 1e4 host rows (host clock after a synchronise;
    includes the upload and the copy back);
  * Polars' loop (one pl_isotonic_regression call per group) on the first K of those groups, scaled up to 1e3 groups.
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
    shapes = [("1e4 x 1e4", [(int(1e4 * args.scale), 10_000)]),
              ("1e6 x 100", [(int(1e6 * args.scale), 100)]),
              ("1e7 x 10", [(int(1e7 * args.scale), 10)]),
              ("1e6 x 100 + one 1e7-row group", [(int(1e6 * args.scale), 100), (1, int(1e7 * args.scale))])]
    for name, parts in shapes:
        sizes = torch.cat([torch.full((g,), s, dtype=torch.int64) for g, s in parts])
        offsets = torch.cat([torch.zeros(1, dtype=torch.int64), torch.cumsum(sizes, 0)]).cuda()
        n, G = int(offsets[-1]), sizes.numel()
        y = torch.randn(n, dtype=torch.float64, device="cuda", generator=gen)
        # one random walk per group: the cumulative sum less the value before the group's first row
        cs = torch.cumsum(y, 0)
        start = torch.repeat_interleave(torch.cat([torch.zeros(1, dtype=torch.float64, device="cuda"),
                                                   cs[offsets[1:-1] - 1]]), sizes.cuda())
        y = cs - start
        del cs, start
        out = torch.empty(n, dtype=torch.float64, device="cuda")
        st = torch.empty(G, dtype=torch.int32, device="cuda")
        ts = event_times(torch, lambda: check(L.pdsb_dev_grouped_isotonic_f64(
            y.data_ptr(), None, offsets.data_ptr(), G, n, 1, out.data_ptr(), st.data_ptr(), None)), args.repeats)
        m, lo, hi = float(np.median(ts)), min(ts), max(ts)
        assert int(st.abs().sum()) == 0
        print(json.dumps({"case": "pdsb_dev_grouped_isotonic_f64", "shape": name, "groups": G, "rows": n,
                          "ms_median": m * 1e3, "ms_min": lo * 1e3, "ms_max": hi * 1e3,
                          "hbm_fraction_16B": 16.0 * n / m / PEAK}), flush=True)
        if name == "1e4 x 1e4":
            st1 = torch.empty(1, dtype=torch.int32, device="cuda")
            ts = event_times(torch, lambda: check(L.pdsb_dev_isotonic_f64(y.data_ptr(), None, n, 1, out.data_ptr(),
                                                                          st1.data_ptr(), None)), args.repeats)
            m, lo, hi = float(np.median(ts)), min(ts), max(ts)
            print(json.dumps({"case": "pdsb_dev_isotonic_f64 on the same rows as one column", "rows": n,
                              "ms_median": m * 1e3, "ms_min": lo * 1e3, "ms_max": hi * 1e3,
                              "hbm_fraction_16B": 16.0 * n / m / PEAK}), flush=True)
        del y, out, st, offsets
        torch.cuda.empty_cache()

    G, s = 1000, 10_000
    rng = np.random.default_rng(2)
    y = np.cumsum(rng.standard_normal((G, s)), axis=1).ravel()
    offsets = pa.chunked_array([pa.array(np.arange(G + 1, dtype=np.int64) * s)])
    ya = pa.chunked_array([pa.array(y)])
    kw = {"has_weights": False, "increasing": True}

    def fast():
        return _harness.call_plugin("pl_isotonic_regression_by", [offsets, ya], ["__offsets__", "y"], kw)

    ts = host_times(torch, fast, args.repeats)
    print(json.dumps({"case": "pl_isotonic_regression_by e2e (plugin, host columns)", "groups": G, "rows": G * s,
                      "ms_median": float(np.median(ts)) * 1e3, "ms_min": min(ts) * 1e3, "ms_max": max(ts) * 1e3}),
          flush=True)
    K = min(args.loop_groups, G)
    parts = [pa.chunked_array([pa.array(y[g * s:(g + 1) * s])]) for g in range(K)]
    _harness.call_plugin("pl_isotonic_regression", [parts[0]], ["y"], kw)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for p in parts:
        _harness.call_plugin("pl_isotonic_regression", [p], ["y"], kw)
    t = time.perf_counter() - t0
    print(json.dumps({"case": "Polars' loop: pl_isotonic_regression once per group", "groups_timed": K,
                      "rows_per_group": s, "ms_timed": t * 1e3, "ms_scaled_to_groups": t * 1e3 * G / K,
                      "groups": G}), flush=True)


if __name__ == "__main__":
    main()
