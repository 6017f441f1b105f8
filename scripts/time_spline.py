"""Time smooth_spline on device-resident data with CUDA events, one end-to-end plugin call, and the SciPy band solve.

    python scripts/time_spline.py [--repeats R] [--scale S]

Cases (median and range over R timed runs after one warm-up, one JSON line each):
  * pdsb_dev_smooth_spline_f64 on 1e8 resident f64 rows, evenly spaced and jittered x, lambda = 1 and 1e4.  Reported as
    the fraction of the 3.35 TB/s data-sheet HBM3 bandwidth from the algorithmic 24 B/row (read x and y, write g) and
    from the design's own byte count (pass 1 reads x, y; pass 2 reads x, y and writes g; plus the partition outputs
    and separator values of the reduced levels, written once and read once);
  * the reduced levels on their own, measured as a full solve of a system with as many unknowns as the first reduced
    level (2 (P - 1) for P = n / 32 partitions): a stand-in that bounds their cost from above;
  * pds.smooth_spline through the plugin C ABI on 1e7 f64 host rows (host clock after a synchronise; includes the upload
    of the pageable Arrow buffers and the copy back);
  * for scale, tests/spline_oracle.reinsch_f64 (scipy.linalg.solveh_banded on one CPU core) at 1e7 rows.
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

LB = 16       # blocks (2 unknowns each) per partition, as in k14_spline.cu
NF = 14       # doubles per partition output


def design_bytes(n: int) -> float:
    """Bytes the design moves for n rows: 40 B/row at level 0 plus every reduced level's scratch written and read."""
    total = 40.0 * n
    M = (n - 2 + 1) // 2
    while True:
        P = -(-M // LB)
        if P == 1:
            break
        total += 2 * 8 * (NF * P + 2 * (P - 1))
        M = P - 1
    return total


def main():
    import torch

    import polars_ds_extension_b200 as pds
    from polars_ds_extension_b200._lib import check
    from tests import spline_oracle as so

    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--scale", type=float, default=1.0, help="fraction of the default row counts")
    args = ap.parse_args()
    print(json.dumps(device_info(torch)), flush=True)
    L = pds.lib()
    n = int(1e8 * args.scale)
    st = torch.empty(1, dtype=torch.int32, device="cuda")
    gen = torch.Generator(device="cuda").manual_seed(1)
    for kind in ("even", "jitter"):
        x = torch.arange(n, dtype=torch.float64, device="cuda")          # mean spacing 1
        if kind == "jitter":
            x += (torch.rand(n, dtype=torch.float64, device="cuda", generator=gen) - 0.5) * 0.6
        y = torch.sin(x * (10.0 / n)) + 0.1 * torch.randn(n, dtype=torch.float64, device="cuda", generator=gen)
        g = torch.empty(n, dtype=torch.float64, device="cuda")
        for lam in (1.0, 1e4):
            ts = event_times(torch, lambda: check(L.pdsb_dev_smooth_spline_f64(x.data_ptr(), y.data_ptr(), n, lam,
                                                                               g.data_ptr(), st.data_ptr(), None)),
                             args.repeats)
            assert st.item() == 0
            med, lo, hi = float(np.median(ts)), min(ts), max(ts)
            db = design_bytes(n)
            print(json.dumps({"case": "pdsb_dev_smooth_spline_f64", "x": kind, "lambda": lam, "rows": n,
                              "ms_median": med * 1e3, "ms_min": lo * 1e3, "ms_max": hi * 1e3,
                              "hbm_fraction_24B": 24.0 * n / med / PEAK, "design_bytes_per_row": db / n,
                              "hbm_fraction_design": db / med / PEAK}), flush=True)
        n_red = 2 * (-(-((n - 1) // 2) // LB) - 1) + 2
        ts = event_times(torch, lambda: check(L.pdsb_dev_smooth_spline_f64(x.data_ptr(), y.data_ptr(), n_red, 1.0,
                                                                           g.data_ptr(), st.data_ptr(), None)),
                         args.repeats)
        print(json.dumps({"case": "reduced levels (stand-in: full solve at the first reduced level's size)", "x": kind,
                          "rows": n, "reduced_unknowns": n_red - 2, "ms_median": float(np.median(ts)) * 1e3,
                          "ms_min": min(ts) * 1e3, "ms_max": max(ts) * 1e3}), flush=True)
        del x, y, g
        torch.cuda.empty_cache()
    n = int(1e7 * args.scale)
    rng = np.random.default_rng(2)
    xh = np.arange(n, dtype=np.float64) + rng.uniform(-0.3, 0.3, n)
    yh = np.sin(xh * (10.0 / n)) + 0.1 * rng.standard_normal(n)
    df = pds.Frame({"x": xh, "y": yh})
    e = pds.smooth_spline("x", "y", 1.0)
    ts = host_times(torch, lambda: df.select(e), args.repeats)
    print(json.dumps({"case": "smooth_spline e2e (plugin, host columns)", "rows": n, "ms_median": float(np.median(ts)) * 1e3,
                      "ms_min": min(ts) * 1e3, "ms_max": max(ts) * 1e3}), flush=True)
    ts = []
    for _ in range(3):
        t0 = time.perf_counter()
        so.reinsch_f64(xh, yh, 1.0)
        ts.append(time.perf_counter() - t0)
    print(json.dumps({"case": "reinsch_f64 (scipy solveh_banded, CPU)", "rows": n, "ms_median": float(np.median(ts)) * 1e3,
                      "ms_min": min(ts) * 1e3, "ms_max": max(ts) * 1e3}), flush=True)


if __name__ == "__main__":
    main()
