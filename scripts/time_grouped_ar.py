"""Time group_by().agg(query_ar_coeffs(...)) on the device with CUDA events, through the plugin, and Polars' loop.

    python scripts/time_grouped_ar.py [--repeats R] [--scale S] [--loop-groups K]

Cases (median and range over R timed runs after one warm-up, one JSON line each):
  * pdsb_dev_grouped_ar_lin_reg_* on resident data, with a bias:
      - 1e4 groups x 1e4 rows, f32, lag 8;
      - the same fit as lagged columns materialised on the device (torch gathers) plus pdsb_dev_grouped_lin_reg_f32,
        timed with and without the gathers;
      - 1e6 groups x 100 rows, f32, lag 8;
      - 1e3 groups x 1e4 rows, f64, lag 32 (the generic kernel).
    Each is reported against the 3.35 TB/s data-sheet HBM3 bandwidth for the s bytes per row it reads, and against the
    data-sheet FP32 rate (67 TFLOP/s; FP64 34) for the (L+2)(L+3)/2 FMAs per row of the moments pass;
  * pl_ar_coeffs_by_f32 through the plugin C ABI on 1e3 groups x 1e4 host rows, lag 8 (host clock after a synchronise;
    includes the upload and the copy back);
  * Polars' loop (one pl_lr_f32 call per group on x.shift(i).slice(8)) on the first K of those groups, scaled up to
    1e3 groups, and labelled as scaled.
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

from scripts.timing import PEAK, device_info, event_times, host_times  # noqa: E402

FMA_PEAK = {4: 67e12 / 2, 8: 34e12 / 2}     # FMA/s: the data sheet's FP32 / FP64 (non-tensor) FLOP/s over 2


def main():
    import pyarrow as pa
    import torch

    import polars_ds_extension_b200 as pds
    from polars_ds_extension_b200 import Frame, _harness
    from polars_ds_extension_b200._lib import METHOD_LSTSQ, SolveOpts, check

    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=7)
    ap.add_argument("--scale", type=float, default=1.0, help="fraction of the default group counts")
    ap.add_argument("--loop-groups", type=int, default=50, help="groups the per-group loop is timed on")
    args = ap.parse_args()
    print(json.dumps(device_info(torch)), flush=True)
    L = pds.lib()
    gen = torch.Generator(device="cuda").manual_seed(1)
    cases = [("1e4 x 1e4", 10_000, 10_000, 8, torch.float32), ("1e6 x 100", 1_000_000, 100, 8, torch.float32),
             ("1e3 x 1e4 f64, lag 32", 1_000, 10_000, 32, torch.float64)]
    for name, G, s, lag, dt in cases:
        G = max(1, int(G * args.scale))
        n = G * s
        sfx = "f32" if dt == torch.float32 else "f64"
        esz = 4 if dt == torch.float32 else 8
        q = lag + 1
        tol = 1e-6 if dt == torch.float32 else 1e-12
        x = torch.randn(n, dtype=dt, device="cuda", generator=gen)
        offsets = torch.arange(0, n + 1, s, dtype=torch.int64, device="cuda")
        beta = torch.empty((G, q), dtype=torch.float64, device="cuda")
        status = torch.empty(G, dtype=torch.int32, device="cuda")
        o = SolveOpts(p=lag, t=1, add_bias=1, method=METHOD_LSTSQ, singular_x_tol=tol)
        fn = getattr(L, f"pdsb_dev_grouped_ar_lin_reg_{sfx}")

        def ar():
            check(fn(x.data_ptr(), None, offsets.data_ptr(), G, n, lag, C.byref(o), beta.data_ptr(), status.data_ptr(),
                     None))

        ts = event_times(torch, ar, args.repeats)
        m, lo, hi = float(np.median(ts)), min(ts), max(ts)
        assert int((status == 0).sum()) == G
        rows = G * (s - lag)
        nm = (lag + 2) * (lag + 3) // 2
        print(json.dumps({"case": f"pdsb_dev_grouped_ar_lin_reg_{sfx}", "shape": name, "groups": G, "rows": n,
                          "lag": lag, "bias": True, "ms_median": m * 1e3, "ms_min": lo * 1e3, "ms_max": hi * 1e3,
                          "bytes_per_row": esz, "hbm_fraction": n * esz / m / PEAK,
                          "fma_per_row": nm, "fma_fraction": rows * nm / m / FMA_PEAK[esz]}), flush=True)
        if name == "1e4 x 1e4":
            # the same fit on lagged columns materialised on the device: target rows t = lag .. s-1 of every group
            t = (torch.arange(s - lag, device="cuda") + lag).repeat(G) + \
                torch.arange(G, device="cuda").repeat_interleave(s - lag) * s
            so = torch.arange(0, rows + 1, s - lag, dtype=torch.int64, device="cuda")
            X = torch.empty((lag, rows), dtype=dt, device="cuda")
            y = torch.empty(rows, dtype=dt, device="cuda")
            b2 = torch.empty_like(beta)
            s2 = torch.empty_like(status)
            lr = getattr(L, f"pdsb_dev_grouped_lin_reg_{sfx}")

            def gather():
                torch.index_select(x, 0, t, out=y)
                for i in range(1, lag + 1):
                    torch.index_select(x, 0, t - i, out=X[i - 1])

            def fit():
                check(lr(X.data_ptr(), rows, y.data_ptr(), so.data_ptr(), G, rows, lag, C.byref(o), b2.data_ptr(),
                         s2.data_ptr(), None))

            gts = event_times(torch, lambda: (gather(), fit()), args.repeats)
            fts = event_times(torch, fit, args.repeats)
            gm, glo, ghi = float(np.median(gts)), min(gts), max(gts)
            fm, flo, fhi = float(np.median(fts)), min(fts), max(fts)
            same = bool(torch.equal(beta, b2) and torch.equal(status, s2))
            print(json.dumps({"case": "lagged columns gathered on the device + pdsb_dev_grouped_lin_reg_f32",
                              "groups": G, "rows": n, "lag": lag, "bit_identical_to_ar": same,
                              "ms_median": gm * 1e3, "ms_min": glo * 1e3, "ms_max": ghi * 1e3,
                              "fit_only_ms_median": fm * 1e3, "fit_only_ms_min": flo * 1e3, "fit_only_ms_max": fhi * 1e3,
                              "fit_bytes_per_row": (lag + 1) * esz,
                              "fit_only_hbm_fraction": rows * (lag + 1) * esz / fm / PEAK}), flush=True)
            del t, so, X, y, b2, s2
        del x, offsets, beta, status
        torch.cuda.empty_cache()

    G, s, lag = max(1, int(1000 * args.scale)), 10_000, 8
    rng = np.random.default_rng(2)
    xh = rng.standard_normal(G * s).astype(np.float32)
    offsets = pa.chunked_array([pa.array(np.arange(G + 1, dtype=np.int64) * s)])
    xa = pa.chunked_array([pa.array(xh)])
    import polars_ds_extension_b200.config as cfg

    cfg.LIN_REG_EXPR_F64 = False
    e = pds.query_ar_coeffs("x", lag=lag)
    kw = dict(e.kwargs, lag=lag)

    def fast():
        return _harness.call_plugin("pl_ar_coeffs_by_f32", [offsets, xa], ["__offsets__", "x"], kw)

    ts = host_times(torch, fast, args.repeats)
    print(json.dumps({"case": "pl_ar_coeffs_by_f32 e2e (plugin, host columns)", "groups": G, "rows": G * s, "lag": lag,
                      "ms_median": float(np.median(ts)) * 1e3, "ms_min": min(ts) * 1e3, "ms_max": max(ts) * 1e3}),
          flush=True)
    K = min(args.loop_groups, G)
    parts = [Frame({"x": xh[g * s:(g + 1) * s]}) for g in range(K)]
    parts[0].evaluate(e)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for part in parts:
        part.evaluate(e)
    t = time.perf_counter() - t0
    print(json.dumps({"case": "Polars' loop: pl_lr_f32 on the lagged columns once per group (scaled)",
                      "groups_timed": K, "rows_per_group": s, "ms_timed": t * 1e3,
                      "ms_scaled_to_groups": t * 1e3 * G / K, "groups": G}), flush=True)


if __name__ == "__main__":
    main()
