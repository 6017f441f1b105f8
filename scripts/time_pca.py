"""Time the PCA path on device-resident data with CUDA events, and one end-to-end principal_components call.

    python scripts/time_pca.py [--repeats R]

Cases (median and range over R timed runs after one warm-up, one JSON line each):
  * pdsb_dev_pca_f32 on a 1e8 x 32 f32 column-major matrix and pdsb_dev_pca_f64 on 5e7 x 32 (moments pass + eigen
    kernel); algorithmic bytes = n p s (one read of X);
  * pdsb_dev_project_{f32,f64} at k = 2, 8, 32 on the same matrices; algorithmic bytes = n (p s + 8 k);
  * pds.principal_components(k=2) through the plugin C ABI on 1e7 x 32 float64 host columns (host clock; includes the
    upload of the pageable Arrow buffers, both device passes and the copy back).
Each device case is reported as the fraction of the 3.35 TB/s data-sheet HBM3 bandwidth its byte count would take.  The
device name and power limit are read in the same run.  Writes nothing to disk.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from scripts.timing import PEAK, device_info, event_times, host_times  # noqa: E402


def report(case, n, p, dtype, nbytes, ts, **extra):
    med = float(np.median(ts))
    print(json.dumps({"case": case, "rows": n, "features": p, "dtype": dtype, **extra, "ms_median": med * 1e3,
                      "ms_min": min(ts) * 1e3, "ms_max": max(ts) * 1e3, "bytes": nbytes,
                      "hbm_fraction": nbytes / med / PEAK}), flush=True)


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
    p = 32
    for dtype, n in (("f32", int(1e8 * args.scale)), ("f64", int(5e7 * args.scale))):
        tt = torch.float32 if dtype == "f32" else torch.float64
        s = 4 if dtype == "f32" else 8
        g = torch.Generator(device="cuda").manual_seed(1)
        X = (torch.randn((p, n), device="cuda", dtype=tt, generator=g) *
             torch.linspace(2.0, 0.1, p, device="cuda", dtype=tt)[:, None])
        sig = torch.empty(p, dtype=torch.float64, device="cuda")
        V = torch.empty(p * p, dtype=torch.float64, device="cuda")
        st = torch.empty(2, dtype=torch.int32, device="cuda")
        fn_pca = getattr(L, f"pdsb_dev_pca_{dtype}")
        t = event_times(torch, lambda: check(fn_pca(X.data_ptr(), n, None, n, p, sig.data_ptr(), V.data_ptr(),
                                                    st.data_ptr(), None)), args.repeats)
        report(f"pdsb_dev_pca_{dtype}", n, p, dtype, n * p * s, t)
        fn_prj = getattr(L, f"pdsb_dev_project_{dtype}")
        for k in (2, 8, 32):
            out = torch.empty(n * k, dtype=torch.float64, device="cuda")
            t = event_times(torch, lambda: check(fn_prj(X.data_ptr(), n, n, p, V.data_ptr(), k, out.data_ptr(), n,
                                                        None)), args.repeats)
            report(f"pdsb_dev_project_{dtype}", n, p, dtype, n * (p * s + 8 * k), t, k=k)
            del out
        del X
        torch.cuda.empty_cache()
    n = int(1e7 * args.scale)
    rng = np.random.default_rng(2)
    df = pds.Frame({f"x{j}": rng.standard_normal(n) * (2.0 - j / 20) for j in range(p)})
    e = pds.principal_components(*[f"x{j}" for j in range(p)], k=2, center=False)
    ts = host_times(torch, lambda: df.select(e), args.repeats)
    print(json.dumps({"case": "principal_components e2e (plugin, host columns)", "rows": n, "features": p,
                      "dtype": "f64", "k": 2, "ms_median": float(np.median(ts)) * 1e3, "ms_min": min(ts) * 1e3,
                      "ms_max": max(ts) * 1e3}), flush=True)


if __name__ == "__main__":
    main()
