"""Time GLM.fit_by's device path (K16 with a GLM row rule) on device-resident data, and the loop of GLM.fit it replaces.

    python scripts/time_grouped_glm.py [--repeats R] [--scale S] [--sample G]

Cases (median and range over R timed runs after one warm-up, one JSON line each), f64 [X | y] column-major, a bias:
  * poisson, 1e4 groups of 1e4 rows, 8 features;
  * gamma, 1e4 groups of 1e4 rows, 8 features;
  * poisson, 1e6 groups of 100 rows, 8 features;
  * poisson, 1e3 groups of 1e3 rows, 64 features;
  each with the iterations the call ran, the time per iteration, the algorithmic bytes per iteration (the rows of the
  groups still running times (p + 1) * 8: pass A reads X and y once per iteration, w and z never reach memory) and the
  share of the 3.35 TB/s data-sheet HBM3 bandwidth they imply.  The running groups per iteration come from extra calls
  with max_iter = 1, 2, ... outside the timed runs.  For scale, the loop of GLM.fit (pdsb_glm_fit: upload, then per
  iteration a row pass, a moments pass, a solve and a synchronise) over G sampled groups, timed on the host and scaled
  to all groups: labelled "scaled".
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

from scripts.timing import PEAK, device_info, event_times  # noqa: E402

S = 8          # bytes per f64 value
TOL = 1e-8


def case(torch, family, n_groups, rows, p, repeats, sample):
    from polars_ds_extension_b200 import device as dev
    from polars_ds_extension_b200._lib import GLM_GAMMA, GLM_MAX_ITER, GLM_POISSON
    from polars_ds_extension_b200.linear_models import _glm_fit

    fid = {"poisson": GLM_POISSON, "gamma": GLM_GAMMA}[family]
    n = n_groups * rows
    gen = torch.Generator(device="cuda").manual_seed(7)
    X = 0.5 * torch.randn((p, n), dtype=torch.float64, device="cuda", generator=gen)
    w = torch.linspace(-0.5, 0.5, p, dtype=torch.float64, device="cuda") / max(1.0, p / 8) ** 0.5
    eta = torch.clamp(w @ X, -2.0, 2.0)
    if family == "poisson":
        y = torch.poisson(torch.exp(eta + 0.5), generator=gen)
    else:    # gamma(shape 2) with mean exp(0.3 eta): the inverse link's eta stays positive
        mean = torch.exp(0.3 * eta)
        y = torch._standard_gamma(torch.full_like(mean, 2.0), generator=gen) * mean / 2.0
    offsets = torch.arange(0, n + 1, rows, dtype=torch.int64, device="cuda")
    out = {}

    def fit(max_iter=100):
        out["r"] = dev.grouped_glm(X, y, offsets, fid, add_bias=True, tol=TOL, max_iter=max_iter)

    ts = event_times(torch, fit, repeats)
    beta, status, n_iter = out["r"]
    iters = int(n_iter.max())
    running_rows = [n]
    for k in range(1, iters):
        fit(k)
        running_rows.append(int((out["r"][1] == GLM_MAX_ITER).sum()) * rows)
    fit()
    nbytes = [r * (p + 1) * S for r in running_rows]
    m = float(np.median(ts))
    d = {"case": f"{family}: {n_groups} groups x {rows} rows x {p} features, bias", "rows": n, "groups": n_groups,
         "ms_median": m * 1e3, "ms_min": min(ts) * 1e3, "ms_max": max(ts) * 1e3, "iterations": iters,
         "ms_per_iteration": m * 1e3 / iters, "gbytes_per_iteration": [b / 1e9 for b in nbytes],
         "hbm_fraction": sum(nbytes) / m / PEAK, "converged": int((status == 0).sum())}
    # the loop of GLM.fit over `sample` groups, scaled to all of them
    picks = np.linspace(0, n_groups - 1, min(sample, n_groups)).astype(np.int64)
    Xh = [X[:, g * rows:(g + 1) * rows].T.contiguous().cpu().numpy() for g in picks]
    yh = [y[g * rows:(g + 1) * rows].cpu().numpy().reshape(-1, 1) for g in picks]
    _glm_fit(fid, Xh[0], yh[0], True, 100, TOL)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for a, b in zip(Xh, yh):
        _glm_fit(fid, a, b, True, 100, TOL)
    per_group = (time.perf_counter() - t0) / len(picks)
    d.update({"loop_sampled_groups": len(picks), "loop_ms_per_group": per_group * 1e3,
              "loop_ms_all_groups_scaled": per_group * n_groups * 1e3})
    print(json.dumps(d), flush=True)
    del X, y, eta
    torch.cuda.empty_cache()


def main():
    import torch

    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--scale", type=float, default=1.0, help="fraction of the default group counts")
    ap.add_argument("--sample", type=int, default=20, help="groups timed in the GLM.fit loop")
    args = ap.parse_args()
    print(json.dumps(device_info(torch)), flush=True)
    sc = lambda k: max(1, int(k * args.scale))      # noqa: E731
    case(torch, "poisson", sc(1e4), 10_000, 8, args.repeats, args.sample)
    case(torch, "gamma", sc(1e4), 10_000, 8, args.repeats, args.sample)
    case(torch, "poisson", sc(1e6), 100, 8, args.repeats, args.sample)
    case(torch, "poisson", sc(1e3), 1_000, 64, args.repeats, args.sample)


if __name__ == "__main__":
    main()
