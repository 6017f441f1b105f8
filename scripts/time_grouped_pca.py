"""Time grouped PCA (K18): group_by(key).agg(singular_values(...)) and principal_components(...).over(key) on
device-resident data with CUDA events, each pass alone from a separate torch.profiler run, and the plugin end to end
against Polars' per-group loop.

    python scripts/time_grouped_pca.py [--repeats R] [--scale S] [--out DIR]

Cases (median and range over R timed runs after one warm-up, one JSON line each):
  * C3's shape, 1e8 rows x 8 f32 features in ~1e4 groups of ~1e4 rows: pdsb_dev_grouped_pca_f32 with center (pass 1 sums
    + pass 2 centred Gram + the eigen stage; bytes 2 p s per row), then that plus pdsb_dev_grouped_project_f32 with k = 2
    (principal_components(k=2).over; the projection reads p s and writes 8 k bytes per row);
  * 1e6 groups x 100 rows x 8 f32, center;
  * 1e3 groups x 1e3 rows x 64 f64, center;
  * a torch.profiler run over the first case (written under DIR when given): each kernel's device time per call;
  * the plugin on host columns, 1e3 groups x ~1e3 rows x 8 f32: fast=True (one pl_singular_values_by call) and Polars'
    loop (fast=False) on a 1 % slice of the groups, for scale.
Algorithmic bytes are given with their share of the 3.35 TB/s data-sheet HBM3 bandwidth.  The device name and power
limit are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from scripts.timing import PEAK, device_info, event_times, host_times, line  # noqa: E402


def frame(torch, sizes, p, dtype, seed):
    n = int(sum(sizes))
    ld = (n + 3) // 4 * 4
    gen = torch.Generator(device="cuda").manual_seed(seed)
    X = (torch.randn((p, ld), dtype=dtype, device="cuda", generator=gen) * 2.0 + 10.0)
    offsets = torch.tensor(np.concatenate([[0], np.cumsum(sizes)]), dtype=torch.int64, device="cuda")
    return X, offsets, n


def device_case(torch, dev, label, sizes, p, dtype, repeats, k=None, profile_dir=None):
    X, offsets, n = frame(torch, sizes, p, dtype, 5)
    s = X.element_size()
    ng = len(sizes)
    res = {}

    def fit():
        res["r"] = dev.grouped_pca(X, offsets, center=True, n=n)

    line(f"{label}: grouped_pca (center; sums + centred Gram + eigen)", n, ng, event_times(torch, fit, repeats),
         2 * p * s * n)
    st = res["r"][3]
    assert int((st[:, 0] != 0).sum()) == 0
    if k is not None:
        def pcs():
            mean, _, V, _ = dev.grouped_pca(X, offsets, center=True, n=n)
            dev.grouped_project(X, offsets, V, k, mean=mean, n=n)

        line(f"{label}: grouped_pca + grouped_project (k={k})", n, ng, event_times(torch, pcs, repeats),
             3 * p * s * n + 8 * k * n)
    if profile_dir is not None:
        from torch.profiler import ProfilerActivity, profile

        fit()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(repeats):
                fit()
            torch.cuda.synchronize()
        per = {}
        for ev in prof.key_averages():
            if ev.device_type.name == "CUDA" and ev.count:
                per[ev.key] = (getattr(ev, "device_time_total", getattr(ev, "cuda_time_total", 0.0)) / repeats) * 1e-3
        for name, ms in sorted(per.items(), key=lambda kv: -kv[1]):
            nb = p * s * n if ("pca_sums" in name or "pca_gram" in name) else None
            d = {"case": f"{label}: profiler, per call", "kernel": name[:90], "ms": ms}
            if nb:
                d.update({"gbytes": nb / 1e9, "hbm_fraction": nb / (ms * 1e-3) / PEAK})
            print(json.dumps(d), flush=True)
        os.makedirs(profile_dir, exist_ok=True)
        prof.export_chrome_trace(os.path.join(profile_dir, "grouped_pca_trace.json"))
    del X
    torch.cuda.empty_cache()


def main():
    import torch

    import polars_ds_extension_b200 as pds
    from polars_ds_extension_b200 import device as dev

    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--scale", type=float, default=1.0, help="fraction of the default row counts")
    ap.add_argument("--out", default=None, help="directory for the profiler trace")
    args = ap.parse_args()
    print(json.dumps(device_info(torch)), flush=True)
    rng = np.random.default_rng(6)
    sc = args.scale
    n = int(1e8 * sc)
    k = max(1, int(1e4 * sc))
    sizes = rng.integers(8000, 12001, k)
    sizes = np.maximum(1, (sizes * (n / sizes.sum())).astype(np.int64)).tolist()
    device_case(torch, dev, "C3 ~1e4 groups of ~1e4 rows x 8 f32", sizes, 8, torch.float32, args.repeats, k=2,
                profile_dir=args.out)
    device_case(torch, dev, "1e6 groups of 100 rows x 8 f32", [100] * max(1, int(1e6 * sc)), 8, torch.float32,
                args.repeats)
    device_case(torch, dev, "1e3 groups of 1e3 rows x 64 f64", [1000] * max(1, int(1e3 * sc)), 64, torch.float64,
                args.repeats)

    # the plugin on host columns: one batched call, and Polars' loop on 1 % of the groups
    ngh = max(100, int(1e3 * sc))
    gid = np.sort(rng.integers(0, ngh, ngh * 1000))
    Xh = (rng.standard_normal((len(gid), 8)) * np.linspace(3, 0.2, 8) + 5.0).astype(np.float32)
    xs = [f"x{i}" for i in range(8)]
    df = pds.Frame({x: Xh[:, i] for i, x in enumerate(xs)} | {"g": gid})
    e = pds.singular_values(*xs, center=True, as_ratio=True)

    line("group_by('g').agg(singular_values(as_ratio=True), fast=True): one pl_singular_values_by call", len(gid),
         ngh, host_times(torch, lambda: df.group_by("g").agg(e, fast=True), args.repeats))
    cut = gid < max(1, ngh // 100)
    small = df.filter(cut)
    line("group_by('g').agg(singular_values(as_ratio=True), fast=False) on 1 % of the groups: Polars' loop",
         int(cut.sum()), max(1, ngh // 100), host_times(torch, lambda: small.group_by("g").agg(e, fast=False), 1))


if __name__ == "__main__":
    main()
