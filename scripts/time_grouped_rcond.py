"""Time group_by(key).agg(lin_reg_w_rcond(...)): the batched fit on device-resident data with CUDA events, next to
pl_lr_by's device sequence (the same moments pass, then a QR solve per group) on the same frame, and the plugin end to
end against Polars' per-group loop.

    python scripts/time_grouped_rcond.py [--repeats R] [--scale S]

Cases (median and range over R timed runs after one warm-up, one JSON line each), each timed in turn with
pdsb_dev_grouped_lin_reg_rcond_* and pdsb_dev_grouped_lin_reg_* (bias, rcond 1e-6 / singular_x_tol 1e-6):
  * 1e8 rows x 8 f32 features in ~1e4 groups of ~1e4 rows, column-major: the moments pass reads (p + 1) s bytes per
    row, so the share of the 3.35 TB/s data-sheet HBM3 bandwidth is given;
  * 1e6 groups x 100 rows x 8 f32 features: the per-group solve's share grows;
  * 1e3 groups x 1e3 rows x 64 f64 features: the largest Jacobi the pass runs (q = 65).
Then group_by("g").agg(lin_reg_w_rcond(...)) through the plugin on 1e3 groups of ~1e3 rows (host columns, f32):
fast=False (one pl_lr_w_rcond_f32 call per group, Polars' loop) once, and fast=True (one pl_lr_w_rcond_by_f32 call).
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

from scripts.timing import device_info, host_times, line  # noqa: E402


def device_case(torch, L, label, sizes, p, dtype, repeats):
    from polars_ds_extension_b200._lib import METHOD_LSTSQ, METHOD_RCOND, SOLVER_QR, SolveOpts, check

    n, ng = int(sum(sizes)), len(sizes)
    s = 4 if dtype == torch.float32 else 8
    sfx = "f32" if s == 4 else "f64"
    ld = (n + 3) // 4 * 4
    gen = torch.Generator(device="cuda").manual_seed(5)
    Z = torch.randn((p + 1, ld), dtype=dtype, device="cuda", generator=gen)
    X, y = Z[:p], Z[p]
    offsets = torch.tensor(np.concatenate([[0], np.cumsum(sizes)]), dtype=torch.int64, device="cuda")
    q = p + 1
    beta = torch.empty((ng, q), dtype=torch.float64, device="cuda")
    sv = torch.empty((ng, q), dtype=torch.float64, device="cuda")
    status = torch.empty(ng, dtype=torch.int32, device="cuda")
    beta2 = torch.empty((ng, q), dtype=torch.float64, device="cuda")
    status2 = torch.empty(ng, dtype=torch.int32, device="cuda")
    orc = SolveOpts(p=p, t=1, add_bias=1, method=METHOD_RCOND, tol=1e-6)
    olr = SolveOpts(p=p, t=1, add_bias=1, method=METHOD_LSTSQ, solver=SOLVER_QR, singular_x_tol=1e-6)
    ptr = lambda t: C.c_void_p(t.data_ptr())     # noqa: E731
    rc_fn = getattr(L, f"pdsb_dev_grouped_lin_reg_rcond_{sfx}")
    lr_fn = getattr(L, f"pdsb_dev_grouped_lin_reg_{sfx}")

    def rcond():
        check(rc_fn(ptr(X), ld, ptr(y), ptr(offsets), ng, n, p, C.byref(orc), ptr(beta), ptr(sv), ptr(status), None))

    def lin_reg():
        check(lr_fn(ptr(X), ld, ptr(y), ptr(offsets), ng, n, p, C.byref(olr), ptr(beta2), ptr(status2), None))

    cases = [("pl_lr_w_rcond_by's device sequence", rcond), ("pl_lr_by's device sequence", lin_reg)]
    for _, fn in cases:      # warm-up
        fn()
    torch.cuda.synchronize()
    times = {name: [] for name, _ in cases}
    for _ in range(repeats):
        for name, fn in cases:
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fn()
            b.record()
            torch.cuda.synchronize()
            times[name].append(a.elapsed_time(b) * 1e-3)
    for name, _ in cases:
        line(f"{label}: {name}", n, ng, times[name], (p + 1) * s * n)
    assert int((status != 0).sum()) == 0 and bool(torch.isfinite(beta).all())
    diff = float((beta - beta2).abs().max() / beta2.abs().max())
    print(json.dumps({"case": f"{label}: max |beta_rcond - beta_lr| / max |beta_lr|", "value": diff}), flush=True)
    del Z
    torch.cuda.empty_cache()


def main():
    import torch

    import polars_ds_extension_b200 as pds
    import polars_ds_extension_b200.config as cfg

    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--scale", type=float, default=1.0, help="fraction of the default row counts")
    args = ap.parse_args()
    print(json.dumps(device_info(torch)), flush=True)
    L = pds.lib()
    rng = np.random.default_rng(6)
    k = max(1, int(1e4 * args.scale))
    sizes = rng.integers(8000, 12001, k)
    sizes = np.maximum(1, (sizes * (1e8 * args.scale / sizes.sum())).astype(np.int64))
    device_case(torch, L, "~1e4 groups of ~1e4 rows x 8 f32", sizes.tolist(), 8, torch.float32, args.repeats)
    device_case(torch, L, "1e6 groups of 100 rows x 8 f32", [100] * max(1, int(1e6 * args.scale)), 8, torch.float32,
                args.repeats)
    device_case(torch, L, "1e3 groups of 1e3 rows x 64 f64", [1000] * max(1, int(1e3 * args.scale)), 64, torch.float64,
                args.repeats)

    # the plugin end to end on host columns: Polars' per-group loop against one batched call
    cfg.LIN_REG_EXPR_F64 = False
    P = 8
    ngh = max(2, int(1e3 * args.scale))
    gid = np.sort(rng.integers(0, ngh, ngh * 1000))
    nh = len(gid)
    Xh = rng.standard_normal((nh, P)).astype(np.float32)
    yh = (Xh @ (np.arange(P) / P - 0.5) + 0.1 * rng.standard_normal(nh)).astype(np.float32)
    xs = [f"x{i}" for i in range(P)]
    df = pds.Frame({"y": yh} | {x: Xh[:, i] for i, x in enumerate(xs)} | {"g": gid})
    e = pds.lin_reg_w_rcond(*xs, target="y", add_bias=True, rcond=1e-6)

    ngs = len(np.unique(gid))
    line("group_by('g').agg(lin_reg_w_rcond, fast=False): one pl_lr_w_rcond_f32 call per group", nh, ngs,
         host_times(torch, lambda: df.group_by("g").agg(e, fast=False), 1))
    line("group_by('g').agg(lin_reg_w_rcond, fast=True): one pl_lr_w_rcond_by_f32 call", nh, ngs,
         host_times(torch, lambda: df.group_by("g").agg(e, fast=True), args.repeats))


if __name__ == "__main__":
    main()
