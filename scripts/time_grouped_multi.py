"""Time group_by(key).agg(lin_reg(target=[...])): the batched multi-target fit on device-resident data with CUDA events,
next to t calls of pl_lr_by's device sequence (one per target) on the same frame, and the plugin end to end against
Polars' per-group loop.

    python scripts/time_grouped_multi.py [--repeats R] [--scale S]

Cases (median and range over R timed runs after one warm-up, one JSON line each; the two ways alternate within each
run), a bias and singular_x_tol 1e-6 (f32) / 1e-12 (f64):
  * ~1e4 groups of ~1e4 rows x 8 f32 features, t = 3: K5's register kernel (p + t - 1 = 10 "features");
  * the same frame with t = 8: K5's tile kernel (15 "features");
  * 1e6 groups x 100 rows x 8 f32 features, t = 3: the per-group solve's share grows;
  * 1e3 groups x 1e3 rows x 32 f64 features, t = 16: the tile kernel.
The batched fit's moments pass reads (p + t) s bytes per row, t pl_lr_by calls read t (p + 1) s; both are given, with
their share of the 3.35 TB/s data-sheet HBM3 bandwidth, and how far the two results are apart.
Then group_by("g").agg(lin_reg(target=[3 targets])) through the plugin on 1e3 groups of ~1e4 rows (host columns, f32):
fast=False (one pl_lr_multi_f32 call per group, Polars' loop) once, and fast=True (one pl_lr_multi_by_f32 call).
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


def device_case(torch, L, label, sizes, p, t, dtype, repeats):
    from polars_ds_extension_b200._lib import METHOD_LSTSQ, SOLVER_QR, SolveOpts, check

    n, ng = int(sum(sizes)), len(sizes)
    s = 4 if dtype == torch.float32 else 8
    sfx = "f32" if s == 4 else "f64"
    ld = (n + 3) // 4 * 4
    gen = torch.Generator(device="cuda").manual_seed(5)
    Z = torch.randn((t + p, ld), dtype=dtype, device="cuda", generator=gen)      # [y_0 .. y_{t-1} | x_0 .. x_{p-1}]
    X = Z[t:]
    offsets = torch.tensor(np.concatenate([[0], np.cumsum(sizes)]), dtype=torch.int64, device="cuda")
    q = p + 1
    beta = torch.empty((ng, t, q), dtype=torch.float64, device="cuda")
    status = torch.empty(ng, dtype=torch.int32, device="cuda")
    beta1 = torch.empty((t, ng, q), dtype=torch.float64, device="cuda")
    status1 = torch.empty((t, ng), dtype=torch.int32, device="cuda")
    o = SolveOpts(p=p, t=t, add_bias=1, method=METHOD_LSTSQ, solver=SOLVER_QR, singular_x_tol=1e-6 if s == 4 else 1e-12)
    o1 = SolveOpts(p=p, t=1, add_bias=1, method=METHOD_LSTSQ, solver=SOLVER_QR, singular_x_tol=o.singular_x_tol)
    ptr = lambda a: C.c_void_p(a.data_ptr())     # noqa: E731
    multi_fn = getattr(L, f"pdsb_dev_grouped_lin_reg_multi_{sfx}")
    lr_fn = getattr(L, f"pdsb_dev_grouped_lin_reg_{sfx}")

    def multi():
        check(multi_fn(ptr(Z), ld, t, p, ptr(offsets), ng, n, C.byref(o), ptr(beta), ptr(status), None))

    def per_target():
        for c in range(t):
            check(lr_fn(ptr(X), ld, ptr(Z[c]), ptr(offsets), ng, n, p, C.byref(o1), ptr(beta1[c]), ptr(status1[c]),
                        None))

    cases = [("pl_lr_multi_by's device sequence", multi, (p + t) * s * n),
             (f"{t} x pl_lr_by's device sequence", per_target, t * (p + 1) * s * n)]
    for _, fn, _ in cases:      # warm-up
        fn()
    torch.cuda.synchronize()
    times = {name: [] for name, _, _ in cases}
    for _ in range(repeats):
        for name, fn, _ in cases:
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fn()
            b.record()
            torch.cuda.synchronize()
            times[name].append(a.elapsed_time(b) * 1e-3)
    for name, _, nbytes in cases:
        line(f"{label}: {name}", n, ng, times[name], nbytes)
    assert int((status != 0).sum()) == 0 and bool(torch.isfinite(beta).all())
    ref = beta1.permute(1, 0, 2)
    diff = float((beta - ref).abs().max() / ref.abs().max())
    same = bool(torch.equal(beta, ref)) and bool(torch.equal(status, status1[0]))
    print(json.dumps({"case": f"{label}: max |beta_multi - beta_pl_lr_by| / max |beta_pl_lr_by|", "value": diff,
                      "bit_for_bit": same}), flush=True)
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
    sizes = np.maximum(1, (sizes * (1e8 * args.scale / sizes.sum())).astype(np.int64)).tolist()
    device_case(torch, L, "~1e4 groups of ~1e4 rows x 8 f32, t = 3", sizes, 8, 3, torch.float32, args.repeats)
    device_case(torch, L, "~1e4 groups of ~1e4 rows x 8 f32, t = 8", sizes, 8, 8, torch.float32, args.repeats)
    device_case(torch, L, "1e6 groups of 100 rows x 8 f32, t = 3", [100] * max(1, int(1e6 * args.scale)), 8, 3,
                torch.float32, args.repeats)
    device_case(torch, L, "1e3 groups of 1e3 rows x 32 f64, t = 16", [1000] * max(1, int(1e3 * args.scale)), 32, 16,
                torch.float64, args.repeats)

    # the plugin end to end on host columns: Polars' per-group loop against one batched call
    cfg.LIN_REG_EXPR_F64 = False
    P, T = 8, 3
    ngh = max(2, int(1e3 * args.scale))
    gid = np.sort(rng.integers(0, ngh, ngh * 10_000))
    nh = len(gid)
    Xh = rng.standard_normal((nh, P)).astype(np.float32)
    Yh = (Xh @ np.cos(np.arange(P)[:, None] + np.arange(T)[None, :]) + 0.1 * rng.standard_normal((nh, T)))
    Yh = Yh.astype(np.float32)
    xs = [f"x{i}" for i in range(P)]
    ys = [f"y{c}" for c in range(T)]
    df = pds.Frame({y: Yh[:, c] for c, y in enumerate(ys)} | {x: Xh[:, i] for i, x in enumerate(xs)} | {"g": gid})
    e = pds.lin_reg(*xs, target=ys, add_bias=True)

    ngs = len(np.unique(gid))
    line("group_by('g').agg(lin_reg(target=[3]), fast=False): one pl_lr_multi_f32 call per group", nh, ngs,
         host_times(torch, lambda: df.group_by("g").agg(e, fast=False), 1))
    line("group_by('g').agg(lin_reg(target=[3]), fast=True): one pl_lr_multi_by_f32 call", nh, ngs,
         host_times(torch, lambda: df.group_by("g").agg(e, fast=True), args.repeats))


if __name__ == "__main__":
    main()
