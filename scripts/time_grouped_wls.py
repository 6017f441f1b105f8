"""Time group_by(key).agg(lin_reg(weights=w)) and lin_reg(weights=w, return_pred=True).over(key): the batched weighted
fit on device-resident data with CUDA events, next to pl_lr_by's device sequence on the same frame, and the plugin end
to end against Polars' per-group loop.

    python scripts/time_grouped_wls.py [--repeats R] [--scale S] [--loop-groups K]

Cases (median and range over R timed runs after one warm-up, one JSON line each; the two fits alternate within each
run), with a bias:
  * ~1e4 groups of ~1e4 rows x 8 f32 features: K5's register kernel;
  * 1e6 groups x 100 rows x 8 f32 features: the per-group solve's share grows;
  * 1e3 groups x 1e3 rows x 64 f64 features: K5's tile kernel;
  * fit + predict (the device sequence of lin_reg(weights=w, return_pred=True).over) at the first shape.
The weighted fit's moments pass reads (p + 2) s bytes per row, pl_lr_by's (p + 1) s; both are given with their share of
the 3.35 TB/s data-sheet HBM3 bandwidth, and the ratio of the two medians next to (p + 2) / (p + 1).  With w = 1 the two
fits must agree bit for bit, which each shape checks.
Then group_by("g").agg(lin_reg(weights=w)) through the plugin on 1e3 groups of 1e4 rows (host columns, f32): fast=True
(one pl_wls_by_f32 call), and Polars' loop (one weighted pl_lr_f32 call per group) on the first K groups, scaled to all
of them and labelled as scaled.  The device name and power limit are read in the same run.  Writes nothing to disk.
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

from scripts.timing import device_info, event_times, host_times, line  # noqa: E402


def device_case(torch, L, label, sizes, p, dtype, repeats, with_predict=False):
    from polars_ds_extension_b200._lib import METHOD_LSTSQ, SOLVER_QR, SolveOpts, check

    n, ng = int(sum(sizes)), len(sizes)
    s = 4 if dtype == torch.float32 else 8
    sfx = "f32" if s == 4 else "f64"
    ld = (n + 31) // 32 * 32
    gen = torch.Generator(device="cuda").manual_seed(5)
    Z = torch.randn((p + 1, ld), dtype=dtype, device="cuda", generator=gen)      # [x_0 .. x_{p-1} | y]
    X, y = Z[:p], Z[p]
    w = torch.rand(ld, dtype=dtype, device="cuda", generator=gen) + 0.5
    ones = torch.ones(ld, dtype=dtype, device="cuda")
    offsets = torch.tensor(np.concatenate([[0], np.cumsum(sizes)]), dtype=torch.int64, device="cuda")
    q = p + 1
    beta = torch.empty((ng, q), dtype=torch.float64, device="cuda")
    status = torch.empty(ng, dtype=torch.int32, device="cuda")
    beta1 = torch.empty_like(beta)
    status1 = torch.empty_like(status)
    # the single weighted call's settings (no ridge, no gate), and pl_lr_by's with them
    o = SolveOpts(p=p, t=1, add_bias=1, method=METHOD_LSTSQ, solver=SOLVER_QR, singular_x_tol=0.0)
    ptr = lambda a: C.c_void_p(a.data_ptr())     # noqa: E731
    wls_fn = getattr(L, f"pdsb_dev_grouped_wls_lin_reg_{sfx}")
    lr_fn = getattr(L, f"pdsb_dev_grouped_lin_reg_{sfx}")

    def wls(wt=w):
        check(wls_fn(ptr(X), ld, ptr(y), ptr(wt), ptr(offsets), ng, n, p, C.byref(o), ptr(beta), ptr(status), None))

    def by():
        check(lr_fn(ptr(X), ld, ptr(y), ptr(offsets), ng, n, p, C.byref(o), ptr(beta1), ptr(status1), None))

    cases = [("pl_wls_by's device sequence", wls, (p + 2) * s * n), ("pl_lr_by's device sequence", by, (p + 1) * s * n)]
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
    ratio = float(np.median(times[cases[0][0]]) / np.median(times[cases[1][0]]))
    wls(ones)
    torch.cuda.synchronize()
    same = bool(torch.equal(beta, beta1)) and bool(torch.equal(status, status1))
    print(json.dumps({"case": f"{label}: weighted / unweighted median", "value": ratio,
                      "bytes_ratio": (p + 2) / (p + 1), "unit_weights_bit_for_bit": same}), flush=True)
    if with_predict:
        pred = torch.empty(n, dtype=dtype, device="cuda")
        resid = torch.empty(n, dtype=dtype, device="cuda")
        valid = torch.empty(n, dtype=torch.uint8, device="cuda")

        def step():
            wls()
            check(getattr(L, f"pdsb_dev_grouped_predict_{sfx}")(ptr(X), ld, ptr(y), ptr(offsets), ng, n, p, 1, ptr(beta),
                                                                ptr(status), None, ptr(pred), ptr(resid), ptr(valid),
                                                                None))

        line(f"{label}: weighted fit + predict (the over step)", n, ng, event_times(torch, step, repeats),
             (p + 2) * s * n + (p + 1) * s * n + 2 * s * n)
    del Z, w, ones
    torch.cuda.empty_cache()


def main():
    import pyarrow as pa
    import torch

    import polars_ds_extension_b200 as pds
    import polars_ds_extension_b200.config as cfg
    from polars_ds_extension_b200 import Frame, _harness

    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--scale", type=float, default=1.0, help="fraction of the default row counts")
    ap.add_argument("--loop-groups", type=int, default=50, help="groups of Polars' loop that are timed")
    args = ap.parse_args()
    print(json.dumps(device_info(torch)), flush=True)
    L = pds.lib()
    rng = np.random.default_rng(6)
    k = max(1, int(1e4 * args.scale))
    sizes = rng.integers(8000, 12001, k)
    sizes = np.maximum(1, (sizes * (1e8 * args.scale / sizes.sum())).astype(np.int64)).tolist()
    device_case(torch, L, "~1e4 groups of ~1e4 rows x 8 f32", sizes, 8, torch.float32, args.repeats, with_predict=True)
    device_case(torch, L, "1e6 groups of 100 rows x 8 f32", [100] * max(1, int(1e6 * args.scale)), 8, torch.float32,
                args.repeats)
    device_case(torch, L, "1e3 groups of 1e3 rows x 64 f64", [1000] * max(1, int(1e3 * args.scale)), 64, torch.float64,
                args.repeats)

    # the plugin end to end on host columns: one batched call against Polars' per-group loop
    cfg.LIN_REG_EXPR_F64 = False
    P, G, m = 8, max(2, int(1e3 * args.scale)), 10_000
    Xh = rng.standard_normal((G * m, P)).astype(np.float32)
    yh = (Xh @ np.cos(np.arange(P)) + 0.1 * rng.standard_normal(G * m)).astype(np.float32)
    wh = rng.uniform(0.5, 2.0, G * m).astype(np.float32)
    xs = [f"x{i}" for i in range(P)]
    e = pds.lin_reg(*xs, target="y", add_bias=True, weights="w")
    ins = ([pa.chunked_array([pa.array(np.arange(G + 1, dtype=np.int64) * m)]), pa.chunked_array([pa.array(wh)]),
            pa.chunked_array([pa.array(yh)])] + [pa.chunked_array([pa.array(Xh[:, i])]) for i in range(P)])
    names = ["__offsets__", "w", "y"] + xs
    line("pl_wls_by_f32 e2e (plugin, host columns)", G * m, G,
         host_times(torch, lambda: _harness.call_plugin("pl_wls_by_f32", ins, names, e.kwargs), args.repeats))
    K = min(args.loop_groups, G)
    parts = [Frame({"w": wh[g * m:(g + 1) * m], "y": yh[g * m:(g + 1) * m]}
                   | {x: Xh[g * m:(g + 1) * m, i] for i, x in enumerate(xs)}) for g in range(K)]
    parts[0].evaluate(e)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for part in parts:
        part.evaluate(e)
    t = time.perf_counter() - t0
    print(json.dumps({"case": "Polars' loop: weighted pl_lr_f32 once per group (scaled)", "groups_timed": K,
                      "rows_per_group": m, "ms_timed": t * 1e3, "ms_scaled_to_groups": t * 1e3 * G / K, "groups": G}),
          flush=True)


if __name__ == "__main__":
    main()
