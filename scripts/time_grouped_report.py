"""Time group_by(key).agg(lin_reg_report(...)): the batched report on device-resident data with CUDA events, next to
lin_reg(return_pred=True).over(key)'s device sequence on the same frame, and the plugin end to end against Polars'
per-group loop.

    python scripts/time_grouped_report.py [--repeats R] [--scale S]

Cases (median and range over R timed runs after one warm-up, one JSON line each):
  * C3's shape, 1e8 rows x 8 f32 features with a bias in ~1e4 groups of ~1e4 rows, column-major.  In each repeat, in
    turn: pdsb_dev_grouped_report_f32 with std_err "se", pl_lr_pred_by's device sequence (pdsb_dev_grouped_lin_reg_f32
    then pdsb_dev_grouped_predict_f32), and pdsb_dev_grouped_report_f32 with "hc3".  Both read the frame twice; the
    report writes nothing per row, the predict pass writes pred, resid and a validity byte.  Bytes per row: report
    2 (p + 1) s; fit + predict 2 (p + 1) s + 2 s (the validity byte not counted); the share of the 3.35 TB/s data-sheet
    HBM3 bandwidth they imply.
  * group_by("g").agg(lin_reg_report(...)) through the plugin on 1e3 groups of ~1e3 rows (host columns, f32): fast=False
    (one pl_lin_reg_report_f32 call per group, Polars' loop) once, and fast=True (one pl_lin_reg_report_by_f32 call).
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

P = 8
S = 4          # bytes per f32 value


def device_cases(torch, L, sizes, repeats):
    from polars_ds_extension_b200._lib import METHOD_LSTSQ, SOLVER_QR, SolveOpts, check

    n, ng = int(sum(sizes)), len(sizes)
    ld = (n + 3) // 4 * 4
    gen = torch.Generator(device="cuda").manual_seed(5)
    Z = torch.randn((P + 1, ld), dtype=torch.float32, device="cuda", generator=gen)
    X, y = Z[:P], Z[P]
    offsets = torch.tensor(np.concatenate([[0], np.cumsum(sizes)]), dtype=torch.int64, device="cuda")
    out = torch.empty((ng, 8, P + 1), dtype=torch.float64, device="cuda")
    rstatus = torch.empty(ng, dtype=torch.int32, device="cuda")
    beta = torch.empty((ng, P + 1), dtype=torch.float64, device="cuda")
    status = torch.empty(ng, dtype=torch.int32, device="cuda")
    pred = torch.empty(ld, dtype=torch.float32, device="cuda")
    resid = torch.empty(ld, dtype=torch.float32, device="cuda")
    valid = torch.empty(ld, dtype=torch.uint8, device="cuda")
    o = SolveOpts(p=P, t=1, add_bias=1, method=METHOD_LSTSQ, solver=SOLVER_QR, singular_x_tol=1e-6)
    ptr = lambda t: C.c_void_p(t.data_ptr())     # noqa: E731

    def report(se_type):
        check(L.pdsb_dev_grouped_report_f32(ptr(X), ld, ptr(y), None, ptr(offsets), ng, n, P, 1, se_type, ptr(out),
                                            ptr(rstatus), None))

    def step():
        check(L.pdsb_dev_grouped_lin_reg_f32(ptr(X), ld, ptr(y), ptr(offsets), ng, n, P, C.byref(o), ptr(beta),
                                             ptr(status), None))
        check(L.pdsb_dev_grouped_predict_f32(ptr(X), ld, ptr(y), ptr(offsets), ng, n, P, 1, ptr(beta), ptr(status),
                                             None, ptr(pred), ptr(resid), ptr(valid), None))

    cases = [("grouped report, std_err=se", lambda: report(0), 2 * (P + 1) * S * n),
             ("fit + predict (pl_lr_pred_by's device sequence)", step, (2 * (P + 1) + 2) * S * n),
             ("grouped report, std_err=hc3", lambda: report(4), 2 * (P + 1) * S * n)]
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
        line(f"C3 ~1e4 groups of ~1e4 rows: {name}", n, ng, times[name], nbytes)
    assert int((rstatus != 0).sum()) == 0 and bool(torch.isfinite(out).all())
    del Z, pred, resid, valid
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
    n = int(1e8 * args.scale)
    k = max(1, int(1e4 * args.scale))
    sizes = rng.integers(8000, 12001, k)
    sizes = np.maximum(1, (sizes * (n / sizes.sum())).astype(np.int64))
    device_cases(torch, L, sizes.tolist(), args.repeats)

    # the plugin end to end on host columns: Polars' per-group loop against one batched call
    cfg.LIN_REG_EXPR_F64 = False
    ngh = max(2, int(1e3 * args.scale))
    gid = np.sort(rng.integers(0, ngh, ngh * 1000))
    nh = len(gid)
    Xh = rng.standard_normal((nh, P)).astype(np.float32)
    yh = (Xh @ (np.arange(P) / P - 0.5) + 0.1 * rng.standard_normal(nh)).astype(np.float32)
    xs = [f"x{i}" for i in range(P)]
    df = pds.Frame({"y": yh} | {x: Xh[:, i] for i, x in enumerate(xs)} | {"g": gid})
    e = pds.lin_reg_report(*xs, target="y", add_bias=True, std_err="hc3")

    ngs = len(np.unique(gid))
    line("group_by('g').agg(lin_reg_report(hc3), fast=False): one pl_lin_reg_report_f32 call per group", nh, ngs,
         host_times(torch, lambda: df.group_by("g").agg(e, fast=False), 1))
    line("group_by('g').agg(lin_reg_report(hc3), fast=True): one pl_lin_reg_report_by_f32 call", nh, ngs,
         host_times(torch, lambda: df.group_by("g").agg(e, fast=True), args.repeats))


if __name__ == "__main__":
    main()
