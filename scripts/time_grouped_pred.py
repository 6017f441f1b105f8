"""Time lin_reg(return_pred=True).over(key): the batched fit, the segmented predict pass and the whole step on
device-resident data with CUDA events, the plugin call end to end, and Polars' per-group loop for scale.

    python scripts/time_grouped_pred.py [--repeats R] [--scale S]

Cases (median and range over R timed runs after one warm-up, one JSON line each), f32 [X | y] column-major:
  * C3's shape, 1e8 rows x 8 features in ~1e4 groups of ~1e4 rows: pdsb_dev_grouped_lin_reg_f32 (the fit),
    pdsb_dev_grouped_predict_f32 (the predict pass) and both in a row (the step), each with its algorithmic bytes and
    the share of the 3.35 TB/s data-sheet HBM3 bandwidth they imply; next to pdsb_dev_predict_f32 on the same n x p,
    which moves the same bytes as the predict pass;
  * 1e6 groups of 100 rows, and one 5e7-row group followed by 1e5 groups of 500 rows (1e8 rows each);
  * the pl_lr_pred_by_f32 plugin call on 1e7 host rows in 1e4 groups (host clock after a synchronise: upload, fit,
    predict and copy back), and Frame.select(expr.over("g", fast=True)) on the same frame with its rows interleaved
    across groups (adds the sort by key and the inverse permutation);
  * for scale, over("g", fast=False) (one pl_lr_pred_f32 call per group, Polars' loop) and fast=True on the first 1 %
    of the rows in key order.
Bytes per row: fit (p + 1) s; predict (p + 1) s read + 2 s written (+1 validity byte, not counted); step the sum.
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

from scripts.timing import device_info, event_times, host_times, line  # noqa: E402

P = 8
S = 4          # bytes per f32 value


def device_cases(torch, L, sizes, label, repeats, with_k4):
    from polars_ds_extension_b200._lib import METHOD_LSTSQ, SOLVER_QR, SolveOpts, check

    n, ng = int(sum(sizes)), len(sizes)
    ld = (n + 3) // 4 * 4
    gen = torch.Generator(device="cuda").manual_seed(3)
    Z = torch.randn((P + 1, ld), dtype=torch.float32, device="cuda", generator=gen)
    X, y = Z[:P], Z[P]
    offsets = torch.tensor(np.concatenate([[0], np.cumsum(sizes)]), dtype=torch.int64, device="cuda")
    beta = torch.empty((ng, P + 1), dtype=torch.float64, device="cuda")
    status = torch.empty(ng, dtype=torch.int32, device="cuda")
    pred = torch.empty(ld, dtype=torch.float32, device="cuda")
    resid = torch.empty(ld, dtype=torch.float32, device="cuda")
    valid = torch.empty(ld, dtype=torch.uint8, device="cuda")
    o = SolveOpts(p=P, t=1, add_bias=1, method=METHOD_LSTSQ, solver=SOLVER_QR, singular_x_tol=1e-6)
    ptr = lambda t: C.c_void_p(t.data_ptr())     # noqa: E731

    def fit():
        check(L.pdsb_dev_grouped_lin_reg_f32(ptr(X), ld, ptr(y), ptr(offsets), ng, n, P, C.byref(o), ptr(beta),
                                             ptr(status), None))

    def predict():
        check(L.pdsb_dev_grouped_predict_f32(ptr(X), ld, ptr(y), ptr(offsets), ng, n, P, 1, ptr(beta), ptr(status), None,
                                             ptr(pred), ptr(resid), ptr(valid), None))

    def step():
        fit()
        predict()

    fit_b, pred_b = (P + 1) * S * n, (P + 3) * S * n
    line(f"{label}: grouped_lin_reg (fit)", n, ng, event_times(torch, fit, repeats), fit_b)
    line(f"{label}: grouped_predict (predict pass)", n, ng, event_times(torch, predict, repeats), pred_b)
    line(f"{label}: fit + predict (step)", n, ng, event_times(torch, step, repeats), fit_b + pred_b)
    assert int((status != 0).sum()) == 0 and bool(valid[:n].all())
    if with_k4:
        b1 = beta[:1].contiguous()
        st1 = torch.zeros(4, dtype=torch.int32, device="cuda")

        def k4():
            check(L.pdsb_dev_predict_f32(ptr(X), ld, ptr(y), ld, None, None, n, P, 1, 1, ptr(b1), ptr(st1), ptr(pred),
                                         ptr(resid), ld, ptr(valid), None, None))

        line(f"{label}: pdsb_dev_predict_f32 on the same n x p (one group)", n, 1, event_times(torch, k4, repeats),
             pred_b)
    del Z, pred, resid, valid
    torch.cuda.empty_cache()


def main():
    import pyarrow as pa
    import torch

    import polars_ds_extension_b200 as pds
    import polars_ds_extension_b200.config as cfg
    from polars_ds_extension_b200 import _harness

    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--scale", type=float, default=1.0, help="fraction of the default row counts")
    args = ap.parse_args()
    print(json.dumps(device_info(torch)), flush=True)
    L = pds.lib()
    rng = np.random.default_rng(4)
    n = int(1e8 * args.scale)
    k = max(1, int(1e4 * args.scale))
    sizes = rng.integers(8000, 12001, k)
    sizes = np.maximum(1, (sizes * (n / sizes.sum())).astype(np.int64))
    device_cases(torch, L, sizes.tolist(), "C3 ~1e4 groups of ~1e4 rows", args.repeats, True)
    device_cases(torch, L, [100] * (n // 100), "1e6 groups of 100 rows", args.repeats, False)
    device_cases(torch, L, [n // 2] + [500] * (n // 2 // 500), "one 5e7-row group + 1e5 groups of 500 rows",
                 args.repeats, False)

    # the plugin end to end on host columns
    cfg.LIN_REG_EXPR_F64 = False
    nh = int(1e7 * args.scale)
    ngh = max(1, int(1e4 * args.scale))
    gid = np.sort(rng.integers(0, ngh, nh))
    Xh = rng.standard_normal((nh, P)).astype(np.float32)
    yh = (Xh @ (np.arange(P) / P - 0.5) + 0.1 * rng.standard_normal(nh)).astype(np.float32)
    counts = np.bincount(gid, minlength=ngh)
    offs = pa.array(np.concatenate([[0], np.cumsum(counts)]).astype(np.int64))
    xs = [f"x{i}" for i in range(P)]
    e = pds.lin_reg(*xs, target="y", add_bias=True, return_pred=True)
    ins = [offs, pa.array(yh)] + [pa.array(np.ascontiguousarray(Xh[:, i])) for i in range(P)]
    names = ["__offsets__", "y"] + xs

    line("pl_lr_pred_by_f32 plugin call (host columns in key order)", nh, ngh,
         host_times(torch, lambda: _harness.call_plugin("pl_lr_pred_by_f32", ins, names, e.kwargs), args.repeats))
    perm = rng.permutation(nh)
    df = pds.Frame({"y": yh[perm]} | {x: Xh[perm, i] for i, x in enumerate(xs)} | {"g": gid[perm]})
    line("Frame.select(expr.over('g', fast=True)) (rows interleaved across groups)", nh, ngh,
         host_times(torch, lambda: df.select(e.over("g", fast=True)), args.repeats))
    cut = nh // 100          # the first 1 % of the rows in key order: ~1 % of the groups, whole
    sl = pds.Frame({"y": yh[:cut]} | {x: Xh[:cut, i] for i, x in enumerate(xs)} | {"g": gid[:cut]})
    ngs = len(np.unique(gid[:cut]))
    line("1 % slice: over('g', fast=False), one pl_lr_pred_f32 call per group", cut, ngs,
         host_times(torch, lambda: sl.select(e.over("g")), 1))
    line("1 % slice: over('g', fast=True)", cut, ngs,
         host_times(torch, lambda: sl.select(e.over("g", fast=True)), args.repeats))


if __name__ == "__main__":
    main()
