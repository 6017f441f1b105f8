"""Time `MixedModel.fit_df` on 1e7 rows x 32 float64 features from a mapping of numpy columns, with 1e4 balanced
groups, with 1e5 groups of random sizes (many distinct sizes D) and with 1e6 groups of 10 rows.

    python scripts/time_mixed.py [--rows N] [--features P] [--repeats R]

Prints one JSON line per case: D, the deviance evaluations, and the median and range over R timed calls (after one
untimed call) of two times: `fit_df` as a user calls it (the Python preparation -- null handling, the dense codes, the
between test, X = [1 | features] -- plus the device fit) and the device fit alone (`pdsb_mixed_fit` on the prepared
arrays: code sort, upload, group pass, buckets, REML search, result copy).  Both are host clocks started after a device
synchronise and read after another.  The device name and power limit are read in the same run.  Writes nothing to
disk.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from scripts.timing import device_info, host_times  # noqa: E402


def data(n: int, p: int, n_groups: int, balanced: bool, rng):
    if balanced:
        sizes = np.full(n_groups, n // n_groups)
    else:
        sizes = rng.multinomial(n, rng.dirichlet(np.full(n_groups, 0.5)))
    g = rng.permutation(np.repeat(np.arange(n_groups), sizes)).astype(np.int64)
    cols = {f"x{j}": rng.standard_normal(g.size) for j in range(p)}
    y = sum(cols[f"x{j}"] * (((j % 7) - 3) / 20.0) for j in range(p))
    cols["y"] = y + rng.standard_normal(n_groups)[g] + rng.standard_normal(g.size)
    cols["g"] = g
    return cols, int(np.unique(sizes).size)


def timed(fn, repeats, torch):
    times = [t * 1e3 for t in host_times(torch, fn, repeats)]
    return {"median": float(np.median(times)), "min": min(times), "max": max(times)}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--features", type=int, default=32)
    ap.add_argument("--repeats", type=int, default=3)
    a = ap.parse_args()

    import torch

    from polars_ds_extension_b200.linear_models import MixedModel, _columns_of, _group_column, _mixed_fit, _mixed_inputs

    dev = device_info(torch)
    rng = np.random.default_rng(2024)
    feats = [f"x{j}" for j in range(a.features)]
    for name, groups, balanced in (("balanced", 10_000, True), ("random_sizes", 100_000, False),
                                   ("many_small", 1_000_000, True)):
        cols, D = data(a.rows, a.features, groups, balanced, rng)
        fit_df = timed(lambda: MixedModel().fit_df(cols, features=feats, target="y", group="g"), a.repeats, torch)
        keys, null = _group_column(cols, "g")
        X, y, codes, G, between = _mixed_inputs(_columns_of(cols, feats + ["y"]), keys, null, "skip")
        *_, evals = _mixed_fit(X, y, codes, G, between, 200, 1e-10)
        device = timed(lambda: _mixed_fit(X, y, codes, G, between, 200, 1e-10), a.repeats, torch)
        print(json.dumps({"case": name, "rows": int(codes.size), "features": a.features, "groups": groups, "D": D,
                          "evals": evals, "fit_df_ms": fit_df, "device_fit_ms": device, "gpu": dev}), flush=True)
        del cols, X, y, codes


if __name__ == "__main__":
    main()
