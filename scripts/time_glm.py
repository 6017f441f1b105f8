"""Time `GLM.fit` per family on 1e7 x 32 float64 from host numpy (upload, IRLS loop, result copy).

    python scripts/time_glm.py [--rows N] [--features P] [--repeats R]

Prints one JSON line per family: iterations, the median and range of the fit time over R timed fits (after an
untimed fit that counts the iterations and an untimed warm-up fit), and the device name and power limit read in the
same run.  The time is a host clock around `fit`, started after a device synchronise and read after another.  Writes
nothing to disk.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from scripts.timing import device_info, host_times  # noqa: E402


def data(family: str, n: int, p: int, rng):
    """Well-conditioned data with y in the family's domain (gamma: eta = 1 / mu > 0 on every row)."""
    if family == "gamma":
        X = rng.random((n, p))
        eta = 0.5 + X @ np.full(p, 0.05)
        return X, rng.gamma(shape=2.0, scale=(1.0 / eta) / 2.0)
    X = rng.standard_normal((n, p))
    eta = X @ (((np.arange(p) % 7) - 3) / 20.0) + 0.2
    if family == "gaussian":
        return X, eta + 0.5 * rng.standard_normal(n)
    if family == "poisson":
        return X, rng.poisson(np.exp(eta)).astype(np.float64)
    return X, (rng.random(n) < 1.0 / (1.0 + np.exp(-eta))).astype(np.float64)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--features", type=int, default=32)
    ap.add_argument("--repeats", type=int, default=3)
    a = ap.parse_args()

    import torch

    from polars_ds_extension_b200._lib import GLM_BINOMIAL, GLM_GAMMA, GLM_GAUSSIAN, GLM_POISSON
    from polars_ds_extension_b200.linear_models import _glm_fit

    dev = device_info(torch)
    rng = np.random.default_rng(2024)
    for family, fid in (("gaussian", GLM_GAUSSIAN), ("poisson", GLM_POISSON), ("binomial", GLM_BINOMIAL),
                        ("gamma", GLM_GAMMA)):
        X, y = data(family, a.rows, a.features, rng)
        y = y.reshape(-1, 1)
        _, n_iter = _glm_fit(fid, X, y, True, 100, 1e-8)
        times = [t * 1e3 for t in host_times(torch, lambda: _glm_fit(fid, X, y, True, 100, 1e-8), a.repeats)]
        print(json.dumps({"family": family, "rows": a.rows, "features": a.features, "n_iter": n_iter,
                          "fit_ms_median": float(np.median(times)), "fit_ms_min": min(times), "fit_ms_max": max(times),
                          "gpu": dev}), flush=True)
        del X, y


if __name__ == "__main__":
    main()
