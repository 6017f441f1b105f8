"""Writes tests/golden/report_bits.npz: what pl_lin_reg_report returns, bit for bit, on seeded inputs for every std_err,
both dtypes, with and without a bias, and with skipped nulls.

The file was written with the build that came just before K9's per-row HC weight and its finalize rule moved into
shared device helpers (kernels/report_rows.h, also called by the grouped report).  tests/test_gpu_grouped_report.py
checks that the single report still returns exactly these bits.

    python tests/golden/make_report_bits.py [out.npz]      # needs a GPU
"""
import sys
from pathlib import Path

import numpy as np
import pyarrow as pa

ROOT = Path(__file__).resolve().parents[2]
STD_ERRS = ("se", "hc0", "hc1", "hc2", "hc3")
# (dtype, add_bias, null_policy): nulls are put in only for "skip"
CASES = [(dt, bias, pol) for dt in ("f64", "f32") for bias, pol in ((True, "raise"), (False, "raise"), (True, "skip"))]


def report_frame(dt: str, nulls: bool):
    """x0..x4, y: 3000 rows, seeded; with `nulls`, about 3 % nulls in x1 and y."""
    from polars_ds_extension_b200.frame import Frame

    rng = np.random.default_rng(20261017)
    n, p = 3000, 5
    X = rng.standard_normal((n, p)) + np.linspace(-0.5, 0.5, p)
    y = X @ np.linspace(-1.0, 1.0, p) + 0.7 + 0.3 * rng.standard_normal(n) * (1.0 + np.abs(X[:, 0]))
    npdt = np.float64 if dt == "f64" else np.float32
    d = {f"x{i}": X[:, i].astype(npdt) for i in range(p)}
    d["y"] = y.astype(npdt)
    if nulls:
        for c in ("x1", "y"):
            d[c] = pa.array(d[c], mask=rng.random(n) < 0.03)
    return Frame(d), [f"x{i}" for i in range(p)]


def key(dt, bias, pol, se):
    return f"{dt}_{'bias' if bias else 'nobias'}_{pol}_{se}"


def report_values(res: pa.Array) -> np.ndarray:
    """The 8 numeric fields of a report as an (8, q) array in the result's dtype."""
    return np.stack([res.field(i).to_numpy(zero_copy_only=False) for i in range(1, 9)])


def main(out: Path):
    sys.path.insert(0, str(ROOT))
    import polars_ds_extension_b200 as pds
    import polars_ds_extension_b200.config as cfg

    vals = {}
    for dt, bias, pol in CASES:
        cfg.LIN_REG_EXPR_F64 = dt == "f64"
        df, xs = report_frame(dt, pol == "skip")
        for se in STD_ERRS:
            res = df.evaluate(pds.lin_reg_report(*xs, target="y", add_bias=bias, null_policy=pol, std_err=se))
            vals[key(dt, bias, pol, se)] = report_values(res)
    np.savez(out, **vals)
    print(f"wrote {len(vals)} reports to {out}")


if __name__ == "__main__":
    main(Path(sys.argv[1]) if len(sys.argv) > 1 else Path(__file__).with_name("report_bits.npz"))
