"""Record the outputs of the model paths on seeded inputs, to check that a change of their kernels leaves every bit as
it was.

    python scripts/model_outputs.py --out A.npz [--lib PATH]      # run every case, save outputs and launch counts
    python scripts/model_outputs.py --compare A.npz B.npz         # exit 1 unless both hold the same bytes

The cases: `logistic_reg` coefficients and probabilities, with and without bias, with and without nulls; `GLM.fit` and
`GLM.predict` (response and linear) for all four families on C- and F-ordered inputs; `LR.fit` / `LR.predict`;
`MixedModel.fit_df`.  Next to each output is the number of kernels its call launched (`pdsb_kernel_launch_count`).
`--lib` loads another build of the library, e.g. one of the parent commit.
"""
from __future__ import annotations

import argparse
import os
import sys
from pathlib import Path

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def run(out: str) -> None:
    import pyarrow as pa

    import polars_ds_extension_b200 as pds
    from polars_ds_extension_b200._lib import lib
    from polars_ds_extension_b200.linear_models import GLM, LR, MixedModel
    from scripts.time_glm import data as glm_data

    res = {}

    def rec(name, fn):
        c0 = lib().pdsb_kernel_launch_count()
        v = fn()
        res[f"launches/{name}"] = np.array(lib().pdsb_kernel_launch_count() - c0)
        if hasattr(v, "is_valid"):                       # an Arrow column: its values and its validity
            res[f"{name}/valid"] = np.asarray(v.is_valid().to_numpy(zero_copy_only=False))
            v = v.fill_null(0.0).to_numpy(zero_copy_only=False)
        res[name] = np.asarray(v, dtype=np.float64)

    rng = np.random.default_rng(1234)
    n, p = 300_000, 12
    X = rng.standard_normal((n, p))
    y = (rng.random(n) < 1.0 / (1.0 + np.exp(-(X @ np.linspace(-1.0, 1.0, p) + 0.3)))).astype(np.float64)
    names = [f"x{i}" for i in range(p)]
    drop = rng.random(n) < 0.05
    for nulls in (False, True):
        cols = {nm: X[:, i] for i, nm in enumerate(names)} | {"y": y}
        if nulls:
            cols["x3"] = pa.array(X[:, 3], mask=drop)
        df = pds.Frame(cols)
        for bias in (False, True):
            for l2 in (0.0, 0.05):
                tag = f"logistic/nulls={nulls}/bias={bias}/l2={l2}"
                kw = dict(target="y", add_bias=bias, l2_reg=l2, tol=1e-8)
                rec(f"{tag}/coeffs", lambda: df.evaluate(pds.logistic_reg(*names, **kw))[0].as_py())
                rec(f"{tag}/pred", lambda: df.evaluate(pds.logistic_reg(*names, return_pred=True, **kw)))

    for family in ("gaussian", "poisson", "binomial", "gamma"):
        Xg, yg = glm_data(family, 200_000, 40, rng)      # 40 columns: two column tiles in the transpose
        for order in ("C", "F"):
            Xo = np.asarray(Xg, order=order)
            for bias in (False, True):
                tag = f"glm/{family}/{order}/bias={bias}"
                m = GLM(add_bias=bias, family=family)
                rec(f"{tag}/fit", lambda: (m.fit(Xo, yg), np.append(m.coeffs(), m.bias()))[1])
                rec(f"{tag}/predict", lambda: m.predict(Xo))
                rec(f"{tag}/predict_linear", lambda: m.predict(Xo, linear=True))

    Xl = rng.standard_normal((250_000, 20))
    yl = Xl @ np.linspace(-2.0, 2.0, 20) + 0.5 + rng.standard_normal(250_000)
    for order in ("C", "F"):
        Xo = np.asarray(Xl, order=order)
        lr = LR(has_bias=True)
        rec(f"lr/{order}/fit", lambda: (lr.fit(Xo, yl), np.append(lr.coeffs(), lr.bias()))[1])
        rec(f"lr/{order}/predict", lambda: lr.predict(Xo))

    for groups, pm in ((500, 3), (20_000, 40)):
        g = rng.permutation(np.repeat(np.arange(groups), 200_000 // groups)).astype(np.int64)
        mc = {f"x{j}": rng.standard_normal(g.size) for j in range(pm)}
        mc["y"] = sum(mc[f"x{j}"] * (j % 5 - 2) / 10.0 for j in range(pm)) + rng.standard_normal(groups)[g] \
            + rng.standard_normal(g.size)
        mc["g"] = g
        mm = MixedModel()
        tag = f"mixed/groups={groups}/p={pm}"
        rec(f"{tag}/fit", lambda: (mm.fit_df(mc, features=[f"x{j}" for j in range(pm)], target="y", group="g"),
                                   np.concatenate([mm.coeffs_, mm.std_errors_, mm.dfs_,
                                                   [mm.gamma_, mm.resid_variance_]]))[1])
    np.savez(out, **res)
    print(f"{len(res)} arrays -> {out}")


def compare(a: str, b: str) -> int:
    A, B = np.load(a), np.load(b)
    bad = sorted(set(A.files) ^ set(B.files))
    for k in sorted(set(A.files) & set(B.files)):      # bytes, so -0.0 != 0.0 and NaN payloads count
        if A[k].dtype != B[k].dtype or A[k].shape != B[k].shape or A[k].tobytes() != B[k].tobytes():
            bad.append(k)
    for k in bad:
        print("DIFFERENT", k)
    print(f"{len(set(A.files) & set(B.files))} arrays compared, {len(bad)} different")
    return 1 if bad else 0


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out")
    ap.add_argument("--lib")
    ap.add_argument("--compare", nargs=2)
    a = ap.parse_args()
    if a.compare:
        sys.exit(compare(*a.compare))
    if a.lib:
        import polars_ds_extension_b200._lib as L
        L.LIB_PATH = Path(a.lib).resolve()
    run(a.out)


if __name__ == "__main__":
    main()
