"""Record the outputs of the model paths on seeded inputs, to check that a change of their kernels leaves every bit as
it was.

    python scripts/model_outputs.py --out A.npz [--lib PATH]      # run every case, save outputs and launch counts
    python scripts/model_outputs.py --compare A.npz B.npz         # exit 1 unless both hold the same bytes

The cases: `logistic_reg` coefficients and probabilities, with and without bias, with and without nulls; `GLM.fit` and
`GLM.predict` (response and linear) for all four families on C- and F-ordered inputs; `LR.fit` / `LR.predict`;
`MixedModel.fit_df`; `rolling_lin_reg` / `recursive_lin_reg` on every pass-C kernel (see `online_cases`), with the kernel
that ran (`pdsb_last_online_path`).  Next to each output is the number of kernels its call launched
(`pdsb_kernel_launch_count`).
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
    online_cases(res, rng)
    np.savez(out, **res)
    print(f"{len(res)} arrays -> {out}")


def online_cases(res, rng) -> None:
    """rolling / recursive lin_reg: every pass-C kernel, both dtypes, the window lengths where the kernels branch (under
    64 rows, a direct head under half a chain, a prefix difference with a head walk, a multiple of a chain), nulls under
    skip and under a fill policy, and recursive row shards continuing from preceding moments."""
    import pyarrow as pa
    import torch

    import polars_ds_extension_b200 as pds
    import polars_ds_extension_b200.config as cfg
    from polars_ds_extension_b200 import device as dev
    from polars_ds_extension_b200._lib import lib

    def data(n, p, f64, nulls=None):
        X = rng.standard_normal((n, p))
        y = X @ (((np.arange(p) % 7) - 3) / 4.0) + 0.1 * rng.standard_normal(n) + 0.5
        if nulls == "x":
            rows = np.flatnonzero(rng.random(n) < 0.05)
            X[rows, rng.integers(0, p, rows.size)] = np.nan
        elif nulls == "y":
            y[rng.random(n) < 0.05] = np.nan
        elif nulls == "burst":
            X[1500:2300, 0] = np.nan
        dt = np.float64 if f64 else np.float32
        return X.astype(dt), y.astype(dt)

    def rec(tag, fn):
        c0 = lib().pdsb_kernel_launch_count()
        outs = fn()
        res[f"launches/{tag}"] = np.array(lib().pdsb_kernel_launch_count() - c0)
        res[f"{tag}/route"] = np.array(lib().pdsb_last_online_path())
        for k, v in zip(("coeffs", "pred", "valid"), outs):
            res[f"{tag}/{k}"] = v.cpu().numpy() if hasattr(v, "cpu") else np.asarray(v)

    def dev_call(X, y, **kw):
        dt = torch.float64 if X.dtype == np.float64 else torch.float32
        Xt = torch.from_numpy(np.ascontiguousarray(X.T)).to(device="cuda", dtype=dt)
        yt = torch.from_numpy(y).to(device="cuda", dtype=dt)
        return lambda: dev.online_lin_reg(Xt, yt, **kw)

    n = 20_011                                           # neither a multiple of 64 nor of 1024
    i = 0
    for f64 in (False, True):
        for D in (1, 8, 9, 10, 12, 13, 20):
            for window in (0, 2, 63, 64, 300, 600, 1024, 1536):
                bias = D > 1 and i % 2 == 0
                i += 1
                X, y = data(n if D < 13 else 5003, D - bias, f64)
                lam = 0.25 if window and window < 3 * D else 0.0
                rec(f"online/{'f64' if f64 else 'f32'}/D={D}/bias={bias}/w={window}",
                    dev_call(X, y, window=window, min_rows=window or D, add_bias=bias, l2_reg=lam))
    for f64, D, window, nulls in ((False, 8, 600, "x"), (False, 8, 0, "y"), (False, 9, 64, "burst"), (False, 5, 2, "x"),
                                  (False, 12, 1024, "y"), (True, 8, 300, "burst"), (True, 10, 0, "x"),
                                  (True, 13, 1536, "x"), (False, 20, 0, "burst")):
        bias = D % 2 == 0
        X, y = data(n if D < 13 else 5003, D - bias, f64, nulls)
        rec(f"online-skip/{'f64' if f64 else 'f32'}/D={D}/w={window}/{nulls}",
            dev_call(X, y, window=window, min_rows=min(window, max(D, window // 2)) if window else D, add_bias=bias,
                     l2_reg=0.1, skip=True))                # min_rows a window can reach

    # recursive row shards: the second continues the first from its (p + 2)^2 moments
    for f64 in (False, True):
        p, n0 = 8, 3000
        X, y = data(n, p, f64, "x")
        Z = np.column_stack([X, y, np.ones(n)]).astype(np.float64)[:n0]
        Z = Z[np.isfinite(Z).all(1)]
        m0 = torch.from_numpy((Z[:, :, None] * Z[:, None, :]).sum(0)).to("cuda")
        dt = torch.float64 if f64 else torch.float32
        Xt = torch.from_numpy(np.ascontiguousarray(X[n0:].T)).to(device="cuda", dtype=dt)
        yt = torch.from_numpy(y[n0:]).to(device="cuda", dtype=dt)
        for skip in (False, True):
            rec(f"online-shard/{'f64' if f64 else 'f32'}/skip={skip}",
                lambda: dev.recursive_shard(Xt, yt, 20, m0, n0, add_bias=True, l2_reg=0.01, skip=skip))

    # fill policy through the plugin: null features filled with 0.5; a null target drops its row
    f64_was = cfg.LIN_REG_EXPR_F64
    try:
        for f64 in (False, True):
            cfg.LIN_REG_EXPR_F64 = f64
            for where in ("x", "y"):
                X, y = data(5003, 4, True, where)
                cols = {f"x{j}": pa.array(X[:, j], mask=np.isnan(X[:, j])) for j in range(4)}
                cols["y"] = pa.array(y, mask=np.isnan(y))
                df = pds.Frame(cols)
                xs = [f"x{j}" for j in range(4)]
                for window in (128, 0):
                    e = (pds.rolling_lin_reg(*xs, target="y", window_size=window, add_bias=True, l2_reg=0.1,
                                             min_valid_rows=64, null_policy="0.5") if window else
                         pds.recursive_lin_reg(*xs, target="y", start_with=20, add_bias=True, l2_reg=0.1,
                                               null_policy="0.5"))

                    def plugin(e=e):
                        r = df.evaluate(e)
                        co = r.field("coeffs")
                        return (co.flatten().to_numpy(zero_copy_only=False), r.field("pred").fill_null(0.0).to_numpy(
                            zero_copy_only=False), np.asarray(co.is_valid().to_numpy(zero_copy_only=False)))
                    rec(f"online-fill/{'f64' if f64 else 'f32'}/w={window}/{where}", plugin)
    finally:
        cfg.LIN_REG_EXPR_F64 = f64_was


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
