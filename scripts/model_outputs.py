"""Record the outputs of the model paths on seeded inputs, to check that a change of their kernels leaves every bit as
it was.

    python scripts/model_outputs.py --out A.npz [--lib PATH]      # run every case, save outputs and launch counts
    python scripts/model_outputs.py --compare A.npz B.npz         # exit 1 unless both hold the same bytes

The cases: `logistic_reg` coefficients and probabilities, with and without bias, with and without nulls; `GLM.fit` and
`GLM.predict` (response and linear) for all four families on C- and F-ordered inputs; `LR.fit` / `LR.predict`;
`MixedModel.fit_df`; `rolling_lin_reg` / `recursive_lin_reg` on every pass-C kernel (see `online_cases`), with the kernel
that ran (`pdsb_last_online_path`); the predict passes and the grouped fits (see `predict_cases`).  Next to each output is the number of kernels its call launched
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
    predict_cases(res, rng)
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


def predict_cases(res, rng) -> None:
    """The predict passes and the grouped fits: K4 column-major (vector and scalar routes) and on the row-blocked frame,
    K5's grouped fit (register and generic moments kernels) and its segmented predict, K16's grouped logistic_reg and
    K17's grouped report, the plugin symbols built on them, and the f32 `moments_small` route of pl_lr with the moments
    kernel that ran (`pdsb_last_moments_path`)."""
    import pyarrow as pa
    import torch

    import polars_ds_extension_b200 as pds
    import polars_ds_extension_b200.config as cfg
    from polars_ds_extension_b200 import device as dev
    from polars_ds_extension_b200._lib import lib

    def host(v):
        if hasattr(v, "cpu"):
            return v.cpu().numpy()
        if isinstance(v, pa.ChunkedArray):
            v = v.combine_chunks()
        if isinstance(v, pa.StructArray):
            return {f.name: host(v.field(i)) for i, f in enumerate(v.type)}
        if isinstance(v, (pa.ListArray, pa.LargeListArray)):
            return {"values": host(v.flatten()), "valid": np.asarray(v.is_valid().to_numpy(zero_copy_only=False))}
        if isinstance(v, pa.Array) and (pa.types.is_string(v.type) or pa.types.is_large_string(v.type)):
            return np.asarray(v.fill_null("").to_pylist(), dtype=str)
        if isinstance(v, pa.Array):
            return {"values": np.asarray(v.fill_null(0).to_numpy(zero_copy_only=False)),
                    "valid": np.asarray(v.is_valid().to_numpy(zero_copy_only=False))}
        if isinstance(v, (list, tuple)):
            return {str(i): host(x) for i, x in enumerate(v)}
        return np.asarray(v)

    def put(tag, v):
        if isinstance(v, dict):
            for k, x in v.items():
                put(f"{tag}/{k}", x)
        else:
            res[tag] = v

    def rec(tag, fn, path=False):
        c0 = lib().pdsb_kernel_launch_count()
        v = fn()
        torch.cuda.synchronize()
        res[f"launches/{tag}"] = np.array(lib().pdsb_kernel_launch_count() - c0)
        if path:
            res[f"{tag}/moments_path"] = np.array(lib().pdsb_last_moments_path())
        put(tag, host(v))
        return v

    cuda = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a)).to(device="cuda", dtype=dt)

    # K4 column-major: X (p, ld); the scalar route reads X from an offset view, which is not 16-byte aligned
    n, p = 100_003, 7
    for dt in (torch.float32, torch.float64):
        for route in ("vec", "scalar"):
            for t in (1, 3):
                for bias in (False, True):
                    Xa = cuda(rng.standard_normal((p, n + 1)), dt)
                    X = Xa[:, 1:] if route == "scalar" else Xa[:, :n]
                    Y = cuda(rng.standard_normal((t, n)), dt)
                    beta = cuda(rng.standard_normal((t, p + bias)), torch.float64)
                    masked = bias
                    mask = cuda(rng.random(n) < 0.9, dt) if masked else None
                    w = cuda(rng.random(n) + 0.5, dt)
                    ssr = torch.zeros(8, dtype=torch.float64, device="cuda")
                    for gated in (False, True) if t == 1 and not bias else (False,):
                        status = torch.full((1,), int(gated), dtype=torch.int32, device="cuda")
                        valid = torch.zeros(n, dtype=torch.uint8, device="cuda")
                        tag = f"predict/{str(dt)[6:]}/{route}/t={t}/bias={bias}/mask={masked}/gated={gated}"
                        rec(tag, lambda: dev.predict(X, Y, beta, status, bias, mask=mask, w=w, valid=valid, ssr=ssr)
                            + (valid, ssr))

    # K4 on the frame: X before Y, Y before X, and apart
    n, p, t = 50_001, 6, 2
    Z = cuda(rng.standard_normal((p + t + 3, n)), torch.float32)
    ncols = Z.shape[0]
    frame = dev.to_frame(Z)
    for order, xcol, ycol in (("xy", 0, p), ("yx", t, 0), ("apart", 0, p + 2)):
        for masked, gated in ((False, False), (True, False), (True, True)):
            beta = cuda(rng.standard_normal((t, p + 1)), torch.float64)
            status = torch.full((1,), int(gated), dtype=torch.int32, device="cuda")
            mask = cuda(rng.random(n) < 0.9, torch.float32) if masked else None
            pred = torch.empty((t, n), dtype=torch.float32, device="cuda")
            resid = torch.empty_like(pred)
            valid = torch.zeros(n, dtype=torch.uint8, device="cuda")
            ssr = torch.zeros(8, dtype=torch.float64, device="cuda")
            rec(f"predict_frame/{order}/mask={masked}/gated={gated}",
                lambda: dev.predict_frame(frame, n, ncols, xcol, p, ycol, t, beta, status, True, pred, resid, mask=mask,
                                          valid=valid, ssr=ssr) + (valid, ssr))

    # K5: empty groups, 1-row groups, groups longer than 8192 rows, and 1e5 small groups
    sizes = np.concatenate([[0, 1, 20_000, 3, 0, 9_000, 1, 40, 8_192, 8_193], rng.integers(2, 8, 100_000), [0]])
    offs = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    n = int(offs[-1])
    for dt in (torch.float32, torch.float64):
        for p in (4, 14):
            X = cuda(rng.standard_normal((p, n)), dt)
            y = cuda(rng.standard_normal(n), dt)
            doff = cuda(offs, torch.int64)
            tag = f"grouped/{str(dt)[6:]}/p={p}"
            beta, status = rec(f"{tag}/fit", lambda: dev.grouped_lin_reg(X, y, doff, add_bias=True, l2_reg=0.01))
            mask = cuda(rng.random(n) < 0.95, dt)
            ld = (n + 4) // 4 * 4                          # a multiple of the vector width, above n
            Xa = cuda(rng.standard_normal((p, ld)), dt)
            ya = cuda(rng.standard_normal(ld), dt)
            for route, Xr, yr in (("aligned", Xa[:, :n], ya[:n]), ("unaligned", Xa[:, 1:n + 1], ya[1:n + 1])):
                rec(f"{tag}/predict/{route}", lambda: dev.grouped_predict(Xr, yr, doff, beta, status, True, mask=mask))
            # K17 (every std_err, with and without a bias, null rows as NaN, the y validity) and K16 (f64) on the same groups
            Xn = X.clone()
            Xn[0, cuda(rng.random(n) < 0.01, torch.bool)] = float("nan")
            ymask = cuda(rng.random(n) < 0.97, dt)
            for se in range(5):
                rec(f"{tag}/report/se={se}", lambda: dev.grouped_report(Xn, y, doff, add_bias=se % 2 == 0, se_type=se,
                                                                        ymask=ymask if se < 3 else None))
            if dt == torch.float64:
                yb = cuda(rng.random(n) < 0.5, dt)
                for bias in (False, True):
                    rec(f"{tag}/logistic/bias={bias}",
                        lambda: dev.grouped_logistic(X, yb, doff, add_bias=bias, l2_reg=0.05, max_iter=20,
                                                     mask=mask if bias else None))

    # the plugin symbols: pl_lr_by / pl_lr_pred_by (l1, positive, nulls under skip, one gated group), pl_lr_pred,
    # pl_lr_multi_pred, and pl_lr on the moments_small route
    f64_was = cfg.LIN_REG_EXPR_F64
    try:
        for f64 in (False, True):
            cfg.LIN_REG_EXPR_F64 = f64
            dts = "f64" if f64 else "f32"
            ng, per, p = 300, 200, 5
            n = ng * per
            X = rng.standard_normal((n, p))
            y = X @ np.linspace(-1.0, 1.0, p) + 0.1 * rng.standard_normal(n)
            g = rng.permutation(np.repeat(np.arange(ng), per))
            g[g == 7] = 8                                  # group 7 is gone; group 3 keeps 3 rows: gated with a bias
            g[np.flatnonzero(g == 3)[3:]] = 4
            cols = {f"x{j}": X[:, j] for j in range(p)} | {"y": y, "g": g}
            cols["x1"] = pa.array(X[:, 1], mask=rng.random(n) < 0.03)
            df = pds.Frame(cols)
            xs = [f"x{j}" for j in range(p)]
            for name, kw in (("ols", {}), ("l1", {"l1_reg": 0.01}), ("positive", {"positive": True}),
                             ("ridge-positive", {"l2_reg": 0.1, "positive": True})):
                kw = dict(target="y", add_bias=True, null_policy="skip", **kw)
                rec(f"plugin/{dts}/lr_by/{name}", lambda: df.group_by("g").agg(pds.lin_reg(*xs, **kw), fast=True)["coeffs"])
                e = pds.lin_reg(*xs, return_pred=True, **kw)
                rec(f"plugin/{dts}/lr_pred_by/{name}", lambda: df.evaluate(e.over("g", fast=True)))
                rec(f"plugin/{dts}/lr_pred/{name}", lambda: df.evaluate(e))
            # K17 and K16 through the plugin on the register (p = 5) and generic (p = 14) routes: nulls in a feature and in
            # y under skip, group 3's 3 rows gated
            Xw = rng.standard_normal((n, 14))
            yb = (rng.random(n) < 1.0 / (1.0 + np.exp(-Xw[:, :3].sum(1)))).astype(np.float64)
            cw = {f"x{j}": Xw[:, j] for j in range(14)} | {"y": pa.array(y, mask=rng.random(n) < 0.02), "yb": yb, "g": g}
            cw["x2"] = pa.array(Xw[:, 2], mask=rng.random(n) < 0.03)
            dw = pds.Frame(cw)
            for pw in (5, 14):
                xw = [f"x{j}" for j in range(pw)]
                for bias in (False, True):
                    for se in ("se", "hc0", "hc1", "hc2", "hc3"):
                        e = pds.lin_reg_report(*xw, target="y", add_bias=bias, null_policy="skip", std_err=se)
                        rec(f"plugin/{dts}/report_by/p={pw}/bias={bias}/{se}",
                            lambda: dw.group_by("g").agg(e, fast=True)[e.out_name or e.symbol])
                    if f64:                                # logistic_reg is f64 only
                        kw = dict(target="yb", add_bias=bias, null_policy="skip", l2_reg=0.01, tol=1e-8)
                        e = pds.logistic_reg(*xw, **kw)
                        rec(f"plugin/f64/logistic_by/p={pw}/bias={bias}",
                            lambda: dw.group_by("g").agg(e, fast=True)[e.out_name])
                        e = pds.logistic_reg(*xw, return_pred=True, **kw)
                        rec(f"plugin/f64/logistic_pred_by/p={pw}/bias={bias}", lambda: dw.evaluate(e.over("g", fast=True)))
            Y2 = np.column_stack([y, X @ np.linspace(1.0, -1.0, p)])
            dm = pds.Frame({f"x{j}": X[:, j] for j in range(p)} | {"y0": Y2[:, 0], "y1": Y2[:, 1]})
            rec(f"plugin/{dts}/lr_multi_pred",
                lambda: dm.evaluate(pds.lin_reg(*xs, target=["y0", "y1"], add_bias=True, return_pred=True)))
        cfg.LIN_REG_EXPR_F64 = False
        n = 70_000
        X = rng.standard_normal((n, 4)).astype(np.float32)
        ds = pds.Frame({f"x{j}": X[:, j] for j in range(4)} | {"y": X @ np.array([1.0, -2.0, 0.5, 3.0], np.float32)})
        rec("plugin/f32/lr/moments_small", lambda: ds.evaluate(pds.lin_reg("x0", "x1", "x2", "x3", target="y")), path=True)
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
