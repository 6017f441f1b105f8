#!/usr/bin/env python
"""Contact with the REAL reference (polars + polars-ds 0.12.1), when a box can install it.

    python tests/golden/make_ref_fixtures.py [--log FILE] [--out tests/golden/ref_fixtures.npz]

What it does, in order, logging every step to --log (default: ref_install.log in the system temp directory):

  1. tries to make `polars` / `polars_ds` importable:  already importable -> use it;  else
     `pip install --target baseline/_ref polars polars-ds==0.12.1` from the index, then from /opt/wheelhouse
     (`--no-index --find-links`), then the reference source tree itself (needs cargo + maturin);
  2. if the import works: replays every lifted reference test of tests/cases.py with a recording backend, re-evaluates
     each recorded (frame, expression) through the real `polars_ds` plugin (register_plugin_function on the
     reference's own .so) for f64 and f32, and freezes inputs + reference outputs into --out.  tests/
     test_ref_fixtures.py then holds the oracle (CPU) and the CUDA path (GPU) to that file;
  3. also evaluates one expression through OUR .so under the real Polars (`PluginExpr.to_polars()`), which is the
     only way to verify the SeriesExport / CallerContext ABI against a real polars-ffi;
  4. if nothing installs: exits 3 after writing the reason to the log (the "parity unpinned at the Rust boundary"
     statement in DESIGN.md rests on such an attempt).

Nothing here runs in the product path or in the -m gpu tests, which need neither the reference nor a network.
"""
from __future__ import annotations

import argparse
import importlib
import os
import subprocess
import sys
import tempfile
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))
REF_DIR = ROOT / "baseline" / "_ref"


def log(fh, msg):
    line = f"[{time.strftime('%H:%M:%S')}] {msg}"
    print(line, flush=True)
    fh.write(line + "\n")
    fh.flush()


def try_import(fh):
    for extra in (None, str(REF_DIR)):
        if extra and extra not in sys.path:
            sys.path.insert(0, extra)
        try:
            importlib.invalidate_caches()
            pl = importlib.import_module("polars")
            pds = importlib.import_module("polars_ds")
            log(fh, f"import ok: polars {pl.__version__}, polars_ds {getattr(pds, '__version__', '?')} "
                    f"({Path(pds.__file__).parent})")
            return pl, pds
        except Exception as e:  # noqa: BLE001
            log(fh, f"import failed ({'sys.path' if extra is None else extra}): {type(e).__name__}: {e}")
    return None


def run(fh, cmd, timeout=900):
    log(fh, "$ " + " ".join(cmd))
    try:
        r = subprocess.run(cmd, capture_output=True, text=True, timeout=timeout)
        tail = (r.stdout + r.stderr).strip().splitlines()[-12:]
        for ln in tail:
            log(fh, "    " + ln)
        log(fh, f"    -> exit {r.returncode}")
        return r.returncode == 0
    except Exception as e:  # noqa: BLE001
        log(fh, f"    -> {type(e).__name__}: {e}")
        return False


def try_install(fh):
    REF_DIR.mkdir(parents=True, exist_ok=True)
    pip = [sys.executable, "-m", "pip", "install", "--disable-pip-version-check", "--target", str(REF_DIR)]
    attempts = [
        pip + ["--timeout", "10", "--retries", "0", "polars", "polars-ds==0.12.1"],
        pip + ["--no-index", "--find-links", "/opt/wheelhouse", "polars", "polars-ds==0.12.1"],
    ]
    if Path("/root/reference/pyproject.toml").exists():
        attempts.append(pip + ["--no-index", "--no-build-isolation", "--find-links", "/opt/wheelhouse", "/root/reference"])
    for tool in ("cargo", "rustc", "maturin"):
        r = subprocess.run(["bash", "-lc", f"command -v {tool} || echo absent"], capture_output=True, text=True)
        log(fh, f"{tool}: {r.stdout.strip()}")
    for cmd in attempts:
        if run(fh, cmd) and try_import(fh):
            return True
    return False


class Recorder:
    """Oracle backend that also records every (frame, expression) it is asked to evaluate."""

    def __init__(self):
        from tests.backends import OracleBackend

        self.inner = OracleBackend()
        self.calls = []
        self.name = "oracle"

    def eval(self, frame, e):
        self.calls.append((frame, e))
        return self.inner.eval(frame, e)

    def group_eval(self, frame, key, e, fast=False):
        return self.inner.group_eval(frame, key, e, fast=fast)


def reference_eval(pl, pds_ref, frame, e):
    """Evaluate a recorded PluginExpr with the reference's own plugin library."""
    from polars.plugins import register_plugin_function

    df = pl.from_arrow(__import__("pyarrow").table({k: v for k, v in frame.columns.items()}))

    def to_pl(c):
        x = pl.col(c.name)
        if c.cast_to:
            x = x.cast(pl.Float32 if c.cast_to == "f32" else pl.Float64)
        if c.agg == "var":
            x = x.var()
        if c.rechunked:
            x = x.rechunk()
        if c.shift_by:
            x = x.shift(c.shift_by)
        if c.slice_offset:
            x = x.slice(c.slice_offset)
        if c.alias_name:
            x = x.alias(c.alias_name)
        return x

    expr = register_plugin_function(
        plugin_path=Path(pds_ref.__file__).parent, args=[to_pl(a) for a in e.args], function_name=e.symbol,
        kwargs=e.kwargs, returns_scalar=e.returns_scalar, changes_length=e.changes_length,
        pass_name_to_apply=e.pass_name_to_apply)
    return df.select(expr.alias("out"))["out"].to_arrow()


def make_fixtures(fh, pl, pds_ref, out_path):
    import inspect
    import pickle

    import numpy as np

    import polars_ds_extension_b200.config as cfg
    from tests import cases
    from tests.backends import PluginBackend

    norm = PluginBackend().normalize
    store = {}
    n_ok = n_fail = 0
    for f64 in (True, False):
        cfg.LIN_REG_EXPR_F64 = f64
        for name, fn in inspect.getmembers(cases, inspect.isfunction):
            if not name.startswith("case_"):
                continue
            rec = Recorder()
            try:
                fn(rec)
            except Exception as e:  # noqa: BLE001  (a case may need a backend feature the recorder lacks)
                log(fh, f"  {name} ({'f64' if f64 else 'f32'}): oracle raised {type(e).__name__}: {e}")
            for k, (frame, e) in enumerate(rec.calls[:64]):
                key = f"{name}/{'f64' if f64 else 'f32'}/{k}"
                try:
                    res = norm(e, reference_eval(pl, pds_ref, frame, e))
                    store[key] = pickle.dumps({"columns": {c: v.to_pylist() for c, v in frame.columns.items()},
                                               "symbol": e.symbol, "args": e.args, "kwargs": e.kwargs, "ref": res})
                    n_ok += 1
                except Exception as ex:  # noqa: BLE001
                    store[key] = pickle.dumps({"symbol": e.symbol, "kwargs": e.kwargs, "error": f"{type(ex).__name__}: {ex}"})
                    n_fail += 1
    cfg.LIN_REG_EXPR_F64 = True
    np.savez_compressed(out_path, **{k: np.frombuffer(v, dtype=np.uint8) for k, v in store.items()})
    log(fh, f"fixtures: {n_ok} reference evaluations frozen, {n_fail} raised; wrote {out_path}")


def check_our_so_under_polars(fh, pl):
    """The ABI check proper: a real Polars dlopen()s _polars_ds_b200.so and calls pl_lr through polars-ffi."""
    import numpy as np

    import polars_ds_extension_b200 as ours

    rng = np.random.default_rng(0)
    x = rng.standard_normal((1000, 3))
    y = x @ np.array([0.5, -0.25, 1.0]) + 0.01 * rng.standard_normal(1000)
    df = pl.DataFrame({"x1": x[:, 0], "x2": x[:, 1], "x3": x[:, 2], "y": y})
    try:
        out = df.select(ours.lin_reg("x1", "x2", "x3", target="y").to_polars().alias("c"))["c"].to_list()
        log(fh, f"OUR .so under real Polars: pl_lr -> {out}")
    except Exception as e:  # noqa: BLE001
        log(fh, f"OUR .so under real Polars FAILED: {type(e).__name__}: {e}")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log", default=os.path.join(tempfile.gettempdir(), "ref_install.log"))
    ap.add_argument("--out", default=str(ROOT / "tests" / "golden" / "ref_fixtures.npz"))
    ap.add_argument("--no-install", action="store_true")
    a = ap.parse_args()
    os.makedirs(os.path.dirname(a.log), exist_ok=True)
    with open(a.log, "a") as fh:
        log(fh, f"== reference contact attempt on {os.uname().nodename}, python {sys.version.split()[0]}")
        got = try_import(fh)
        if not got and not a.no_install and try_install(fh):
            got = try_import(fh)
        if not got:
            log(fh, "RESULT: polars / polars_ds are not importable and cannot be installed on this box "
                    "(no index access, no wheels in /opt/wheelhouse, no Rust toolchain): parity stays pinned to the "
                    "reference tests' external checkers, not to outputs of the Rust binary.")
            return 3
        pl, pds_ref = got
        make_fixtures(fh, pl, pds_ref, a.out)
        check_our_so_under_polars(fh, pl)
        log(fh, "RESULT: reference fixtures generated")
        return 0


if __name__ == "__main__":
    sys.exit(main())
