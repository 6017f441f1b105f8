"""CPU-side checks of the drop-in boundary: the C-ABI library loads, exports every symbol the headers declare,
its schema twins answer without a GPU, the kwargs/pickle + Arrow import path reaches the device check and fails
LOUDLY (no CPU fallback) when there is no GPU, and the Student-t code shared with the report kernel matches scipy."""
import ctypes as C
import re
from pathlib import Path

import numpy as np
import pytest

import polars_ds_extension_b200 as pds
from polars_ds_extension_b200 import _harness
from polars_ds_extension_b200._lib import lib, LIB_PATH
from tests.helpers import has_gpu

ROOT = Path(__file__).resolve().parent.parent


def _declared_exprs(header):
    text = (ROOT / "include" / header).read_text()
    return [n for n in re.findall(r"PDSB_DECLARE_EXPR\((\w+)\)", text) if n != "name"]


def _declared_symbols():
    syms = set()
    h = (ROOT / "include" / "pdsb.h").read_text()
    syms |= set(re.findall(r"\b(pdsb_[a-z0-9_]+)\s*\(", h))
    for header in sorted(p.name for p in (ROOT / "include").glob("polars_plugin*.h")):
        for name in _declared_exprs(header):
            syms.add(f"_polars_plugin_{name}")
            syms.add(f"_polars_plugin_field_{name}")
    syms |= {"_polars_plugin_get_version", "_polars_plugin_get_last_error_message"}
    return syms


def test_library_exports_the_declared_symbols_at_their_pinned_counts():
    assert LIB_PATH.exists(), "build with python -m polars_ds_extension_b200.build"
    L = lib()
    missing = [s for s in sorted(_declared_symbols()) if not hasattr(L, s)]
    assert not missing, missing
    assert len(_declared_exprs("polars_plugin_abi.h")) == 20        # 18 lin_reg symbols + 2 logistic
    assert len(_declared_exprs("polars_plugin_group_abi.h")) == 20  # the batched group symbols
    assert len(_declared_exprs("polars_plugin_num_abi.h")) == 5     # PCA, smooth_spline, isotonic_regression
    L._polars_plugin_get_version.restype = C.c_uint32
    assert L._polars_plugin_get_version() == 1          # major 0, minor 1
    assert L.pdsb_version() == 0x000100


def test_schema_twins():
    import pyarrow as pa

    for sym in _harness.PLUGIN_SYMBOLS:
        f = _harness.field_of(sym)
        T = pa.float32() if sym.endswith("_f32") else pa.float64()
        base = sym[:-4] if sym.endswith("_f32") else sym
        if base in ("pl_lr", "pl_lr_multi", "pl_logistic_coeffs"):
            assert f.name == "coeffs" and f.type == pa.large_list(pa.field("item", T))
        elif base == "pl_logistic_pred":          # #[polars_expr(output_type=Float64)], logistic_regression.rs:50
            assert f.type == pa.float64()
        elif base in ("pl_lr_pred", "pl_lr_multi_pred"):
            assert [c.name for c in f.type] == ["pred", "resid"] and f.type.field(0).type == T
        elif base == "pl_lr_w_rcond":
            assert [c.name for c in f.type] == ["coeffs", "singular_values"]
        elif base in ("pl_lin_reg_report", "pl_wls_report"):
            assert f.name == "lin_reg_report"
            assert [c.name for c in f.type] == ["features", "beta", "std_err", "t", "p>|t|", "0.025", "0.975", "r2", "adj_r2"]
        else:
            assert [c.name for c in f.type] == ["coeffs", "pred"]


@pytest.mark.skipif(has_gpu(), reason="checks the loud failure on a box without a GPU")
def test_fails_loudly_without_gpu():
    df = pds.Frame({"x1": np.arange(10.0), "y": np.arange(10.0) * 2})
    with pytest.raises(pds.PdsbError, match="no CPU fallback"):
        df.select(pds.lin_reg("x1", target="y"))
    with pytest.raises(pds.PdsbError, match="no CPU fallback"):
        df.select(pds.rolling_lin_reg("x1", target="y", window_size=3))


def test_kwargs_validation_happens_before_compute():
    # a kwargs dict without the required serde fields is rejected by the pickle reader (LRKwargs, linear_regression.rs:27-45)
    import pyarrow as pa

    with pytest.raises(pds.PdsbError, match="missing field|no CPU fallback"):
        _harness.call_plugin("pl_lr", [pa.array([1.0, 2.0]), pa.array([1.0, 2.0])], ["y", "x"], {"bias": True})
    with pytest.raises(pds.PdsbError, match="numeric|no CPU fallback"):
        _harness.call_plugin("pl_lr", [pa.array(["a", "b"]), pa.array([1.0, 2.0])], ["y", "x"],
                             {"bias": False, "null_policy": "raise", "solver": "qr", "l1_reg": 0.0, "l2_reg": 0.0, "tol": 0.0})


def test_student_t_matches_scipy():
    from scipy import stats

    L = lib()
    for df in [1.0, 2.0, 3.5, 10.0, 30.0, 297.0, 1e4, 1e6]:
        for t in [0.0, 0.1, 1.0, 2.5, 7.0, 40.0]:
            ref = stats.t.sf(t, df)
            got = L.pdsb_student_t_sf(t, df)
            assert abs(got - ref) <= 1e-11 * max(ref, 1e-300) + 1e-300 or abs(got - ref) / ref < 1e-9, (df, t, got, ref)
        ref = stats.t.ppf(0.975, df)
        assert abs(L.pdsb_student_t_ppf(0.975, df) - ref) / ref < 1e-10, df


def test_python_wrappers_build_reference_kwargs():
    e = pds.lin_reg("a", "b", target="y", add_bias=True, l2_reg=0.1)
    assert e.symbol == "pl_lr" and [c.out_name for c in e.args] == ["y", "a", "b"] and e.args[0].cast_to == "f64"
    assert e.kwargs == {"bias": True, "null_policy": "skip", "l1_reg": 0.0, "l2_reg": 0.1, "solver": "qr", "tol": 1e-5,
                        "max_iter": 200, "weighted": False, "positive": False, "singular_x_tol": 1e-12}
    e = pds.rolling_lin_reg("a", "b", target="y", window_size=5, l2_reg=-0.2)
    assert e.kwargs == {"null_policy": "raise", "n": 5, "bias": False, "lambda": 0.2, "min_size": 2}
    e = pds.lin_reg_report("a", target="y", weights="w")
    assert e.symbol == "pl_wls_report" and [c.out_name for c in e.args] == ["w", "y", "y", "a"] and e.args[1].agg == "var"
    with pytest.raises(ValueError):
        pds.rolling_lin_reg("a", target="y", window_size=1)
    with pytest.raises(ValueError):
        pds.lin_reg("a", target=[])


def test_headers_are_plain_c(tmp_path):
    """include/*.h is the drop-in boundary: it must compile as C99 (no C++-isms), and a C program that links against
    the shared library must resolve every model / online entry point it declares."""
    import shutil
    import subprocess
    from pathlib import Path

    if shutil.which("gcc") is None:
        pytest.skip("gcc not available")
    root = Path(__file__).resolve().parents[1]
    src = tmp_path / "hdr.c"
    src.write_text('#include "pdsb.h"\n#include "polars_plugin_abi.h"\n#include "polars_plugin_num_abi.h"\n'
                   '#include "polars_plugin_group_abi.h"\n'
                   "int main(void) { pdsb_matrix m; pdsb_solve_opts o; (void)m; (void)o; return pdsb_version() < 0; }\n")
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", f"-I{root / 'include'}",
                    "-fsyntax-only", str(src)], check=True)
    so = root / "polars_ds_extension_b200" / "_polars_ds_b200.so"
    exe = tmp_path / "hdr"
    subprocess.run(["gcc", "-std=c99", f"-I{root / 'include'}", str(src), "-o", str(exe), str(so),
                    f"-Wl,-rpath,{so.parent}"], check=True)


def test_pickle_reader_survives_garbage():
    """The kwargs bytes come from another process image (Polars): truncated, bit-flipped, foreign-protocol or hostile
    payloads (huge length fields, huge memo indices) must come back as an error string, never as a crash or an
    exception unwinding through the C ABI."""
    import pickle
    import random

    import pyarrow as pa

    kw = {"bias": True, "null_policy": "skip", "solver": "qr", "l1_reg": 0.0, "l2_reg": 0.1, "tol": 1e-5,
          "max_iter": 200, "weighted": False, "positive": False, "singular_x_tol": 1e-12}
    good = pickle.dumps(kw, protocol=5)
    ins = [pa.array([1.0, 2.0, 3.0]), pa.array([1.0, 2.5, 3.0])]
    rng = random.Random(0)
    errors = 0

    def run(b):
        nonlocal errors
        try:
            _harness.call_plugin("pl_lr", ins, ["y", "x"], {}, raw_kwargs=b)
        except pds.PdsbError:
            errors += 1

    for k in range(len(good)):
        run(good[:k])
    assert errors == len(good)                       # every strict prefix is rejected
    for _ in range(1500):
        b = bytearray(good)
        for _ in range(rng.randint(1, 4)):
            b[rng.randrange(len(b))] = rng.randrange(256)
        run(bytes(b))
    hostile = [
        b"\x80\x05}\x8d" + (2 ** 63).to_bytes(8, "little") + b"x",          # BINUNICODE8 with an absurd length
        b"\x80\x05}\x8c\x01ar\xff\xff\xff\xff.",                          # LONG_BINPUT to memo slot 4e9
        b"\x80\x05}X\xff\xff\xff\x7fabc.",                                 # BINUNICODE longer than the payload
        b"\x80\x05}j\xff\xff\xff\x7f.",                                    # LONG_BINGET of a slot that does not exist
    ]
    assert hostile[0][0] == 0x80 and hostile[0][3] == 0x8d                  # real opcodes, not ASCII backslashes
    before = errors
    for h in hostile:
        run(h)
    assert errors == before + len(hostile)
    for proto in (2, 3, 4):
        run(pickle.dumps(kw, protocol=proto))        # older protocols decode as well (then stop at the device check)
    assert errors > len(good)


def test_c_client_example_builds_and_fails_loudly_without_gpu(tmp_path):
    """examples/c_client.c is the smallest non-Python consumer of the host layer; it must compile as C99 against
    include/pdsb.h, link, and — on a machine without a CUDA device — exit 2 with the library's error string."""
    import shutil
    import subprocess
    from pathlib import Path

    import torch

    if shutil.which("gcc") is None:
        pytest.skip("gcc not available")
    root = Path(__file__).resolve().parents[1]
    so = root / "polars_ds_extension_b200" / "_polars_ds_b200.so"
    exe = tmp_path / "c_client"
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", f"-I{root / 'include'}",
                    str(root / "examples" / "c_client.c"), str(so), f"-Wl,-rpath,{so.parent}", "-o", str(exe)], check=True)
    r = subprocess.run([str(exe)], capture_output=True, text=True)
    if torch.cuda.is_available():
        assert r.returncode == 0, r.stderr + r.stdout
        assert "coeffs = [2.0" in r.stdout
    else:
        assert r.returncode == 2 and "no CPU fallback" in r.stderr


def test_inputs_are_moved_and_released_like_polars_ffi():
    """polars-ffi's import_series moves every chunk out of its box (ptr::read) and releases it through the ArrowArray's
    own callback; SeriesExport::release only drops the boxes and the schema.  The harness mimics that, so a plugin that
    left the arrays to the export's release callback would leak them: the numpy buffers behind the inputs must be
    unreferenced again after the call — also on the error path (this runs without a GPU too)."""
    import gc
    import sys

    import pyarrow as pa

    y = np.arange(1000.0)
    x = np.arange(1000.0) * 0.5
    base = (sys.getrefcount(y), sys.getrefcount(x))
    ins = [pa.chunked_array([pa.array(y[:400]), pa.array(y[400:])]), pa.array(x)]
    kw = {"bias": False, "null_policy": "raise", "solver": "qr", "l1_reg": 0.0, "l2_reg": 0.0, "tol": 0.0}
    held = (sys.getrefcount(y), sys.getrefcount(x))
    assert held[0] > base[0] and held[1] > base[1]
    try:
        out = _harness.call_plugin("pl_lr", ins, ["y", "x"], kw)
        del out
    except pds.PdsbError:
        pass
    try:
        _harness.call_plugin("pl_lr", ins, ["y", "x"], {"bias": True})      # kwargs error path
    except pds.PdsbError:
        pass
    del ins
    gc.collect()
    assert (sys.getrefcount(y), sys.getrefcount(x)) == base
    L = lib()
    L.pdsb_plugin_live_results.restype = C.c_int64
    assert L.pdsb_plugin_live_results() == 0
