"""Polars-free caller of the expression-plugin ABI.

Polars evaluates a plugin expression by exporting every input Series over the Arrow C data interface into a
``SeriesExport``, pickling the kwargs, and calling ``_polars_plugin_<symbol>`` in the shared library
(/root/reference/python/polars_ds/_utils.py:28-38 registers it).  ``call_plugin`` below does exactly that with
pyarrow arrays, so the drop-in boundary can be exercised end to end in an image that has no polars wheel.
"""
from __future__ import annotations

import ctypes as C
import pickle
from typing import Dict, List, Sequence, Union

import pyarrow as pa

from ._lib import lib, PdsbError


class ArrowSchema(C.Structure):
    pass


class ArrowArray(C.Structure):
    pass


ArrowSchema._fields_ = [
    ("format", C.c_char_p), ("name", C.c_char_p), ("metadata", C.c_char_p), ("flags", C.c_int64),
    ("n_children", C.c_int64), ("children", C.POINTER(C.POINTER(ArrowSchema))),
    ("dictionary", C.POINTER(ArrowSchema)), ("release", C.c_void_p), ("private_data", C.c_void_p),
]
ArrowArray._fields_ = [
    ("length", C.c_int64), ("null_count", C.c_int64), ("offset", C.c_int64), ("n_buffers", C.c_int64),
    ("n_children", C.c_int64), ("buffers", C.POINTER(C.c_void_p)), ("children", C.POINTER(C.POINTER(ArrowArray))),
    ("dictionary", C.POINTER(ArrowArray)), ("release", C.c_void_p), ("private_data", C.c_void_p),
]


class SeriesExport(C.Structure):
    pass


_RELEASE_T = C.CFUNCTYPE(None, C.POINTER(SeriesExport))
SeriesExport._fields_ = [
    ("field", C.POINTER(ArrowSchema)), ("arrays", C.POINTER(C.POINTER(ArrowArray))), ("len", C.c_size_t),
    ("release", _RELEASE_T), ("private_data", C.c_void_p),
]

_ARR_REL = C.CFUNCTYPE(None, C.POINTER(ArrowArray))
_SCH_REL = C.CFUNCTYPE(None, C.POINTER(ArrowSchema))


def _release_inputs_cb(se_ptr):
    """Release callback the plugin invokes once per input (it owns the inputs).

    Same contract as polars-ffi's ``c_release_series_export``: it drops the schema and the *boxes* that held the
    ArrowArrays, never the arrays themselves — the importer moved those out (``ptr::read``) and releases each through
    the array's own callback.  A plugin that relies on this callback to release the arrays leaks them; a plugin that
    does not move them out before calling it reads freed boxes under a real Polars."""
    se = se_ptr.contents
    if not se.private_data:
        return
    if se.field and se.field.contents.release:
        _SCH_REL(se.field.contents.release)(se.field)
    se.private_data = None


_RELEASE_INPUTS = _RELEASE_T(_release_inputs_cb)

ArrayLike = Union[pa.Array, pa.ChunkedArray]

_PRIM = {b"f": pa.float32(), b"g": pa.float64(), b"l": pa.int64(), b"U": pa.large_string(), b"u": pa.string()}


def _type_from_schema(s: ArrowSchema) -> pa.DataType:
    """Read (not consume) an ArrowSchema the way polars-ffi's import_field_from_c does."""
    fmt = s.format
    if fmt in _PRIM:
        return _PRIM[fmt]
    kids = [pa.field((s.children[i].contents.name or b"").decode(), _type_from_schema(s.children[i].contents))
            for i in range(s.n_children)]
    if fmt == b"+L":
        return pa.large_list(kids[0])
    if fmt == b"+s":
        return pa.struct(kids)
    raise PdsbError(f"unexpected Arrow format {fmt!r} in a plugin result")


def _chunks(a: ArrayLike) -> List[pa.Array]:
    if isinstance(a, pa.ChunkedArray):
        ch = [c for c in a.chunks]
        return ch if ch else [pa.array([], type=a.type)]
    return [a]


def call_plugin(symbol: str, inputs: Sequence[ArrayLike], names: Sequence[str], kwargs: Dict,
                raw_kwargs: bytes | None = None) -> pa.Array:
    """Call ``_polars_plugin_<symbol>`` like Polars' expression engine does and return the result as a pyarrow array.
    ``raw_kwargs`` (tests only) replaces the pickled kwargs with arbitrary bytes."""
    L = lib()
    fn = getattr(L, f"_polars_plugin_{symbol}")
    fn.restype = None
    n = len(inputs)
    exports = (SeriesExport * n)()
    keep = []
    for i, (arr, name) in enumerate(zip(inputs, names)):
        chunks = _chunks(arr)
        sch = ArrowSchema()
        pa.field(name, chunks[0].type)._export_to_c(C.addressof(sch))
        arrs = (ArrowArray * len(chunks))()
        ptrs = (C.POINTER(ArrowArray) * len(chunks))()
        for j, ch in enumerate(chunks):
            ch._export_to_c(C.addressof(arrs[j]))
            ptrs[j] = C.pointer(arrs[j])
        exports[i].field = C.pointer(sch)
        exports[i].arrays = C.cast(ptrs, C.POINTER(C.POINTER(ArrowArray)))
        exports[i].len = len(chunks)
        exports[i].release = _RELEASE_INPUTS
        exports[i].private_data = 1
        keep.append((sch, arrs, ptrs, chunks))
    payload = pickle.dumps(dict(kwargs), protocol=5) if raw_kwargs is None else bytes(raw_kwargs)
    buf = (C.c_uint8 * max(len(payload), 1)).from_buffer_copy(payload.ljust(1, b"\0"))
    ret = SeriesExport()
    fn(exports, C.c_size_t(n), buf, C.c_size_t(len(payload)), C.byref(ret), None)
    if not ret.private_data:
        msg = L._polars_plugin_get_last_error_message
        msg.restype = C.c_char_p
        raise PdsbError(f"the plugin failed with message: {msg().decode('utf-8', 'replace')}")
    try:
        if ret.len != 1:
            raise PdsbError("plugin returned an unexpected number of chunks")
        # polars-ffi import_series: `ptr::read` = bitwise copy of the ArrowArray out of its box; the box keeps a stale
        # `release` pointer, the copy is the owner.  Then the SeriesExport is dropped (its release frees boxes + schema).
        moved = ArrowArray()
        C.memmove(C.addressof(moved), C.addressof(ret.arrays[0].contents), C.sizeof(ArrowArray))
        # the field is only READ (import_field_from_c takes a reference); the export's release drops it
        out = pa.Array._import_from_c(C.addressof(moved), _type_from_schema(ret.field.contents))
    finally:
        ret.release(C.byref(ret))
    for sch_i, arrs, _ptrs, _chunks_i in keep:       # the plugin must have moved out (and released) every input chunk
        for j in range(len(arrs)):
            if arrs[j].release:
                raise PdsbError("plugin did not take ownership of an input chunk")
    del keep
    return out


def field_of(symbol: str, in_fields: Sequence[pa.Field] = ()) -> pa.Field:
    """Call the schema twin ``_polars_plugin_field_<symbol>`` with the input fields and import the declared output field."""
    L = lib()
    fn = getattr(L, f"_polars_plugin_field_{symbol}")
    fn.restype = None
    ins = (ArrowSchema * max(len(in_fields), 1))()
    for i, f in enumerate(in_fields):
        f._export_to_c(C.addressof(ins[i]))
    out = ArrowSchema()
    fn(ins if in_fields else None, C.c_size_t(len(in_fields)), C.byref(out))
    for i in range(len(in_fields)):
        if ins[i].release:
            _SCH_REL(ins[i].release)(C.byref(ins[i]))
    return pa.Field._import_from_c(C.addressof(out))


PLUGIN_SYMBOLS = [
    f"{base}{sfx}"
    for sfx in ("", "_f32")
    for base in ("pl_lr", "pl_lr_pred", "pl_lr_multi", "pl_lr_multi_pred", "pl_lr_w_rcond", "pl_lin_reg_report",
                 "pl_wls_report", "pl_recursive_lr", "pl_rolling_lr")
] + ["pl_logistic_coeffs", "pl_logistic_pred"]        # float64 only, like the reference (logistic_regression.rs:10-99)

# num_ext/pca.rs (declared in polars_plugin_num_abi.h): Float64 only, no kwargs
PCA_SYMBOLS = ["pl_singular_values", "pl_pca", "pl_principal_components"]

# num_ext/splines.rs (declared in polars_plugin_num_abi.h): Float64 inputs and output, kwargs {"lambda"}
SPLINE_SYMBOLS = ["pl_smooth_spline"]

# num_ext/isotonic_regression.rs (declared in polars_plugin_num_abi.h): Float64 inputs and output, kwargs
# {"has_weights", "increasing"}
ISOTONIC_SYMBOLS = ["pl_isotonic_regression"]

# The batched group symbols, all declared in polars_plugin_group_abi.h: every group of an over(key) or a
# group_by(key).agg(...) in one call.  Inputs [offsets (Int64), ...] in key order; the output is the single-call symbol's,
# one row per group (agg) or per input row (over).
GROUPED_SYMBOLS = [
    # group_by().agg(lin_reg): [offsets, y, features...], LRKwargs; pl_lr's List of coefficients per group
    "pl_lr_by", "pl_lr_by_f32",
    # lin_reg(return_pred=True).over(key): [offsets, y, features...], LRKwargs; pl_lr_pred's {pred, resid} per row
    "pl_lr_pred_by", "pl_lr_pred_by_f32",
    # group_by().agg(logistic_reg) and logistic_reg(return_pred=True).over(key): [offsets, y, features...], LRKwargs,
    # Float64 only; pl_logistic_coeffs's List per group and pl_logistic_pred's Float64 per row
    "pl_logistic_by", "pl_logistic_pred_by",
    # group_by().agg(lin_reg_report): [offsets, y, features...] (no var(y) input), pl_lin_reg_report's kwargs; a LargeList
    # of pl_lin_reg_report's structs per group
    "pl_lin_reg_report_by", "pl_lin_reg_report_by_f32",
    # group_by().agg(singular_values / pca) and principal_components(...).over(key): [offsets, (k: UInt32 literal),
    # features...], un-centred, kwargs {"center": bool}, Float64 only; a List of singular values or of pca structs per
    # group, or pc1..pck per row
    "pl_singular_values_by", "pl_pca_by", "pl_principal_components_by",
    # isotonic_regression(...).over(key): [offsets, y (, w)], kwargs {"has_weights", "increasing"}, Float64 only;
    # pl_isotonic_regression's Float64 per row
    "pl_isotonic_regression_by",
    # recursive_lin_reg(...).over(key): [offsets, y, features...], pl_recursive_lr's kwargs; pl_recursive_lr's
    # {coeffs, pred} per row
    "pl_recursive_lr_by", "pl_recursive_lr_by_f32",
    # group_by().agg(query_ar_coeffs(x, lag)): [offsets, x], pl_lr's kwargs plus "lag"; pl_lr(_f32)'s List of
    # coefficients per group
    "pl_ar_coeffs_by", "pl_ar_coeffs_by_f32",
    # group_by().agg(lin_reg_w_rcond): [offsets, y, features...], pl_lr_w_rcond's kwargs; a one-struct LargeList of
    # pl_lr_w_rcond's {coeffs, singular_values} per group
    "pl_lr_w_rcond_by", "pl_lr_w_rcond_by_f32",
    # group_by().agg(lin_reg(target=[...])): [offsets, target_0 .. target_{t-1}, features...], pl_lr_multi's kwargs;
    # pl_lr_multi's struct of one List per target, one row per group
    "pl_lr_multi_by", "pl_lr_multi_by_f32",
]

# The batched weighted least-squares symbols, declared in polars_plugin_wls_abi.h: group_by(key).agg(lin_reg(weights=w))
# and lin_reg(weights=w, return_pred=True).over(key) in one call.  Inputs [offsets (Int64), w, y, features...] in key
# order, pl_lr's kwargs with "weighted" set; pl_lr's List of coefficients per group and pl_lr_pred's {pred, resid} per row
WLS_GROUP_SYMBOLS = ["pl_wls_by", "pl_wls_by_f32", "pl_wls_pred_by", "pl_wls_pred_by_f32"]
