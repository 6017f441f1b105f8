"""Two evaluators of the same PluginExpr on the same Frame:

  * ``OracleBackend``  — the CPU oracle (oracle/lin_reg_oracle.py), the checker;
  * ``PluginBackend``  — the product: the pickled kwargs + Arrow inputs go through ``_polars_plugin_<symbol>`` in
    _polars_ds_b200.so exactly like Polars would call it (needs a GPU).

Both return the same plain-python structures so every lifted reference test can run against either.
"""
from __future__ import annotations

import numpy as np
import pyarrow as pa

from oracle import lin_reg_oracle as orc
from polars_ds_extension_b200.frame import Frame, PluginExpr


def _np_col(a: pa.ChunkedArray):
    """ChunkedArray -> oracle Col pieces (values with 0 at nulls, validity or None)."""
    arr = a.combine_chunks() if isinstance(a, pa.ChunkedArray) else a
    valid = None
    if arr.null_count:
        valid = np.asarray(arr.is_valid().to_numpy(zero_copy_only=False), dtype=bool)
        arr = arr.fill_null(False if pa.types.is_boolean(arr.type) else 0)
    return arr.to_numpy(zero_copy_only=False), valid


def _masked(pa_arr):
    arr = pa_arr
    valid = np.asarray(arr.is_valid().to_numpy(zero_copy_only=False), dtype=bool)
    vals = arr.fill_null(0).to_numpy(zero_copy_only=False)
    return vals, valid


class OracleBackend:
    name = "oracle"

    def eval(self, frame: Frame, e: PluginExpr):
        f32 = e.symbol.endswith("_f32")
        base = e.symbol[:-4] if f32 else e.symbol
        cols = []
        for a in e.args:
            vals, valid = _np_col(frame._eval_arg(a))
            cols.append(orc.Col(a.out_name, vals, valid))
        fn = getattr(orc, base)
        return fn(cols, dict(e.kwargs), f32=f32)

    def group_eval(self, frame: Frame, key: str, e: PluginExpr, fast: bool = False):
        keys = frame.columns[key].to_numpy(zero_copy_only=False)
        uniq, first = np.unique(keys, return_index=True)
        out = []
        for k in [uniq[i] for i in np.argsort(first)]:
            out.append(self.eval(frame.filter(keys == k), e))
        return out


def _list_or_none(scalar):
    v = scalar.as_py()
    return None if v is None else np.asarray(v)


class PluginBackend:
    name = "plugin"

    def eval(self, frame: Frame, e: PluginExpr):
        res = frame.evaluate(e)
        return self.normalize(e, res)

    def normalize(self, e: PluginExpr, res: pa.Array):
        f32 = e.symbol.endswith("_f32")
        base = e.symbol[:-4] if f32 else e.symbol
        if base in ("pl_lr", "pl_logistic_coeffs"):
            return _list_or_none(res[0])
        if base == "pl_logistic_pred":
            return _masked(res)
        if base == "pl_lr_pred":
            return {"pred": _masked(res.field("pred")), "resid": _masked(res.field("resid"))}
        if base == "pl_lr_multi":
            return {res.type.field(i).name: _list_or_none(res.field(i)[0]) for i in range(res.type.num_fields)}
        if base == "pl_lr_multi_pred":
            return {res.type.field(i).name: _masked(res.field(i)) for i in range(res.type.num_fields)}
        if base == "pl_lr_w_rcond":
            return {"coeffs": _list_or_none(res.field("coeffs")[0]),
                    "singular_values": _list_or_none(res.field("singular_values")[0])}
        if base in ("pl_lin_reg_report", "pl_wls_report"):
            out = {}
            for i in range(res.type.num_fields):
                nm = res.type.field(i).name
                col = res.field(i)
                if nm == "features":
                    out[nm] = col.to_pylist()
                elif nm in ("r2", "adj_r2"):
                    out[nm] = col[0].as_py()
                else:
                    out[nm] = col.to_numpy(zero_copy_only=False)
            return out
        if base in ("pl_recursive_lr", "pl_rolling_lr"):
            co = res.field("coeffs")
            valid = np.asarray(co.is_valid().to_numpy(zero_copy_only=False), dtype=bool)
            width = None
            flat = co.values.to_numpy(zero_copy_only=False)
            offs = co.offsets.to_numpy()
            coeffs = [flat[offs[i]:offs[i + 1]].copy() if valid[i] else None for i in range(len(co))]
            return {"coeffs": coeffs, "pred": _masked(res.field("pred"))}
        raise ValueError(base)

    def group_eval(self, frame: Frame, key: str, e: PluginExpr, fast: bool = False):
        r = frame.group_by(key).agg(e, fast=fast)
        res = r[e.out_name or e.symbol]
        if fast:
            return [_list_or_none(res[i]) for i in range(len(res))]
        return [self.normalize(e, x) for x in res]
