"""A minimal, Polars-shaped frame so the plugin expressions can be evaluated without a polars wheel.

Only what the lin_reg tests of the reference need: named columns (pyarrow arrays, nulls allowed), ``select``,
``filter`` / ``slice`` / ``limit``, and ``group_by(key).agg(expr)`` which — like Polars (SURVEY.md §3.6) — gathers each
group's rows and calls the plugin symbol once per group.  ``group_by(...).agg(expr, fast=True)`` and
``expr.over(key, fast=True)`` call the expression's batched symbol instead (one launch sequence for all groups; see
``_BY_GROUP``, and ``_WLS_BY_GROUP`` for weighted lin_reg).
"""
from __future__ import annotations

from dataclasses import dataclass, field, replace
from typing import Any, Dict, List, Optional, Sequence, Tuple

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc

from . import _harness


@dataclass(frozen=True)
class ColExpr:
    """Column reference with the few transformations expr_linear.py applies (cast, var, rechunk, alias)."""
    name: str
    cast_to: Optional[str] = None      # "f32" | "f64"
    agg: Optional[str] = None          # "var"
    alias_name: Optional[str] = None
    rechunked: bool = False
    shift_by: int = 0                  # pl.Expr.shift(n): rows move down by n, nulls enter at the top
    slice_offset: int = 0              # pl.Expr.slice(offset): drop the first `offset` rows (applied after the shift)
    centered: bool = False             # e - e.mean(), the mean over the non-null values (applied last)
    lit_u32: Optional[int] = None      # pl.lit(v, dtype=pl.UInt32): a one-row UInt32 input, `name` unused

    def cast(self, dtype: str) -> "ColExpr":
        return replace(self, cast_to=dtype)

    def var(self) -> "ColExpr":
        return replace(self, agg="var")

    def alias(self, name: str) -> "ColExpr":
        return replace(self, alias_name=name)

    def rechunk(self) -> "ColExpr":
        return replace(self, rechunked=True)

    def shift(self, n: int = 1) -> "ColExpr":
        return replace(self, shift_by=self.shift_by + int(n))

    def slice(self, offset: int) -> "ColExpr":
        return replace(self, slice_offset=self.slice_offset + int(offset))

    def center(self) -> "ColExpr":
        return replace(self, centered=True)

    @property
    def out_name(self) -> str:
        return self.alias_name if self.alias_name is not None else self.name


def col(name: str) -> ColExpr:
    return ColExpr(name)


def lit_u32(v: int) -> ColExpr:
    return ColExpr("literal", lit_u32=int(v))


def _list_post(arr: pa.Array, step: str) -> pa.Array:
    """``out.list.eval(...)`` of the singular_values wrapper.  ``pl.count()`` inside ``list.eval`` counts the list's own
    elements, so the explained variance divides by (list length - 1), as the reference expression is written."""
    out = []
    for v in arr.to_pylist():
        if v is None:
            out.append(None)
            continue
        x = np.asarray(v, dtype=np.float64)
        with np.errstate(divide="ignore", invalid="ignore"):
            out.append((x ** 2 / np.float64(len(x) - 1) if step == "explained_var" else x / x.sum()).tolist())
    return pa.array(out, type=arr.type)


@dataclass
class PluginExpr:
    """What ``polars.plugins.register_plugin_function`` would capture: symbol, input expressions, kwargs, flags."""
    symbol: str
    args: List[ColExpr]
    kwargs: Optional[Dict[str, Any]]   # None: the symbol takes no kwargs (called with an empty buffer)
    returns_scalar: bool = False
    changes_length: bool = False
    pass_name_to_apply: bool = True
    out_name: str = ""
    list_post: Tuple[str, ...] = ()    # "explained_var" / "ratio": list.eval post-steps applied to the result in order
    over_key: Optional[str] = None     # pl.Expr.over(key): evaluated per group, results in the frame's row order
    over_fast: bool = False            # over(key, fast=True): one call of the batched symbol for all groups

    def alias(self, name: str) -> "PluginExpr":
        return replace(self, out_name=name)

    def over(self, key: str, fast: bool = False) -> "PluginExpr":
        """``pl.Expr.over(key)``.  ``fast=False`` calls the expression's own symbol once per group, as Polars does;
        ``fast=True`` (lin_reg or logistic_reg with ``return_pred=True``, principal_components, isotonic_regression and
        recursive_lin_reg) fits and predicts every group in one call.  A weighted lin_reg (``weights=w``) goes to the
        batched weighted least-squares symbol ``pl_wls_pred_by``."""
        if fast and _by_group(self.symbol, per_row=True) is None:
            raise ValueError("fast over is only available for lin_reg predictions (return_pred=True), "
                             "logistic_reg predictions (return_pred=True), principal_components, isotonic_regression and "
                             "recursive_lin_reg")
        return replace(self, over_key=key, over_fast=bool(fast))

    def to_polars(self):  # pragma: no cover - needs a polars wheel
        import polars as pl
        from pathlib import Path
        from polars.plugins import register_plugin_function

        def to_pl(c: ColExpr):
            if c.lit_u32 is not None:
                return pl.lit(c.lit_u32, dtype=pl.UInt32)
            e = pl.col(c.name)
            if c.cast_to:
                e = e.cast(pl.Float32 if c.cast_to == "f32" else pl.Float64)
            if c.agg == "var":
                e = e.var()
            if c.rechunked:
                e = e.rechunk()
            if c.shift_by:
                e = e.shift(c.shift_by)
            if c.slice_offset:
                e = e.slice(c.slice_offset)
            if c.centered:
                e = e - e.mean()
            if c.alias_name:
                e = e.alias(c.alias_name)
            return e

        out = register_plugin_function(
            plugin_path=Path(__file__).parent, args=[to_pl(a) for a in self.args], function_name=self.symbol,
            kwargs=self.kwargs, returns_scalar=self.returns_scalar, changes_length=self.changes_length,
            pass_name_to_apply=self.pass_name_to_apply,
        )
        for step in self.list_post:
            if step == "explained_var":
                out = out.list.eval(pl.element().pow(2) / (pl.count() - 1))
            else:
                out = out.list.eval(pl.element() / pl.element().sum())
        if self.over_key is not None:
            out = out.over(self.over_key)
        return out


def _base_symbol(symbol: str) -> str:
    return symbol[:-4] if symbol.endswith("_f32") else symbol


# fast=True: the batched symbol of each expression that has one, and whether it returns one value per row (over) or one
# per group (group_by().agg).  An `_f32` expression calls the `_f32` twin of its batched symbol.
_BY_GROUP = {
    "pl_lr": ("pl_lr_by", False),
    "pl_lr_pred": ("pl_lr_pred_by", True),
    "pl_logistic_coeffs": ("pl_logistic_by", False),
    "pl_logistic_pred": ("pl_logistic_pred_by", True),
    "pl_lin_reg_report": ("pl_lin_reg_report_by", False),
    "pl_singular_values": ("pl_singular_values_by", False),
    "pl_pca": ("pl_pca_by", False),
    "pl_principal_components": ("pl_principal_components_by", True),
    "pl_isotonic_regression": ("pl_isotonic_regression_by", True),
    "pl_recursive_lr": ("pl_recursive_lr_by", True),
    "pl_lr_w_rcond": ("pl_lr_w_rcond_by", False),
    "pl_lr_multi": ("pl_lr_multi_by", False),
}
# batched symbols that compute each group's var(y) themselves: the expression's t.var() argument is not passed
_VAR_ON_DEVICE = {"pl_lin_reg_report_by"}
# batched symbols that centre each group's columns themselves: `f - f.mean()` is per group under over / group_by, so the
# raw columns go over with kwargs {"center": bool}
_CENTER_ON_DEVICE = {"pl_singular_values_by", "pl_pca_by", "pl_principal_components_by"}


def _by_group(symbol: str, per_row: bool) -> Optional[str]:
    """The batched symbol of ``symbol`` for ``over`` (per_row) or ``group_by().agg``, or None if it has none."""
    sym, rows = _BY_GROUP.get(_base_symbol(symbol), (None, None))
    return sym if rows is per_row else None


# fast=True on a weighted lin_reg (kwargs["weighted"]): the batched weighted least-squares symbols, checked before
# _BY_GROUP, whose pl_lr_by and pl_lr_pred_by take unweighted fits only.  Same shape as _BY_GROUP.
_WLS_BY_GROUP = {
    "pl_lr": ("pl_wls_by", False),
    "pl_lr_pred": ("pl_wls_pred_by", True),
}


def _wls_by_group(e: PluginExpr, per_row: bool) -> Optional[str]:
    """The batched weighted symbol of ``e`` for ``over`` (per_row) or ``group_by().agg``, or None when ``e`` is not a
    weighted lin_reg of that kind."""
    if not e.kwargs or not e.kwargs.get("weighted"):
        return None
    sym, rows = _WLS_BY_GROUP.get(_base_symbol(e.symbol), (None, None))
    return sym if rows is per_row else None


# A shift or slice has to be taken within each group, so the batched symbols, which get whole columns in group order,
# only take the one pattern that pl_ar_coeffs_by forms on the device
_SHIFT_REFUSED = ("fast group_by / over: an argument with shift or slice is only batched as query_ar_coeffs' "
                  "autoregression (target c.slice(L), features c.shift(1).slice(L) .. c.shift(L).slice(L) of one "
                  "column c); use fast=False")


def _ar_pattern(e: PluginExpr) -> Optional[Tuple[str, Optional[str], int]]:
    """(column, the target's cast, L) when ``e`` is the unweighted lin_reg coefficients of ``c.slice(L)`` on
    ``c.shift(1).slice(L), ..., c.shift(L).slice(L)`` and nothing else (what ``query_ar_coeffs`` builds), else None."""
    if _base_symbol(e.symbol) != "pl_lr" or not e.kwargs or e.kwargs.get("weighted") or len(e.args) < 2:
        return None
    t, feats = e.args[0], e.args[1:]
    lag = len(feats)

    def plain(a: ColExpr) -> bool:
        return a.lit_u32 is None and a.agg is None and not a.centered and a.name == t.name and a.slice_offset == lag

    if not plain(t) or t.shift_by != 0:
        return None
    for i, f in enumerate(feats, 1):
        if not plain(f) or f.shift_by != i or f.cast_to not in (None, t.cast_to):
            return None
    return t.name, t.cast_to, lag


def _group_ids(keys: np.ndarray):
    """(distinct keys in first-seen order, as Polars' maintain_order=True, and each row's index into them)."""
    uniq, first, inv = np.unique(keys, return_index=True, return_inverse=True)
    order = np.argsort(first)
    rank = np.empty(len(order), dtype=np.int64)
    rank[order] = np.arange(len(order), dtype=np.int64)
    return [uniq[i] for i in order], rank[inv.reshape(-1)]


def _key_order(gid: np.ndarray, n_groups: int):
    """Rows sorted stably by group, and the offsets of each group's run in that order."""
    order = np.argsort(gid, kind="stable")
    counts = np.bincount(gid, minlength=n_groups)
    offsets = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    return order, offsets


def _to_arrow(v) -> pa.ChunkedArray:
    if isinstance(v, pa.ChunkedArray):
        return v
    if isinstance(v, pa.Array):
        return pa.chunked_array([v])
    if isinstance(v, np.ndarray):
        return pa.chunked_array([pa.array(v)])
    return pa.chunked_array([pa.array(list(v))])


def _centered(a: pa.ChunkedArray) -> pa.ChunkedArray:
    """``e - e.mean()``: Float32 stays Float32 (its mean is a Float32 scalar), every other dtype becomes Float64."""
    f32 = a.type == pa.float32()
    vals = a.drop_null().to_numpy().astype(np.float64)
    mean = vals.mean() if len(vals) else np.nan
    dt = np.float32 if f32 else np.float64
    chunks = []
    for ch in a.chunks:
        x = ch.to_numpy(zero_copy_only=False).astype(dt) if ch.null_count == 0 else \
            ch.fill_null(0).to_numpy(zero_copy_only=False).astype(dt)
        mask = None if ch.null_count == 0 else ~np.asarray(ch.is_valid().to_numpy(zero_copy_only=False), dtype=bool)
        chunks.append(pa.array(x - dt(mean), mask=mask))
    return pa.chunked_array(chunks, type=pa.float32() if f32 else pa.float64())


class Frame:
    def __init__(self, data: Dict[str, Any]):
        self.columns: Dict[str, pa.ChunkedArray] = {k: _to_arrow(v) for k, v in data.items()}
        lens = {len(v) for v in self.columns.values()}
        if len(lens) > 1:
            raise ValueError("columns have different lengths")
        self.height = lens.pop() if lens else 0

    def __len__(self) -> int:
        return self.height

    def __getitem__(self, name: str) -> pa.ChunkedArray:
        return self.columns[name]

    def with_columns(self, **cols) -> "Frame":
        d = dict(self.columns)
        d.update(cols)
        return Frame(d)

    def slice(self, offset: int, length: Optional[int] = None) -> "Frame":
        return Frame({k: v.slice(offset, length) for k, v in self.columns.items()})

    def limit(self, n: int) -> "Frame":
        return self.slice(0, n)

    def filter(self, mask) -> "Frame":
        m = pa.array(np.asarray(mask, dtype=bool))
        return Frame({k: v.filter(m) for k, v in self.columns.items()})

    def drop_nulls(self) -> "Frame":
        keep = np.ones(self.height, dtype=bool)
        for v in self.columns.values():
            keep &= np.asarray(pc.is_valid(v).to_numpy(zero_copy_only=False), dtype=bool)
        return self.filter(keep)

    # ---- expression evaluation -------------------------------------------------------------------------
    def _eval_arg(self, c: ColExpr) -> pa.ChunkedArray:
        if c.lit_u32 is not None:
            return pa.chunked_array([pa.array([c.lit_u32], type=pa.uint32())])
        a = self.columns[c.name]
        if c.cast_to:
            a = a.cast(pa.float32() if c.cast_to == "f32" else pa.float64())
        if c.agg == "var":
            vals = a.drop_null().to_numpy()
            v = float(np.var(vals.astype(np.float64), ddof=1)) if len(vals) > 1 else None
            a = pa.chunked_array([pa.array([v], type=a.type)])
        if c.rechunked:
            a = pa.chunked_array([a.combine_chunks()]) if a.num_chunks != 1 else a
        if c.shift_by:
            k = c.shift_by
            if k < 0:
                raise ValueError("only forward shifts are needed by the lin_reg callers")
            k = min(k, len(a))
            a = pa.chunked_array([pa.nulls(k, type=a.type)] + a.slice(0, len(a) - k).chunks, type=a.type)
        if c.slice_offset:
            a = a.slice(min(c.slice_offset, len(a)))
        if c.centered:
            a = _centered(a)
        return a

    def evaluate(self, e: PluginExpr) -> pa.Array:
        if e.over_key is not None:
            return self._evaluate_over(e)
        inputs = [self._eval_arg(a) for a in e.args]
        names = [a.out_name for a in e.args]
        # kwargs None: a symbol without kwargs, which Polars calls with an empty buffer
        out = _harness.call_plugin(e.symbol, inputs, names, e.kwargs or {}, raw_kwargs=b"" if e.kwargs is None else None)
        for step in e.list_post:
            out = _list_post(out, step)
        return out

    def _evaluate_over(self, e: PluginExpr) -> pa.Array:
        """``e.over(key)``: the per-row results of each group, in the frame's row order."""
        uniq, gid = _group_ids(self.columns[e.over_key].to_numpy(zero_copy_only=False))
        order, offsets = _key_order(gid, len(uniq))
        inverse = np.empty(len(order), dtype=np.int64)
        inverse[order] = np.arange(len(order), dtype=np.int64)
        inner = replace(e, over_key=None, over_fast=False)
        if not e.over_fast:
            # Polars' loop: one call of the expression's own symbol per group, then every group's rows go back in place
            parts = [self.filter(gid == g).evaluate(inner) for g in range(len(uniq))]
            res = pa.concat_arrays(parts) if parts else self.evaluate(inner)
        else:
            sym = _wls_by_group(e, per_row=True) or _by_group(e.symbol, per_row=True)
            res = self._call_by_group(sym, e, order, offsets)
        return res.take(pa.array(inverse))

    def _call_by_group(self, symbol: str, e: PluginExpr, order: np.ndarray, offsets: np.ndarray) -> pa.Array:
        """One call of the batched group symbol (``_BY_GROUP``; ``_f32`` for an f32 expression): the group offsets, then
        each argument of ``e`` with its rows in group order (without the ``var()`` argument for ``_VAR_ON_DEVICE``; a
        one-row literal as it is; for ``_CENTER_ON_DEVICE`` the columns un-centred, with kwargs ``{"center": ...}``)."""
        if any(a.shift_by or a.slice_offset for a in e.args):
            raise ValueError(_SHIFT_REFUSED)
        take = pa.array(order)
        inputs = [pa.chunked_array([pa.array(offsets)])]
        names = ["__offsets__"]
        kwargs = e.kwargs
        if symbol in _CENTER_ON_DEVICE:
            centred = {a.centered for a in e.args if a.lit_u32 is None}
            if len(centred) > 1:
                raise ValueError("fast group_by / over: either every feature is centred or none is")
            kwargs = {"center": centred == {True}}
        for a in e.args:
            if a.agg == "var" and symbol in _VAR_ON_DEVICE:
                continue
            if a.lit_u32 is not None:
                inputs.append(self._eval_arg(a))
            else:
                if symbol in _CENTER_ON_DEVICE:
                    a = replace(a, centered=False)
                inputs.append(pa.chunked_array([self._eval_arg(a).combine_chunks().take(take)]))
            names.append(a.out_name)
        return _harness.call_plugin(symbol + ("_f32" if e.symbol.endswith("_f32") else ""), inputs, names, kwargs)

    def _call_ar_by_group(self, e: PluginExpr, ar: Tuple[str, Optional[str], int], order: np.ndarray,
                          offsets: np.ndarray) -> pa.Array:
        """One call of ``pl_ar_coeffs_by`` (``_f32`` for an f32 expression) for the autoregression ``ar`` of
        ``_ar_pattern``: the group offsets, then the column once, cast as the target is and in group order, with the
        expression's kwargs plus ``lag``.  The lagged columns are formed on the device, within each group."""
        name, cast_to, lag = ar
        x = self._eval_arg(ColExpr(name, cast_to=cast_to)).combine_chunks().take(pa.array(order))
        inputs = [pa.chunked_array([pa.array(offsets)]), pa.chunked_array([x])]
        symbol = "pl_ar_coeffs_by" + ("_f32" if e.symbol.endswith("_f32") else "")
        return _harness.call_plugin(symbol, inputs, ["__offsets__", name], dict(e.kwargs, lag=lag))

    def select(self, *exprs: PluginExpr) -> Dict[str, pa.Array]:
        return {(e.out_name or e.symbol): self.evaluate(e) for e in exprs}

    def group_by(self, key: str) -> "GroupBy":
        return GroupBy(self, key)


class GroupBy:
    def __init__(self, frame: Frame, key: str):
        self.frame = frame
        self.key = key

    def agg(self, e: PluginExpr, fast: bool = False) -> Dict[str, Any]:
        uniq, gid = _group_ids(self.frame.columns[self.key].to_numpy(zero_copy_only=False))
        if not fast:
            out = [self.frame.filter(gid == g).evaluate(e) for g in range(len(uniq))]
            return {self.key: uniq, (e.out_name or e.symbol): out}
        # batched path: rows sorted stably by key, one call of the batched symbol over the contiguous groups
        wls = _wls_by_group(e, per_row=False)
        if wls is not None:
            res = self.frame._call_by_group(wls, e, *_key_order(gid, len(uniq)))
            return {self.key: uniq, (e.out_name or e.symbol): res}
        ar = _ar_pattern(e)
        if ar is not None:
            res = self.frame._call_ar_by_group(e, ar, *_key_order(gid, len(uniq)))
            return {self.key: uniq, (e.out_name or e.symbol): res}
        sym = _by_group(e.symbol, per_row=False)
        if sym is None:
            raise ValueError("fast group_by is only available for lin_reg coefficients, logistic_reg coefficients, "
                             "lin_reg_report without weights, lin_reg_w_rcond, singular_values and pca")
        res = self.frame._call_by_group(sym, e, *_key_order(gid, len(uniq)))
        for step in e.list_post:
            res = _list_post(res, step)
        return {self.key: uniq, (e.out_name or e.symbol): res}
