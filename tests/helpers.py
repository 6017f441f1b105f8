"""Helpers shared by the test modules: the GPU probe, group offsets, a recording fake of _harness.call_plugin and a
column split into chunks."""
import numpy as np
import pyarrow as pa

from polars_ds_extension_b200 import _harness


def has_gpu():
    try:
        import torch

        return torch.cuda.is_available()
    except Exception:
        return False


def group_offsets(sizes):
    """The Int64 offsets of groups of the given sizes: 0, then the running total."""
    return np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)


def capture_plugin(monkeypatch, result):
    """Replace _harness.call_plugin with a fake that returns `result`; the list it returns collects every call's
    (symbol, inputs, names, kwargs)."""
    calls = []

    def fake(symbol, inputs, names, kwargs, raw_kwargs=None):
        calls.append((symbol, inputs, list(names), kwargs))
        return result

    monkeypatch.setattr(_harness, "call_plugin", fake)
    return calls


def chunked(v, chunks, mask=None):
    """`v` (with validity `mask`: True = null) as one Arrow array, or as a ChunkedArray of `chunks` near-equal parts."""
    if chunks == 1:
        return pa.array(v, mask=mask)
    cut = np.linspace(0, len(v), chunks + 1).astype(int)
    return pa.chunked_array([pa.array(v[a:b], mask=None if mask is None else mask[a:b])
                             for a, b in zip(cut[:-1], cut[1:])])
