"""Multi-GPU INSIDE the library (SURVEY.md §8e): a single plugin call row-sharded over a device group
(pdsb_set_devices / PDS_B200_DEVICES), and the one-process-per-GPU world communicator (pdsb_comm_init_rank), both
ending in one NCCL all-reduce of the f64 moments.  Needs >= 2 GPUs; skipped on a 1-GPU machine.
The host-side partition / collective protocol is covered on CPU by tests/test_multi_cpu.py (gloo, world_size 2)."""
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = Path(__file__).resolve().parents[1]
KW = {"bias": True, "null_policy": "skip", "l1_reg": 0.0, "l2_reg": 0.0, "solver": "qr", "tol": 1e-5, "max_iter": 200,
      "weighted": False, "positive": False, "singular_x_tol": 1e-6}


def _n_gpus():
    import torch

    return torch.cuda.device_count()


def _data(n, p, seed, f32=True, nulls=False):
    import pyarrow as pa

    rng = np.random.default_rng(seed)
    dt = np.float32 if f32 else np.float64
    X = rng.standard_normal((p, n)).astype(dt)
    beta = ((np.arange(p) % 7) - 3) / 4.0
    y = (beta @ X + 0.3 + 0.1 * rng.standard_normal(n)).astype(dt)
    cols = [pa.array(y)] + [pa.array(X[i]) for i in range(p)]
    if nulls:
        m = rng.random(n) < 0.01
        cols[2] = pa.array(X[1], mask=m)                       # validity bitmap crossing the shard boundaries
        cols[0] = pa.chunked_array([pa.array(y[: n // 3 + 5]), pa.array(y[n // 3 + 5:])])      # and a chunked target
    return cols, ["y"] + [f"x{i}" for i in range(p)]


@pytest.mark.skipif("_n_gpus() < 2")
@pytest.mark.parametrize("f32", [True, False])
@pytest.mark.parametrize("nulls", [False, True])
def test_device_group_equals_single_device(f32, nulls):
    """One plugin call over 2 (or all) GPUs == the same call on one GPU: coefficients to f64 round-off of the moments
    sum order, predictions to one ulp of the data dtype; null rows stay null; every GPU did part of the work."""
    from polars_ds_extension_b200 import _harness, parallel
    from polars_ds_extension_b200._lib import lib

    n, p = 5_000_000, 8
    cols, names = _data(n, p, 11, f32, nulls)
    sfx = "_f32" if f32 else ""
    L = lib()
    parallel.set_devices([])
    assert L.pdsb_device_group_size() == 1
    c1 = _harness.call_plugin("pl_lr" + sfx, cols, names, KW)
    p1 = _harness.call_plugin("pl_lr_pred" + sfx, cols, names, KW)
    try:
        parallel.set_devices(list(range(_n_gpus())))
        assert L.pdsb_device_group_size() == _n_gpus()
        ck = _harness.call_plugin("pl_lr" + sfx, cols, names, KW)
        pk = _harness.call_plugin("pl_lr_pred" + sfx, cols, names, KW)
    finally:
        parallel.set_devices([])
    a, b = np.asarray(c1[0].as_py()), np.asarray(ck[0].as_py())
    assert np.max(np.abs(a - b)) <= (2e-7 if f32 else 1e-12) * np.max(np.abs(a))
    for fld in ("pred", "resid"):
        x1, xk = p1.field(fld), pk.field(fld)
        assert x1.null_count == xk.null_count and (x1.null_count > 0) == nulls
        v1 = x1.fill_null(0).to_numpy(zero_copy_only=False)
        vk = xk.fill_null(0).to_numpy(zero_copy_only=False)
        assert np.array_equal(x1.is_valid().to_numpy(zero_copy_only=False), xk.is_valid().to_numpy(zero_copy_only=False))
        assert np.max(np.abs(v1 - vk)) <= (4e-6 if f32 else 1e-11) * max(1.0, np.max(np.abs(v1)))


@pytest.mark.skipif("_n_gpus() < 2")
def test_small_calls_stay_on_one_device():
    from polars_ds_extension_b200 import _harness, parallel

    cols, names = _data(10_000, 3, 5)
    one = _harness.call_plugin("pl_lr_f32", cols, names, KW)
    try:
        parallel.set_devices([0, 1])
        two = _harness.call_plugin("pl_lr_f32", cols, names, KW)       # below PDS_B200_SHARD_MIN_ROWS: not sharded
    finally:
        parallel.set_devices([])
    assert one.equals(two)


@pytest.mark.skipif("_n_gpus() < 2")
def test_world_communicator_fits_one_regression_over_all_ranks(tmp_path):
    """torchrun, 2 ranks: each rank passes ITS rows to the plugin symbol; the coefficients every rank gets are those of
    the fit over the union (checked against numpy on the concatenated data), predictions are those of its own rows."""
    out = tmp_path / "world.npz"
    env = dict(os.environ, PYTHONPATH=str(ROOT))
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
                        "--master-addr", "127.0.0.1", "--master-port", "29731", str(ROOT / "tests" / "_world_worker.py"), str(out)],
                       capture_output=True, text=True, env=env, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    z = np.load(out)
    assert z["ok"].all()
    assert z["coef_err"].max() < 1e-5 and z["pred_err"].max() < 1e-4
