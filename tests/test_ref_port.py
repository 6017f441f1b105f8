"""The C (OpenMP) restatement used as the timed CPU arm (oracle/ref_port.c) agrees with the numpy oracle."""
import numpy as np

from oracle import lin_reg_oracle as orc
from oracle import ref_port


def _data(n, p, seed=208):
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((p, n), dtype=np.float32)
    beta = (((np.arange(p) % 7) - 3.0) / 4.0).astype(np.float32)
    y = (beta @ X + 0.1 * rng.standard_normal(n, dtype=np.float32)).astype(np.float32)
    return X, y, beta


def test_ref_port_matches_numpy_oracle():
    for n, p, bias in [(50_000, 32, False), (20_001, 5, True), (1000, 64, False)]:
        X, y, beta = _data(n, p, seed=p)
        cols = [y] + [np.ascontiguousarray(X[i]) for i in range(p)]
        c, pred, resid, times = ref_port.lr_pred_f32(cols, add_bias=bias)
        kw = {"bias": bias, "null_policy": "skip", "l1_reg": 0.0, "l2_reg": 0.0, "solver": "qr", "tol": 1e-5,
              "max_iter": 200, "weighted": False, "positive": False, "singular_x_tol": 1e-6}
        ocols = [orc.Col("y", y)] + [orc.Col(f"x{i}", X[i]) for i in range(p)]
        oc = orc.pl_lr(ocols, kw, f32=True)
        op = orc.pl_lr_pred(ocols, kw, f32=True)
        assert np.max(np.abs(c - oc)) < 2e-4 * max(1.0, np.max(np.abs(oc)))
        assert np.max(np.abs(pred - op["pred"][0])) < 2e-4 * np.max(np.abs(op["pred"][0]))
        assert np.allclose(resid, y - pred, atol=1e-6)
        assert times["total"] > 0 and ref_port.threads() >= 1


def test_ref_port_gate():
    n = 5000
    rng = np.random.default_rng(3)
    x = rng.standard_normal(n, dtype=np.float32)
    cols = [x * 2, x, (x * 3).astype(np.float32)]          # collinear features -> the rank gate fires -> None
    c, _, _, _ = ref_port.lr_pred_f32(cols)
    assert c is None


def test_cpu_arm_thread_count_follows_quota_and_override(monkeypatch, tmp_path):
    """bench.py's CPU arm runs on the CPUs the process may use: the affinity mask cut to the cgroup quota (a container may
    see 128 cores under `cpu.max 1600000 100000`), PDSB_BENCH_THREADS overrides."""
    import builtins

    import bench

    monkeypatch.setenv("PDSB_BENCH_THREADS", "5")
    assert bench.host_threads() == 5
    monkeypatch.delenv("PDSB_BENCH_THREADS")
    real_open = builtins.open
    fake = tmp_path / "cpu.max"

    def fake_open(path, *a, **k):
        return real_open(fake if path == "/sys/fs/cgroup/cpu.max" else path, *a, **k)

    monkeypatch.setattr(builtins, "open", fake_open)
    fake.write_text("200000 100000\n")
    assert bench.cpu_quota() == 2.0
    assert bench.host_threads() <= 2
    fake.write_text("max 100000\n")
    assert bench.cpu_quota() == 0.0
    assert bench.host_threads() >= 1
