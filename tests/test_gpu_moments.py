"""Device-layer parity of the moments kernels (K2a SIMT and K2b wgmma/TMA) against numpy float64 on the same
seeded inputs, through the C ABI (pdsb_dev_moments_*) with torch-allocated device memory."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _mk(torch, n, p, t, dtype, seed, order="xy", scale=1.0):
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    ld = (n + 31) // 32 * 32
    Z = torch.zeros((p + t, ld), dtype=dtype, device="cuda")
    Z[:, :n] = torch.randn((p + t, n), generator=g, device="cuda", dtype=dtype) * scale + 0.25
    if order == "xy":
        X, Y = Z[:p], Z[p:]
    else:
        Y, X = Z[:t], Z[t:]
    return Z, X, Y, ld


def _ref(X, Y, n, w=None, mask=None):
    Zh = np.concatenate([X[:, :n].double().cpu().numpy(), Y[:, :n].double().cpu().numpy(), np.ones((1, n))], axis=0)
    if mask is not None:
        Zh[-1] = mask[:n].double().cpu().numpy()
    W = np.ones(n) if w is None else w[:n].double().cpu().numpy()
    return (Zh * W) @ Zh.T


@pytest.mark.parametrize("n,p,t,order", [(4096, 4, 1, "xy"), (100_003, 32, 1, "yx"), (1_000_000, 32, 1, "xy"),
                                         (50_000, 8, 3, "yx"), (65_536 * 3 + 17, 62, 1, "xy"), (200_000, 1, 1, "xy"),
                                         (300_000, 14, 1, "xy"), (300_000, 15, 1, "xy"), (77_777, 47, 1, "yx"),
                                         (150_000, 64, 1, "yx")])
def test_tcgen05_moments_vs_numpy(n, p, t, order):
    import torch

    from polars_ds_extension_b200 import device as dev
    from polars_ds_extension_b200._lib import lib

    Z, X, Y, ld = _mk(torch, n, p, t, torch.float32, 7 + p, order)
    ref = _ref(X, Y, n)
    lib().pdsb_set_moments_path(2)          # force the wgmma kernel (errors if the shape were unsupported)
    try:
        M = dev.moments(X, Y, n=n).cpu().numpy()
        assert lib().pdsb_last_moments_path() == 1
    finally:
        lib().pdsb_set_moments_path(0)
    lib().pdsb_set_moments_path(1)
    try:
        Ms = dev.moments(X, Y, n=n).cpu().numpy()
    finally:
        lib().pdsb_set_moments_path(0)
    scale = np.sqrt(np.outer(np.diag(ref), np.diag(ref)))
    # X'X comes from the tensor core, X'y / sum x from the converter lanes, the y block from the side lanes
    assert np.isfinite(M).all()
    err_tc = np.max(np.abs(M - ref) / scale)
    err_simt = np.max(np.abs(Ms - ref) / scale)
    # 3xTF32 with f64 flushes: the dropped lo*lo term is ~2^-22; fp32 (round-toward-zero) accumulation over 256 rows
    assert err_tc < 3e-6, (err_tc, err_simt)
    assert err_simt < 3e-6, err_simt
    assert np.array_equal(M, M.T, equal_nan=True)


@pytest.mark.parametrize("n,p,masked", [(1_000_003, 32, False), (300_000, 20, True), (70_000, 62, False)])
def test_tcgen05_raw_hi_matches_explicit_hi(n, p, masked):
    """The kernel feeds RAW fp32 to the tensor core as the hi operand (it ignores the low 13 mantissa bits); variant 0
    makes the hi rows of the A operand clear those bits themselves.  If the hardware truncates, both are bit-identical
    (the B operand is raw in both: its truncation is what the 3e-6 accuracy bound of the test above proves)."""
    import torch

    from polars_ds_extension_b200 import device as dev
    from polars_ds_extension_b200._lib import lib

    Z, X, Y, ld = _mk(torch, n, p, 1, torch.float32, 21, scale=3.0)
    mask = None
    if masked:
        mask = (torch.rand(ld, device="cuda") > 0.3).float()
        Z[:, :] *= mask[None, :]
    L = lib()
    L.pdsb_set_moments_path(2)
    try:
        L.pdsb_set_tc_variant(0)
        M0 = dev.moments(X, Y, n=n, mask=mask).cpu().numpy()
        L.pdsb_set_tc_variant(1)
        M1 = dev.moments(X, Y, n=n, mask=mask).cpu().numpy()
    finally:
        L.pdsb_set_tc_variant(1)
        L.pdsb_set_moments_path(0)
    assert np.array_equal(M0, M1)


def test_tcgen05_moments_with_mask_and_repro():
    import torch

    from polars_ds_extension_b200 import device as dev
    from polars_ds_extension_b200._lib import lib

    n, p = 500_000, 16
    Z, X, Y, ld = _mk(torch, n, p, 1, torch.float32, 3)
    mask = (torch.rand(ld, device="cuda") > 0.2).float()
    Z[:, :] *= mask[None, :]                      # masked rows are zero in X and Y (packer contract)
    ref = _ref(X, Y, n, mask=mask)
    lib().pdsb_set_moments_path(2)
    try:
        M1 = dev.moments(X, Y, n=n, mask=mask).cpu().numpy()
        M2 = dev.moments(X, Y, n=n, mask=mask).cpu().numpy()
    finally:
        lib().pdsb_set_moments_path(0)
    assert np.array_equal(M1, M2)                 # bit-reproducible
    scale = np.sqrt(np.outer(np.diag(ref), np.diag(ref)))
    assert np.max(np.abs(M1 - ref) / scale) < 3e-6
    assert abs(M1[-1, -1] - float(mask[:n].sum().item())) < 0.5


@pytest.mark.parametrize("dtype", ["f32", "f64"])
def test_simt_moments_weighted(dtype):
    import torch

    from polars_ds_extension_b200 import device as dev

    td = torch.float32 if dtype == "f32" else torch.float64
    n, p, t = 33_333, 5, 2
    Z, X, Y, ld = _mk(torch, n, p, t, td, 11)
    w = torch.rand(ld, device="cuda", dtype=td) + 0.5
    ref = _ref(X, Y, n, w=w)
    M = dev.moments(X, Y, n=n, w=w).cpu().numpy()
    tol = 3e-6 if dtype == "f32" else 1e-12
    assert np.max(np.abs(M - ref) / np.sqrt(np.outer(np.diag(ref), np.diag(ref)))) < tol


@pytest.mark.parametrize("n,p,t,weighted,masked", [(100_000, 4, 1, False, False), (200_131, 32, 1, False, False),
                                                   (65_536, 32, 1, True, False), (70_003, 20, 2, False, True),
                                                   (40_000, 61, 2, True, True), (5_000, 7, 1, False, False),
                                                   (4_096, 1, 1, False, False), (300_007, 8, 1, False, True),
                                                   (123_457, 9, 1, True, True), (90_001, 16, 1, False, False),
                                                   (50_006, 33, 1, True, False), (64_000, 57, 1, False, True),
                                                   (33_333, 64, 1, True, True), (20_000, 64, 1, False, False),
                                                   (7, 3, 1, False, False), (15, 40, 1, True, False),
                                                   (1_000_001, 30, 3, False, False)])
def test_f64_moments_dmma(n, p, t, weighted, masked):
    """The f64 path (the reference's default dtype) on the FP64 tensor cores: one target -> feature blocks on DMMA with
    y / ones / weights as lane-local DFMAs (side kernel), several targets -> all columns in blocks (wide kernel), the
    last n % 8 rows through gram_rows_kernel; against numpy float64, bit-reproducible, symmetric."""
    import torch

    from polars_ds_extension_b200 import device as dev

    Z, X, Y, ld = _mk(torch, n, p, t, torch.float64, 3 + p)
    w = (torch.rand(ld, device="cuda", dtype=torch.float64) + 0.5) if weighted else None
    mask = None
    if masked:
        mask = (torch.rand(ld, device="cuda") > 0.2).double()
        Z[:, :] *= mask[None, :]
    ref = _ref(X, Y, n, w=w, mask=mask)
    M1 = dev.moments(X, Y, n=n, w=w, mask=mask).cpu().numpy()
    M2 = dev.moments(X, Y, n=n, w=w, mask=mask).cpu().numpy()
    assert np.array_equal(M1, M2)
    scale = np.sqrt(np.outer(np.diag(ref), np.diag(ref)))
    assert np.max(np.abs(M1 - ref) / scale) < 1e-12
    assert np.array_equal(M1, M1.T)


def test_f64_moments_unaligned_columns_take_the_direct_kernel():
    """Columns that are not 16-byte aligned (a view that starts at an odd row) cannot use 16-byte loads: same numbers
    from the 4-row direct kernel."""
    import torch

    from polars_ds_extension_b200 import device as dev

    n, p = 50_001, 12
    Z, X, Y, ld = _mk(torch, n + 1, p, 1, torch.float64, 99)
    Xo, Yo = X[:, 1:], Y[:, 1:]
    ref = _ref(Xo, Yo, n)
    M = dev.moments(Xo, Yo, n=n).cpu().numpy()
    scale = np.sqrt(np.outer(np.diag(ref), np.diag(ref)))
    assert np.max(np.abs(M - ref) / scale) < 1e-12


@pytest.mark.parametrize("n,p,t,weighted,masked", [(200_131, 32, 1, True, False), (70_003, 20, 2, True, True),
                                                   (123_457, 9, 1, True, True), (33_333, 64, 1, True, False),
                                                   (50_006, 33, 6, False, False), (15, 40, 1, True, False),
                                                   (90_001, 16, 1, False, True)])
def test_f32_columns_on_the_dmma_kernels(n, p, t, weighted, masked):
    """f32 fits the wgmma kernel does not take (weights, more than 4 targets) or that are forced off it: the same
    DMMA kernels widen the f32 columns on the fly, so products and sums are exact to f64 rounding."""
    import torch

    from polars_ds_extension_b200 import device as dev
    from polars_ds_extension_b200._lib import lib

    Z, X, Y, ld = _mk(torch, n, p, t, torch.float32, 11 + p)
    w = (torch.rand(ld, device="cuda", dtype=torch.float32) + 0.5) if weighted else None
    mask = None
    if masked:
        mask = (torch.rand(ld, device="cuda") > 0.2).float()
        Z[:, :] *= mask[None, :]
    ref = _ref(X, Y, n, w=w, mask=mask)
    lib().pdsb_set_moments_path(1)
    try:
        M1 = dev.moments(X, Y, n=n, w=w, mask=mask).cpu().numpy()
        M2 = dev.moments(X, Y, n=n, w=w, mask=mask).cpu().numpy()
    finally:
        lib().pdsb_set_moments_path(0)
    assert np.array_equal(M1, M2)
    scale = np.sqrt(np.outer(np.diag(ref), np.diag(ref)))
    assert np.max(np.abs(M1 - ref) / scale) < 1e-12
    assert np.array_equal(M1, M1.T)
