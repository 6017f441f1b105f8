"""The wgmma moments kernel computes x . y_j and the column sums on the tensor core: the MMA's B operand carries, after
the feature rows, the targets, their TF32 remainders ylo_j = y_j - trunc_tf32(y_j) and a row of ones, and
X'y_j = D[hi, y_j] + D[lo, y_j] + D[hi, ylo_j] + D[lo, ylo_j],  sum x = D[hi, 1] + D[lo, 1].  The target block
(sum y, y_j . y_k, the masked count) is summed in f64 by the consumer threads.  Every shape the kernel takes is checked
against numpy float64: 1..64 features, 1..4 targets, masked or not, column-major matrices and row-blocked frames, X
before Y and Y before X."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

PS = [1, 15, 16, 17, 32, 33, 48, 64]
TS = [1, 2, 4]


def _data(torch, n, p, t, seed, xmean, ymean, masked):
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    ld = (n + 31) // 32 * 32
    X = torch.randn((p, n), generator=g, device="cuda") + xmean
    Y = torch.randn((t, n), generator=g, device="cuda") + ymean
    mask = None
    if masked:
        mask = torch.zeros(ld, device="cuda")
        mask[:n] = (torch.rand(n, generator=g, device="cuda") > 0.3).float()
        X *= mask[None, :n]                      # masked rows are zero in X and Y (packer contract)
        Y *= mask[None, :n]
    return X, Y, mask, ld


def _ref(X, Y, mask, n):
    ones = np.ones((1, n)) if mask is None else mask[:n].double().cpu().numpy()[None, :]
    Zh = np.concatenate([X.double().cpu().numpy(), Y.double().cpu().numpy(), ones], axis=0)
    return Zh @ Zh.T


def _moments(torch, X, Y, mask, n, ld, layout, order):
    """M through the wgmma kernel; layout "cm" = column-major (p + t, ld) matrix, "frame" = row-blocked frame."""
    from polars_ds_extension_b200 import device as dev
    from polars_ds_extension_b200._lib import lib

    p, t = X.shape[0], Y.shape[0]
    Z = torch.zeros((p + t, ld), dtype=torch.float32, device="cuda")
    xcol, ycol = (0, p) if order == "xy" else (t, 0)
    Z[xcol:xcol + p, :n] = X
    Z[ycol:ycol + t, :n] = Y
    L = lib()
    L.pdsb_set_moments_path(2)                   # force the wgmma kernel (errors if the shape were unsupported)
    try:
        if layout == "cm":
            M = dev.moments(Z[xcol:xcol + p], Z[ycol:ycol + t], n=n, mask=mask)
        else:
            M = dev.moments_frame(dev.to_frame(Z, n=n), n, p + t, xcol, p, ycol, t, mask=mask)
        M = M.cpu().numpy()
        assert L.pdsb_last_moments_path() == 1
    finally:
        L.pdsb_set_moments_path(0)
    return M


def _err(M, ref):
    scale = np.sqrt(np.outer(np.diag(ref), np.diag(ref)))
    assert np.isfinite(M).all()
    assert np.array_equal(M, M.T)
    return float(np.max(np.abs(M - ref) / scale))


@pytest.mark.parametrize("t", TS)
@pytest.mark.parametrize("p", PS)
def test_moments_every_shape_and_layout(p, t):
    """n = 20_011 is not a multiple of the 128-row stage, so the last stage holds rows past n."""
    import torch

    n = 20_011
    for masked in (False, True):
        X, Y, mask, ld = _data(torch, n, p, t, 100 * p + t, 0.5, 0.25, masked)
        ref = _ref(X, Y, mask, n)
        for layout in ("cm", "frame"):
            for order in ("xy", "yx"):
                M = _moments(torch, X, Y, mask, n, ld, layout, order)
                e = _err(M, ref)
                # 3xTF32 with f64 flushes: the dropped lo*lo term is ~2^-22
                assert e < 3e-6, (masked, layout, order, e)
                if masked:
                    assert abs(M[-1, -1] - float(mask[:n].sum())) < 0.5
                else:
                    assert M[-1, -1] == n


@pytest.mark.parametrize("p,t", [(1, 1), (17, 2), (32, 1), (32, 4), (33, 1), (64, 1), (64, 3)])
def test_moments_large_means(p, t):
    """y = 1e3 + N(0, 1): its TF32 truncation is off by up to 0.5 per row, always towards zero, so X'y is wrong by
    ~1e-4 (normalised) without the ylo term.  x = 5 + N(0, 1): dropping the lo half of sum x is off by ~1e-4 too."""
    import torch

    n = 65_536 + 77
    X, Y, mask, ld = _data(torch, n, p, t, 7 + p, 5.0, 1e3, False)
    ref = _ref(X, Y, mask, n)
    for layout in ("cm", "frame"):
        for order in ("xy", "yx"):
            M = _moments(torch, X, Y, mask, n, ld, layout, order)
            assert _err(M, ref) < 3e-6, (layout, order)


@pytest.mark.parametrize("n", [4096 + 1, 128 * 1000 + 33, 128 * 1000 + 96])
def test_moments_partial_last_stage(n):
    """Rows past n in the last stage (and whole 32-row boxes of it) must not count: the row of ones in the tile meets
    zero features there, and the count comes from n."""
    import torch

    p, t = 32, 1
    X, Y, mask, ld = _data(torch, n, p, t, n % 1000, 3.0, 2.0, False)
    ref = _ref(X, Y, mask, n)
    for layout in ("cm", "frame"):
        M = _moments(torch, X, Y, mask, n, ld, layout, "xy")
        assert _err(M, ref) < 3e-6, layout
        assert M[-1, -1] == n
        np.testing.assert_allclose(M[-1, :p], ref[-1, :p], rtol=3e-6)
