"""Row-blocked frame layout ([block][column][128], include/pdsb.h): conversion, moments (wgmma and the SIMT fallback)
and predict on frames agree with the column-major path and with numpy float64."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("n,p,t,order", [(4096, 3, 1, "xy"), (100_003, 32, 1, "xy"), (257_000, 32, 1, "yx"),
                                         (70_001, 62, 1, "xy"), (50_000, 70, 1, "xy"), (33_000, 8, 3, "yx"),
                                         (90_001, 64, 1, "xy"), (64_000, 63, 2, "yx")])
def test_frame_moments_and_predict(n, p, t, order):
    import torch

    from polars_ds_extension_b200 import device as dev
    from polars_ds_extension_b200._lib import lib

    g = torch.Generator(device="cuda")
    g.manual_seed(5 + p)
    ld = (n + 31) // 32 * 32
    Z = torch.zeros((p + t, ld), dtype=torch.float32, device="cuda")
    Z[:, :n] = torch.randn((p + t, n), generator=g, device="cuda") * 1.3 + 0.2
    xcol, ycol = (0, p) if order == "xy" else (t, 0)
    X, Y = Z[xcol:xcol + p], Z[ycol:ycol + t]
    frame = dev.to_frame(Z, n=n)
    # layout contract: element (r, c) at (r // 128) * ncols * 128 + c * 128 + r % 128; padding rows are zero
    fr = frame.view(-1, p + t, 128)
    r = n - 1
    assert float(fr[r // 128, 1, r % 128]) == float(Z[1, r])
    if n % 128:
        assert float(fr[-1, :, n % 128:].abs().max()) == 0.0
    Zh = np.concatenate([X[:, :n].double().cpu().numpy(), Y[:, :n].double().cpu().numpy(), np.ones((1, n))])
    ref = Zh @ Zh.T
    scale = np.sqrt(np.outer(np.diag(ref), np.diag(ref)))
    Mf = dev.moments_frame(frame, n, p + t, xcol, p, ycol, t).cpu().numpy()
    used_tc = lib().pdsb_last_moments_path() == 1
    # tensor-core path: up to 64 features on the tensor core, up to 4 targets on the side lanes
    assert used_tc == (n >= 4096 and p <= 64 and t <= 4)
    Mc = dev.moments(X, Y, n=n).cpu().numpy()
    assert np.isfinite(Mf).all()          # every block is produced, including y_i . y_j (i != j) from the side lanes
    assert np.max(np.abs(Mf - ref) / scale) < 3e-6
    if used_tc:
        assert np.array_equal(Mf, Mc, equal_nan=True)      # same kernel, same stage order: the layout must not change a single bit
    # predict on the frame == predict on the column-major matrix (bit for bit), with and without bias
    beta, status = dev.solve(torch.from_numpy(Mf).cuda(), p, t, add_bias=True)
    pc, rc = dev.predict(X, Y, beta, status, add_bias=True, n=n)
    pf = torch.empty((t, ld), dtype=torch.float32, device="cuda")
    rf = torch.empty((t, ld), dtype=torch.float32, device="cuda")
    ssr = torch.zeros(8, dtype=torch.float64, device="cuda")
    dev.predict_frame(frame, n, p + t, xcol, p, ycol, t, beta, status, True, pf, rf, ssr=ssr)
    assert torch.equal(pf[:, :n], pc[:, :n]) and torch.equal(rf[:, :n], rc[:, :n])
    assert abs(float(ssr[0]) - float((rc[0, :n].double() ** 2).sum())) < 1e-6 * float(ssr[0]) + 1e-12


def test_frame_moments_masked():
    import torch

    from polars_ds_extension_b200 import device as dev

    n, p = 300_001, 20
    ld = (n + 31) // 32 * 32
    Z = torch.zeros((p + 1, ld), dtype=torch.float32, device="cuda")
    Z[:, :n] = torch.randn((p + 1, n), device="cuda")
    mask = (torch.rand(ld, device="cuda") > 0.25).float()
    Z *= mask[None, :]
    frame = dev.to_frame(Z, n=n)
    Mf = dev.moments_frame(frame, n, p + 1, 0, p, p, 1, mask=mask).cpu().numpy()
    Mc = dev.moments(Z[:p], Z[p:], n=n, mask=mask).cpu().numpy()
    assert np.array_equal(Mf, Mc)
    assert abs(Mf[-1, -1] - float(mask[:n].sum())) < 0.5
