"""Every moments route bit for bit on integer data.

Features in [-8, 8] with a row-tag column (row % 251) - 125, targets |y| <= 72, weights 1..4: every product is an
integer below 2^16, and every f32 chain of the routes below sums fewer than 2^24 / (4 * 125^2) = 268 such products of
the tag, so each route's moments are exact.  The f32 chain of each kernel, in rows:
  register kernel (path 3, and K5's grouped register kernel): <= 260 rows per lane (8192-row items rounded up to 128,
                                                                 over 32 lanes);
  wgmma kernel (path 1): 256 rows (two 128-row stages) before its f64 flush;
  tile kernel: 128 rows;
  DMMA kernels: f64 products and sums (f32 columns widened on the fly), exact here whatever the chain.
The device result must therefore equal the int64 moments exactly (np.array_equal), on the route asserted through
pdsb_last_moments_path, and a second call must return the same bits.  One dropped, duplicated or misplaced row changes the
count entry at least, so nothing short of the exact rows passes.
"""
import numpy as np
import pytest

from tests.exact_oracle import exact_moments, f32_chain_ok, int_design

pytestmark = pytest.mark.gpu

# row counts around every stage and chunk: 8-row DMMA blocks and their tail, the 128-row wgmma / tile stage, the 4096-row
# wgmma floor, the 8192-row register-kernel item, a many-item frame and one past 2^21
ROWS = [1, 7, 8, 9, 127, 128, 129, 4095, 4096, 4097, 8191, 8192, 8193, 128 * 1000 + 33, 2 ** 21 + 3]
CHAIN = {3: 260, 1: 256, "tile": 128}


def _torch():
    import torch
    return torch


def _lib():
    from polars_ds_extension_b200._lib import lib
    return lib()


def _upload(d, dtype, order="xy", masked=False, offset=0):
    """(Z, X, Y, mask, w) on the device: Z (p + t, ld) with rows [offset, offset + n) holding the design (masked rows
    zero, as the packer leaves them), X / Y views in `order`."""
    torch = _torch()
    n, p = d.X.shape
    t = d.Y.shape[1]
    ld = (n + offset + 31) // 32 * 32
    blocks = [d.X.T, d.Y.T] if order == "xy" else [d.Y.T, d.X.T]
    Zh = np.zeros((p + t, ld))
    Zh[:, offset:offset + n] = np.concatenate(blocks, axis=0)
    keep = d.kept()
    if masked:
        Zh[:, offset:offset + n] *= keep[None, :]
    Z = torch.from_numpy(Zh).to(dtype).cuda()
    X, Y = (Z[:p], Z[p:]) if order == "xy" else (Z[t:], Z[:t])
    mask = w = None
    if masked:
        mh = np.zeros(ld)
        mh[offset:offset + n] = keep
        mask = torch.from_numpy(mh).to(dtype).cuda()[offset:]
    if d.w is not None:
        wh = np.zeros(ld)
        wh[offset:offset + n] = d.w
        w = torch.from_numpy(wh).to(dtype).cuda()[offset:]
    if offset:
        X, Y = X[:, offset:], Y[:, offset:]
    return Z, X, Y, mask, w


def _moments(X, Y, n, w=None, mask=None, path=0):
    from polars_ds_extension_b200 import device as dev
    L = _lib()
    L.pdsb_set_moments_path(path)
    try:
        M1 = dev.moments(X, Y, n=n, w=w, mask=mask).cpu().numpy()
        route = L.pdsb_last_moments_path()
        M2 = dev.moments(X, Y, n=n, w=w, mask=mask).cpu().numpy()
    finally:
        L.pdsb_set_moments_path(0)
    assert np.array_equal(M1, M2), "not bit-reproducible"
    return M1, route


def _frame_moments(d, order, masked):
    from polars_ds_extension_b200 import device as dev
    torch = _torch()
    n, p = d.X.shape
    t = d.Y.shape[1]
    Z, X, Y, mask, _ = _upload(d, torch.float32, order, masked)
    frame = dev.to_frame(Z, n=n)
    xcol, ycol = (0, p) if order == "xy" else (t, 0)
    L = _lib()
    M1 = dev.moments_frame(frame, n, p + t, xcol, p, ycol, t, mask=mask).cpu().numpy()
    route = L.pdsb_last_moments_path()
    M2 = dev.moments_frame(frame, n, p + t, xcol, p, ycol, t, mask=mask).cpu().numpy()
    assert np.array_equal(M1, M2), "not bit-reproducible"
    return M1, route


def _exact(d, what):
    M = exact_moments(d)
    return M.astype(np.float64)


def _check(M, d, what):
    ref = _exact(d, what)
    bad = np.argwhere(M != ref)
    assert bad.size == 0, f"{what}: {len(bad)} entries differ, first {bad[:3].tolist()}: " \
                          f"{[(M[i, j], ref[i, j]) for i, j in bad[:3]]}"


# ---------------------------------------------------------------------------------------------------------------------
# f32 path 3 (the register kernel): 1..10 features, one target, no mask or weights, from 65 536 rows
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [65_535, 65_536, 65_537])
@pytest.mark.parametrize("p", list(range(1, 11)))
def test_f32_register_route_exact(p, n):
    torch = _torch()
    d = int_design(100 + p, n, p)
    assert f32_chain_ok(d, CHAIN[3])
    _, X, Y, _, _ = _upload(d, torch.float32)
    M, route = _moments(X, Y, n)
    assert route == (3 if n >= 65_536 else 1), route
    _check(M, d, f"path 3 p={p} n={n}")


# ---------------------------------------------------------------------------------------------------------------------
# f32 wgmma (path 1, forced so that <= 10 features do not take the register kernel)
# ---------------------------------------------------------------------------------------------------------------------
WGMMA = [(p, t, (p + t) % 2 == 1, ("cm", "frame")[(p // 16 + t) % 2], ("xy", "yx")[t % 2])
         for p in (1, 15, 16, 17, 32, 33, 48, 64) for t in (1, 2, 3, 4)]


@pytest.mark.parametrize("p,t,masked,layout,order", WGMMA)
def test_f32_wgmma_route_exact(p, t, masked, layout, order):
    torch = _torch()
    n = 20_000 + 37 * p + t
    d = int_design(200 + 7 * p + t, n, p, t, drop_frac=0.2 if masked else 0.0)
    assert f32_chain_ok(d, CHAIN[1])
    if layout == "cm":
        _, X, Y, mask, _ = _upload(d, torch.float32, order, masked)
        M, route = _moments(X, Y, n, mask=mask, path=2)
    else:
        M, route = _frame_moments(d, order, masked)
    assert route == 1, route
    _check(M, d, f"wgmma p={p} t={t} masked={masked} {layout} {order}")


# ---------------------------------------------------------------------------------------------------------------------
# f32 columns widened on the DMMA kernels (forced path 1, weights, six targets), and f64 on the DMMA kernels
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n,p,t,masked", [(50_006, 33, 6, False), (70_003, 20, 6, True), (4_099, 9, 6, False),
                                          (123_457, 5, 1, True)])
def test_f32_on_dmma_exact(n, p, t, masked):
    torch = _torch()
    d = int_design(300 + p, n, p, t, weights=True, drop_frac=0.25 if masked else 0.0)
    _, X, Y, mask, w = _upload(d, torch.float32, "xy", masked)
    M, route = _moments(X, Y, n, w=w, mask=mask, path=1)
    assert route == 0, route
    _check(M, d, f"f32 dmma n={n} p={p} t={t}")


# side kernel: t = 1 and at most 8 feature blocks (p <= 56 here); wide kernel: t > 1, (p + t + 8) / 8 <= 8; the last n % 8
# rows go through the row kernel; a view that starts at an odd row takes the direct kernel
F64_DMMA = [(200_131, 32, 1, True, False, 0), (70_003, 20, 3, True, True, 0), (100_005, 56, 1, False, True, 0),
            (33_335, 9, 2, False, False, 0), (50_001, 12, 1, False, False, 1), (40_003, 30, 4, True, False, 1),
            (15, 40, 1, True, False, 0), (13, 3, 5, False, True, 0)]


@pytest.mark.parametrize("n,p,t,weighted,masked,offset", F64_DMMA)
def test_f64_dmma_exact(n, p, t, weighted, masked, offset):
    torch = _torch()
    d = int_design(400 + p + t, n, p, t, weights=weighted, drop_frac=0.2 if masked else 0.0)
    _, X, Y, mask, w = _upload(d, torch.float64, "yx" if t > 1 else "xy", masked, offset)
    M, _ = _moments(X, Y, n, w=w, mask=mask)
    _check(M, d, f"f64 dmma n={n} p={p} t={t} offset={offset}")


# ---------------------------------------------------------------------------------------------------------------------
# the tile kernel: more than 64 features (f32: beyond wgmma; f64: beyond eight DMMA blocks), and f32 frames
# ---------------------------------------------------------------------------------------------------------------------
TILE = [(p, dt, layout) for p in (65, 87, 123, 175, 258) for dt, layout in (("f32", "cm"), ("f64", "cm"), ("f32", "frame"))]


@pytest.mark.parametrize("p,dt,layout", TILE)
def test_tile_route_exact(p, dt, layout):
    torch = _torch()
    n = 9_000 + 13 * p
    masked = p % 2 == 1
    weighted = dt == "f64" or p == 87
    d = int_design(500 + p, n, p, 1, weights=weighted and layout == "cm", drop_frac=0.1 if masked else 0.0)
    assert f32_chain_ok(d, CHAIN["tile"])
    if layout == "frame":
        M, route = _frame_moments(d, "yx", masked)
    else:
        _, X, Y, mask, w = _upload(d, torch.float32 if dt == "f32" else torch.float64, "xy", masked)
        M, route = _moments(X, Y, n, w=w, mask=mask)
    assert route == 0, route
    _check(M, d, f"tile p={p} {dt} {layout}")


# ---------------------------------------------------------------------------------------------------------------------
# row counts around every stage and chunk, on each route that has a stage or chunk
# ---------------------------------------------------------------------------------------------------------------------
ROUTES = {
    "f32 p=4 (path 3 from 65 536 rows, else wgmma / DMMA)": ("f32", 4, 1, "cm"),
    "f32 p=16 (wgmma from 4096 rows, else DMMA)": ("f32", 16, 1, "cm"),
    "f32 p=20 t=2 frame (wgmma from 4096 rows, else tile)": ("f32", 20, 2, "frame"),
    "f64 p=12 (side DMMA + row tail)": ("f64", 12, 1, "cm"),
    "f64 p=20 t=3 (wide DMMA + row tail)": ("f64", 20, 3, "cm"),
    "f32 p=70 (tile)": ("f32", 70, 1, "cm"),
}


@pytest.mark.parametrize("route", list(ROUTES))
@pytest.mark.parametrize("n", ROWS)
def test_row_counts_exact(route, n):
    torch = _torch()
    dt, p, t, layout = ROUTES[route]
    if p >= 64 and n > 200_000:
        pytest.skip("the int64 reference of 2^21 rows x 70 columns is not needed: the tile stage is 128 rows")
    d = int_design(600 + n % 1000 + p, n, p, t)
    assert f32_chain_ok(d, 260)
    if layout == "frame":
        M, path = _frame_moments(d, "xy", False)
        assert path == (1 if n >= 4096 else 0), path
    else:
        _, X, Y, _, _ = _upload(d, torch.float32 if dt == "f32" else torch.float64)
        M, path = _moments(X, Y, n)
        if dt == "f32" and p == 4:
            assert path == (3 if n >= 65_536 else 1 if n >= 4096 else 0), path
        elif dt == "f32" and p == 16:
            assert path == (1 if n >= 4096 else 0), path
    _check(M, d, f"{route} n={n}")
