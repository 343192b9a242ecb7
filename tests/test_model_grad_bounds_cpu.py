"""The per-component gradient bounds of tests/model_grad_bounds.py, without a GPU: the closed-form Jacobians of the
newer families against torch.func.jacfwd of an independent f64 warp, the kernel-order f32 Jacobians and warps within
the roundings the bounds assume (on random events and on events where the Jacobian cancels), and every bound's
magnitude M at least the f64 gradient it bounds."""
import numpy as np
import pytest
import torch

import camera_motion_reference as CM
import camera_rotation_reference as CR
import depth_grid_reference as DR
import depth_grid_timestamp_reference as DTR
import grid_flow_reference as GR
import grid_flow_timestamp_reference as GTR
import model_grad_bounds as B
import planar_motion_reference as P
from exact_bounds import gamma

H, W = 30, 40
CENTRE = (21.5, 13.2)
INTR = (35.1, 32.4, 21.5, 13.2)
PLANAR = {"affine": (3.0, -2.0, 1.5, -0.7, 0.4, 2.2),
          "homography": (3.0, -2.0, 1.5, -0.7, 0.4, 2.2, 0.02, -0.015)}
OMEGA = (2.0, -3.0, 4.0)
VEL = (1.0, -0.8, 1.5)


def _events(seed, n=400):
    rng = np.random.default_rng(seed)
    x = (rng.random(n) * (W - 1)).astype(np.float32)
    y = (rng.random(n) * (H - 1)).astype(np.float32)
    d = (-rng.integers(0, 410, n) / 4096.0).astype(np.float32)
    return x, y, d, rng


def _torch_camera(x, y, d, omega, v, rho, intr):
    """x', y' of the camera motion in f64 torch: exp([d w]x) by torch.linalg.matrix_exp, then + rho d v and the
    projection (independent of the references' scipy rotation and of the kernel's Rodrigues form)"""
    fx, fy, cx, cy = intr[0], intr[1], intr[2], intr[3]
    b = torch.stack(((x - cx) / fx, (y - cy) / fy, torch.ones_like(x)), -1)
    t = d[:, None] * omega[None, :]
    z = torch.zeros_like(d)
    K = torch.stack((torch.stack((z, -t[:, 2], t[:, 1]), -1), torch.stack((t[:, 2], z, -t[:, 0]), -1),
                     torch.stack((-t[:, 1], t[:, 0], z), -1)), 1)
    Pt = torch.einsum("nij,nj->ni", torch.linalg.matrix_exp(K), b) + (rho * d)[:, None] * v[None, :]
    return torch.stack((cx + fx * Pt[:, 0] / Pt[:, 2], cy + fy * Pt[:, 1] / Pt[:, 2]))


def _jacfwd_per_event(fn, prm, n):
    """(2, K, n) from torch.func.jacfwd of fn(prm) -> (2, n)"""
    return torch.func.jacfwd(fn)(torch.tensor(prm, dtype=torch.float64)).permute(0, 2, 1).numpy().reshape(2, -1, n)


@pytest.mark.parametrize("kind", ["affine", "homography"])
def test_planar_jacobian_is_the_derivative_of_the_warp(kind):
    x, y, d, _ = _events(1)
    t = [torch.from_numpy(a.astype(np.float64)) for a in (x, y, d)]
    got = _jacfwd_per_event(lambda q: torch.stack(P.warp_f64(kind, *t, q, CENTRE)), PLANAR[kind], x.size)
    np.testing.assert_allclose(P.jacobian(kind, x, y, d, PLANAR[kind], CENTRE), got, rtol=1e-10, atol=1e-12)


@pytest.mark.parametrize("model", ["camera_rotation", "camera_motion"])
def test_camera_jacobian_is_the_derivative_of_the_warp(model):
    x, y, d, rng = _events(2)
    rho = rng.uniform(0.2, 1.0, x.size)
    t = [torch.from_numpy(a.astype(np.float64)) for a in (x, y, d)]
    r = torch.from_numpy(rho)
    if model == "camera_rotation":
        row = OMEGA + INTR[:2]
        fn = lambda q: _torch_camera(*t, q[:3], torch.zeros(3, dtype=torch.float64), r, (q[3], q[4]) + INTR[2:])  # noqa: E731
        ref = CR.jacobian(x, y, d, OMEGA, INTR)
    else:
        row = OMEGA + VEL + INTR[:2]
        fn = lambda q: _torch_camera(*t, q[:3], q[3:6], r, (q[6], q[7]) + INTR[2:])  # noqa: E731
        ref = CM.jacobian(x, y, d, rho, OMEGA, VEL, INTR)
    np.testing.assert_allclose(ref, _jacfwd_per_event(fn, row, x.size), rtol=1e-9, atol=1e-10)


def test_rho_jacobian_is_the_derivative_of_the_warp():
    x, y, d, rng = _events(3)
    rho = rng.uniform(0.2, 1.0, x.size)
    t = [torch.from_numpy(a.astype(np.float64)) for a in (x, y, d)]
    om, v = torch.tensor(OMEGA, dtype=torch.float64), torch.tensor(VEL, dtype=torch.float64)
    got = torch.func.jacfwd(lambda r: _torch_camera(*t, om, v, r, INTR))(torch.from_numpy(rho))
    got = torch.diagonal(got, dim1=1, dim2=2).numpy()
    np.testing.assert_allclose(DR.rho_jacobian(x, y, d, rho, OMEGA, VEL, INTR), got, rtol=1e-9, atol=1e-10)


def _cancelling(model, seed):
    """events where a Jacobian entry nearly cancels in f32: for the homography's perspective columns nx = u - d sx ~ 0;
    for the camera models and dx'/drho the events near X = vx / vz and Y = vy / vz (the focus of expansion, where
    vx - X vz ~ 0) and near the principal point (X, Y ~ 0)"""
    x, y, d, rng = _events(seed, 300)
    if model in ("camera_motion", "depth"):
        fx, fy, cx, cy = INTR
        x[:150] = (cx + fx * VEL[0] / VEL[2] + rng.uniform(-0.05, 0.05, 150)).astype(np.float32)
        y[:150] = (cy + fy * VEL[1] / VEL[2] + rng.uniform(-0.05, 0.05, 150)).astype(np.float32)
        x[150:] = (cx + rng.uniform(-0.05, 0.05, 150)).astype(np.float32)
        y[150:] = (cy + rng.uniform(-0.05, 0.05, 150)).astype(np.float32)
    elif model == "camera_rotation":
        x[:] = (INTR[2] + rng.uniform(-0.05, 0.05, x.size)).astype(np.float32)
        y[:] = (INTR[3] + rng.uniform(-0.05, 0.05, x.size)).astype(np.float32)
    else:
        x[:] = (CENTRE[0] + rng.uniform(-0.02, 0.02, x.size)).astype(np.float32)
        y[:] = (CENTRE[1] + rng.uniform(-0.02, 0.02, x.size)).astype(np.float32)
    return x, y, d, rng


def _kernel_order(model, x, y, d, rho, kind):
    if model in PLANAR:
        return B.planar_warp_jac(model, x, y, d, PLANAR[model], CENTRE, kind)
    if model == "camera_rotation":
        return B.camera_warp_jac(x, y, d, OMEGA, INTR, kind=kind)
    return B.camera_warp_jac(x, y, d, OMEGA, INTR, v=VEL, rho=rho, kind=kind, depth_only=model == "depth")


def _closed_form(model, x, y, d, rho):
    if model in PLANAR:
        return P.jacobian(model, x, y, d, PLANAR[model], CENTRE)
    if model == "camera_rotation":
        return CR.jacobian(x, y, d, OMEGA, INTR)
    if model == "camera_motion":
        return CM.jacobian(x, y, d, rho, OMEGA, VEL, INTR)
    return DR.rho_jacobian(x, y, d, rho, OMEGA, VEL, INTR)[:, None, :]


def _f64_warp(model, x, y, d, rho):
    if model in PLANAR:
        t = [torch.from_numpy(a.astype(np.float64)) for a in (x, y, d)]
        return [a.numpy() for a in P.warp_f64(model, *t, torch.tensor(PLANAR[model], dtype=torch.float64), CENTRE)]
    if model == "camera_rotation":
        return CR.warp(x, y, d, OMEGA, INTR)
    return CM.warp(x, y, d, rho, OMEGA, VEL, INTR)


MODELS = ["affine", "homography", "camera_rotation", "camera_motion", "depth"]


@pytest.mark.parametrize("events", ["random", "cancelling"])
@pytest.mark.parametrize("model", MODELS)
def test_f32_jacobian_and_warp_within_the_assumed_roundings(model, events):
    x, y, d, rng = _events(4) if events == "random" else _cancelling(model, 5)
    rho = rng.uniform(0.2, 1.0, x.size).astype(np.float32)
    xw32, yw32, J32 = _kernel_order(model, x, y, d, rho, "f32")
    xw64, yw64, J64 = _kernel_order(model, x, y, d, rho, "f64")
    xe, ye, Je = _kernel_order(model, x, y, d, rho, "err")
    J32, J64, Jv, eJ = B.stack(J32, "f32"), B.stack(J64, "f64"), B.stack(Je, "err"), B.stack(Je, "e")
    exact = _closed_form(model, x, y, d, rho.astype(np.float64))
    # the kernel-order f64 evaluation and the running bound's values are the closed form, so the f32 evaluation is the
    # kernel's arithmetic
    for v in (J64, Jv):
        np.testing.assert_allclose(v, exact, rtol=1e-9, atol=1e-9 * np.abs(exact).max())
    # the running bound is first order: 1% covers the rest
    err = np.abs(J32 - exact)
    ratio = err / (1.01 * B.U32 * eJ + 1e-300)
    assert (ratio <= 1).all(), (model, ratio.max())
    # and it is tight: the largest error reaches a sizeable share of its bound (it is not a window-wide worst case)
    assert ratio.max() > 0.05, (model, ratio.max())
    if events == "cancelling":
        # the f32 Jacobian really cancels here: some entry's error is far above u times its own size
        assert (err > 64 * B.U32 * np.abs(exact)).any()
    xr, yr = _f64_warp(model, x, y, d, rho.astype(np.float64))
    for w32, w64, we in ((xw32, xr, xe), (yw32, yr, ye)):
        np.testing.assert_allclose(np.asarray(w64, np.float64), we.v, rtol=1e-9, atol=1e-9)
        pr = np.abs(np.asarray(w32, np.float64) - w64) / (1.01 * B.U32 * we.e)
        assert (pr <= 1).all() and pr.max() > 0.05, (model, pr.max())
        # a few ulps of the event's own coordinates (x' = cx + fx X), not a window-wide magnitude
        scale = np.abs(w64) + (sum(abs(a) for a in INTR) if model not in PLANAR else sum(map(abs, CENTRE)) + W)
        assert (we.e <= 32 * scale).all(), (model, (we.e / scale).max())


def test_err_bounds_one_rounding_per_operation():
    X = B.Err(0.5)
    r = 3.0 - X * 6.0
    assert r.v == 0.0 and r.e == 3.0              # the product's rounding; the exact difference 0 adds nothing
    q = B.Err(1.0) / B.Err(2.0, 4.0)
    assert q.v == 0.5 and q.e == 0.5 * 4.0 / 2.0 + 0.5
    assert B.rounded(0.5).e == 0 and B.rounded(0.1).e > 0


# ---- M >= |g64| ---------------------------------------------------------------------------------------------------

def _stream(seed, sizes):
    rng = np.random.default_rng(seed)
    n = sum(sizes)
    x = (rng.random(n) * (W - 1)).astype(np.float32)
    y = (rng.random(n) * (H - 1)).astype(np.float32)
    d = (-rng.integers(0, 410, n) / 4096.0).astype(np.float32)
    p = (rng.integers(0, 2, n) * 2 - 1).astype(np.float32)
    return x, y, d, p, np.concatenate(([0], np.cumsum(sizes))).astype(np.int64), rng


SIZES = [700, 0, 1, 900]
G = np.array([1.3, -0.4, 0.0, -2.5])


def _rows(family):
    if family in PLANAR:
        return np.array([PLANAR[family], [-1.0, 2.0, -0.5, 0.8, 0.3, -1.2] + ([0.01, 0.02] if family == "homography" else []),
                         PLANAR[family], PLANAR[family]])
    if family == "camera_rotation":
        return np.array([OMEGA + INTR[:2], (-5.0, 1.5, -2.0) + INTR[:2], OMEGA + INTR[:2], (3.5, 4.0, 1.0) + INTR[:2]])
    return np.array([OMEGA + VEL + INTR[:2], (-1.5, 1.5, -2.0, -1.5, 0.5, -1.0) + INTR[:2], OMEGA + VEL + INTR[:2],
                     (0.5, 1.0, -0.5, 0.4, 0.6, 2.0) + INTR[:2]])


def _param_reference(family, loss, x, y, d, tau, p, rho, off, rows, sigma, name):
    p64 = torch.tensor(rows, dtype=torch.float64, requires_grad=True)
    if family in PLANAR:
        out = (P.contrast(family, x, y, d, p, off, p64, sigma, name, 3.0, (H, W), CENTRE) if loss == "contrast" else
               P.timestamp(family, x, y, d, tau, p, off, p64, sigma, (H, W), CENTRE))
    elif family == "camera_rotation":
        out = (CR.contrast(x, y, d, p, off, p64, sigma, name, CENTRE, img_size=(H, W)) if loss == "contrast" else
               CR.timestamp(x, y, d, tau, p, off, p64, sigma, CENTRE, img_size=(H, W)))
    else:
        out = (CM.contrast(x, y, d, p, rho, off, p64, sigma, name, CENTRE, img_size=(H, W)) if loss == "contrast" else
               CM.timestamp(x, y, d, tau, p, rho, off, p64, sigma, CENTRE, img_size=(H, W)))
    (out[0] * torch.from_numpy(G)).sum().backward()
    return p64.grad.numpy(), [a.detach().numpy() for a in out[1:]]


@pytest.mark.parametrize("loss", ["contrast", "timestamp"])
@pytest.mark.parametrize("family", ["affine", "homography", "camera_rotation", "camera_motion"])
def test_parametric_magnitude_bounds_the_gradient(family, loss):
    x, y, d, p, off, rng = _stream(11, SIZES)
    rho = rng.uniform(0.2, 1.0, x.size).astype(np.float32)
    tau = P.tau_f32(d, off)
    rows = _rows(family)
    for sigma, name in ((0.0, "variance"), (1.0, "soe")):
        g64, imgs = _param_reference(family, loss, x, y, d, tau, p, rho, off, rows, sigma, name)
        r = rho if family == "camera_motion" else None
        if loss == "contrast":
            M, c, E = B.param_contrast_bound(family, x, y, d, p, off, rows, sigma, name, 3.0, G, imgs[0], CENTRE, (H, W), r)
        else:
            M, c, E = B.param_timestamp_bound(family, x, y, d, tau, p, off, rows, sigma, G, *imgs, CENTRE, (H, W), r)
        assert (M >= np.abs(g64)).all(), (family, loss, sigma, M, g64)
        assert (M[[1, 2]] == 0).all() and (M[0] > 0).all()       # the empty and the g_b = 0 windows
        assert (c >= 1).all() and (gamma(c) < 1e-2).all()


@pytest.mark.parametrize("family", ["affine", "homography", "camera_rotation"])
def test_segmentation_magnitudes_bound_both_gradients(family):
    x, y, d, p, off, rng = _stream(12, [500, 0, 600])
    rows = _rows(family)
    R3 = np.stack([rows[[0, 1]], rows[[1, 3]], rows[[3, 0]]])
    w = rng.random((x.size, 2)).astype(np.float32)
    g = np.array([[0.7, -1.1], [0.3, 0.2], [-2.0, 0.0]])
    p64 = torch.tensor(R3, dtype=torch.float64, requires_grad=True)
    w64 = torch.tensor(w, dtype=torch.float64, requires_grad=True)
    if family == "camera_rotation":
        f, iwe = CR.segmentation(x, y, d, p, w64, off, p64, 1.0, "variance", CENTRE, img_size=(H, W))
    else:
        f, iwe = P.segmentation(family, x, y, d, p, w64, off, p64, 1.0, "variance", 3.0, (H, W), CENTRE)
    (f * torch.from_numpy(g)).sum().backward()
    M, c, E, Mw, cw, Ew = B.segmentation_bound(family, x, y, d, p, w, off, R3, 1.0, g, iwe.detach().numpy(), CENTRE, (H, W))
    assert (M >= np.abs(p64.grad.numpy())).all()
    assert (Mw >= np.abs(w64.grad.numpy())).all()
    assert (M[2, 1] == 0).all() and (Mw[off[2]:, 1] == 0).all()


@pytest.mark.parametrize("loss", ["contrast", "timestamp"])
def test_grid_flow_magnitude_bounds_the_node_gradient(loss):
    x, y, d, p, off, rng = _stream(13, [800, 0, 1, 600])
    if loss == "timestamp":
        p[::37] = np.nan
    grids = (rng.standard_normal((4, 2, 3, 4)) * 20).astype(np.float32)
    g64 = torch.from_numpy(grids.astype(np.float64)).requires_grad_(True)
    tau = P.tau_f32(d, off)
    for sigma in (0.0, 1.0):
        if loss == "contrast":
            f, iwe = GR.reference(x, y, d, p, off, g64, H, W, sigma, "variance")
            imgs = iwe.detach().numpy()
        else:
            f, T, C = GTR.reference(x, y, d, tau, p, off, g64, H, W, sigma)
            imgs = (T.detach().numpy(), C.detach().numpy())
        g64.grad = None
        (f * torch.from_numpy(G)).sum().backward()
        M, c, E = B.grid_flow_bound(loss, x, y, d, p, off, grids, H, W, sigma, G, imgs, tau=tau)
        assert (M >= np.abs(g64.grad.numpy())).all()
        assert (M[[1, 2]] == 0).all()


@pytest.mark.parametrize("loss", ["contrast", "timestamp"])
def test_depth_grid_magnitude_bounds_the_node_gradient(loss):
    x, y, d, p, off, rng = _stream(14, [800, 0, 1, 600])
    if loss == "timestamp":
        p[::29] = np.nan
    grids = rng.uniform(0.125, 1.0, (4, 3, 4))
    grids[0, 0, 1] = -0.3
    motion = np.array([OMEGA + VEL, (-1.5, 1.5, -2.0, -1.5, 0.5, -1.0), OMEGA + VEL, (0.5, 1.0, -0.5, 0.4, 0.6, 2.0)])
    g64 = torch.from_numpy(grids).requires_grad_(True)
    tau = P.tau_f32(d, off)
    for sigma in (0.0, 1.0):
        if loss == "contrast":
            f, iwe = DR.contrast(x, y, d, p, off, g64, motion, INTR, sigma, "variance", img_size=(H, W))
            imgs = iwe.detach().numpy()
        else:
            f, T, C = DTR.reference(x, y, d, tau, p, off, g64, motion, INTR, sigma, img_size=(H, W))
            imgs = (T.detach().numpy(), C.detach().numpy())
        g64.grad = None
        (f * torch.from_numpy(G)).sum().backward()
        M, c, E = B.depth_grid_bound(loss, x, y, d, p, off, grids, motion, INTR, sigma, G, imgs, (H, W), tau=tau)
        assert (M >= np.abs(g64.grad.numpy())).all()
        assert (M[[1, 2]] == 0).all()
