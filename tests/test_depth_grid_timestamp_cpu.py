"""The depth-grid average-timestamp loss without a GPU: its f64 reference against the per-event camera-motion timestamp
reference where the interpolated rho is the node, the reference's node gradient against central differences and at
v = 0, and the argument checks of the three torch functions and the C entries, which all run before any CUDA call."""
import ctypes

import numpy as np
import pytest
import torch

import camera_motion_reference as CM
import depth_grid_reference as DR
import depth_grid_timestamp_reference as R

H, W = 12, 16
INTR = (14.3, 12.9, 8.7, 5.2)
MOTION = [(2.0, -3.0, 4.0, 1.0, -0.8, 1.5), (-1.0, 1.5, -2.0, -1.5, 0.5, 2.0)]


def _events(seed, n, integer=False):
    rng = np.random.default_rng(seed)
    if integer:
        x, y = rng.integers(0, W, n).astype(np.float32), rng.integers(0, H, n).astype(np.float32)
    else:
        x, y = (rng.random(n) * (W - 1)).astype(np.float32), (rng.random(n) * (H - 1)).astype(np.float32)
    d = (-rng.integers(0, 410, n) / 4096.0).astype(np.float32)
    p = (rng.integers(0, 2, n) * 2 - 1).astype(np.float32)
    p[::37] = np.nan                                          # in neither polarity image
    return x, y, d, p


@pytest.mark.parametrize("sigma", [0.0, 2.0])
def test_reference_is_the_camera_motion_reference_where_rho_is_the_node(sigma):
    """gh = H, gw = W and events on integer pixels: every event's rho is its pixel's node"""
    x, y, d, p = _events(0, 400, integer=True)
    off = np.array([0, 250, 400])
    tau = CM.tau_f32(d, off)
    rng = np.random.default_rng(1)
    grid = rng.uniform(0.1, 1.0, (2, H, W))
    grid[0, 3, 4] = -0.5                                      # a negative node: its events are dropped
    f, T, C = R.reference(x, y, d, tau, p, off, torch.from_numpy(grid), MOTION, INTR, sigma, img_size=(H, W))
    rho = np.concatenate([grid[b][y[off[b]:off[b + 1]].astype(int), x[off[b]:off[b + 1]].astype(int)]
                          for b in range(2)]).astype(np.float32)
    rows = torch.tensor([list(m) + list(INTR[:2]) for m in MOTION], dtype=torch.float64)
    fr, Tr, Cr = CM.timestamp(x, y, d, tau, p, rho, off, rows, sigma, INTR[2:], img_size=(H, W))
    np.testing.assert_allclose(f.numpy(), fr.detach().numpy(), rtol=1e-12)
    np.testing.assert_allclose(T.numpy(), Tr.detach().numpy(), rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(C.numpy(), Cr.numpy(), rtol=1e-12)


@pytest.mark.parametrize("reverse", [False, True])
def test_reference_node_gradient_matches_central_differences(reverse):
    x, y, d, p = _events(2, 600)
    off = np.array([0, 600])
    rng = np.random.default_rng(3)
    grid = rng.uniform(0.3, 1.0, (1, 3, 4))
    motion = [MOTION[0]]
    # events whose warp lies at least 0.02 px from every integer: the steps below move no floor
    r32 = DR.event_rho_f32(x, y, grid[0], H, W)
    xw, yw = CM.warp(x, y, d, r32, motion[0][:3], motion[0][3:], INTR)
    with np.errstate(invalid="ignore"):
        ok = np.isfinite(xw) & np.isfinite(yw) & (np.abs(xw - np.round(xw)) > 0.02) & (np.abs(yw - np.round(yw)) > 0.02)
    x, y, d, p = x[ok], y[ok], d[ok], p[ok]
    off = np.array([0, int(ok.sum())])
    tau = CM.tau_f32(d, off, reverse)
    g = torch.from_numpy(grid).requires_grad_(True)
    f = R.reference(x, y, d, tau, p, off, g, motion, INTR, 1.0, img_size=(H, W))[0]
    (grad,) = torch.autograd.grad(f.sum(), g)
    assert grad.abs().max() > 0
    h = 3e-4
    num = np.zeros_like(grid)
    for i in range(3):
        for j in range(4):
            e = np.zeros_like(grid)
            e[0, i, j] = h
            fp = R.reference(x, y, d, tau, p, off, torch.from_numpy(grid + e), motion, INTR, 1.0, img_size=(H, W))[0]
            fm = R.reference(x, y, d, tau, p, off, torch.from_numpy(grid - e), motion, INTR, 1.0, img_size=(H, W))[0]
            num[0, i, j] = (fp - fm).item() / (2 * h)
    np.testing.assert_allclose(grad.numpy(), num, rtol=0, atol=2e-3 * np.abs(num).max())


def test_reference_gradient_is_zero_without_translation():
    x, y, d, p = _events(4, 300)
    off = np.array([0, 300])
    g = torch.full((1, 3, 4), 0.5, dtype=torch.float64, requires_grad=True)
    f = R.reference(x, y, d, CM.tau_f32(d, off), p, off, g, [(2.0, -1.0, 3.0, 0.0, 0.0, 0.0)], INTR, 1.0,
                    img_size=(H, W))[0]
    (grad,) = torch.autograd.grad(f.sum(), g)
    assert not grad.any()


def _cpu_events():
    x = torch.zeros(8)
    return x, x, torch.arange(8.0), x


def _warp():
    from event_utils_b200.contrast_max.warps import camera_motion_warp
    return camera_motion_warp(INTR)


def test_argument_checks_run_before_any_cuda_call():
    from event_utils_b200.contrast_max import (camera_rotation_warp, depth_grid_timestamp_candidates_torch,
                                              depth_grid_timestamp_fit_torch, depth_grid_timestamp_objective_torch)
    x, y, t, p = _cpu_events()
    m = torch.zeros(6)
    obj, cand = depth_grid_timestamp_objective_torch, depth_grid_timestamp_candidates_torch
    fit = depth_grid_timestamp_fit_torch
    nan = float("nan")
    with pytest.raises(ValueError, match="camera_motion_warp"):
        obj(x, y, t, p, torch.zeros(3, 4), m, camera_rotation_warp(INTR), (H, W))
    with pytest.raises(ValueError, match="camera_motion_warp"):
        cand(x, y, t, p, torch.zeros(1, 2, 3, 4), m, None, (H, W))
    with pytest.raises(ValueError, match="camera_motion_warp"):
        fit(x, y, t, p, m, object(), (H, W), (0.1, 1.0))
    with pytest.raises(ValueError, match="node grid"):
        obj(x, y, t, p, torch.zeros(13, 4), m, _warp(), (H, W))
    with pytest.raises(ValueError, match="node grid"):
        obj(x, y, t, p, torch.zeros(1, 65, 65), m, _warp(), (100, 100))
    with pytest.raises(ValueError, match=r"\(B,gh,gw\) or \(gh,gw\)"):
        obj(x, y, t, p, torch.zeros(4), m, _warp(), (H, W))
    with pytest.raises(ValueError, match="floating-point"):
        obj(x, y, t, p, torch.zeros(3, 4, dtype=torch.int32), m, _warp(), (H, W))
    with pytest.raises(ValueError, match="motion must have shape"):
        obj(x, y, t, p, torch.zeros(2, 3, 4), torch.zeros(3, 6), _warp(), (H, W))
    with pytest.raises(ValueError, match="blur_sigma must be a number"):
        obj(x, y, t, p, torch.zeros(3, 4), m, _warp(), (H, W), blur_sigma=nan)
    with pytest.raises(ValueError, match="must not require grad"):
        obj(torch.zeros(8, requires_grad=True), y, t, p, torch.zeros(3, 4), m, _warp(), (H, W))
    with pytest.raises(ValueError, match=r"\(B,J,gh,gw\) with J >= 1"):
        cand(x, y, t, p, torch.zeros(1, 0, 3, 4), m, _warp(), (H, W))
    with pytest.raises(ValueError, match="node grid"):
        cand(x, y, t, p, torch.zeros(1, 2, 1, 4), m, _warp(), (H, W))
    with pytest.raises(ValueError, match="motion must have shape"):
        cand(x, y, t, p, torch.zeros(2, 2, 3, 4), torch.zeros(3, 6), _warp(), (H, W))
    with pytest.raises(ValueError, match="blur_sigma must be a number"):
        cand(x, y, t, p, torch.zeros(1, 2, 3, 4), m, _warp(), (H, W), blur_sigma=nan)
    with pytest.raises(ValueError, match="needs inv_depth_range"):
        fit(x, y, t, p, m, _warp(), (H, W), None)
    with pytest.raises(ValueError, match="0 <= lo < hi"):
        fit(x, y, t, p, m, _warp(), (H, W), (-0.1, 1.0))
    with pytest.raises(ValueError, match="0 <= lo < hi"):
        fit(x, y, t, p, m, _warp(), (H, W), (1.0, 1.0))
    with pytest.raises(ValueError, match="0 <= lo < hi"):
        fit(x, y, t, p, m, _warp(), (H, W), (1.0, 0.5))
    with pytest.raises(ValueError, match="inv_depth_range must have shape"):
        fit(x, y, t, p, m, _warp(), (H, W), (0.1, 0.5, 1.0))
    with pytest.raises(ValueError, match="K = gh gw <= 512"):
        fit(x, y, t, p, m, _warp(), (100, 100), (0.1, 1.0), grid_shapes=((3, 4), (16, 33)))
    with pytest.raises(ValueError, match="node grid"):
        fit(x, y, t, p, m, _warp(), (H, W), (0.1, 1.0), grid_shapes=((13, 4),))
    with pytest.raises(ValueError, match="at least one"):
        fit(x, y, t, p, m, _warp(), (H, W), (0.1, 1.0), grid_shapes=())
    with pytest.raises(ValueError, match="smoothness"):
        fit(x, y, t, p, m, _warp(), (H, W), (0.1, 1.0), smoothness=-1.0)
    with pytest.raises(ValueError, match="smoothness"):
        fit(x, y, t, p, m, _warp(), (H, W), (0.1, 1.0), charbonnier_eps=0.0)
    with pytest.raises(ValueError, match="x0 must have shape"):
        fit(x, y, t, p, m, _warp(), (H, W), (0.1, 1.0), x0=torch.zeros(4, 3))
    with pytest.raises(ValueError, match="num_samples must be odd"):
        fit(x, y, t, p, m, _warp(), (H, W), (0.1, 1.0), num_samples=4)
    with pytest.raises(ValueError, match="line_search_steps"):
        fit(x, y, t, p, m, _warp(), (H, W), (0.1, 1.0), line_search_steps=0)
    with pytest.raises(ValueError, match="blur_sigma must be a number or"):
        fit(x, y, t, p, m, _warp(), (H, W), (0.1, 1.0), blur_sigma=[])
    with pytest.raises(ValueError, match="blur_sigma must be a number, got NaN"):
        fit(x, y, t, p, m, _warp(), (H, W), (0.1, 1.0), blur_sigma=[2.0, nan])
    with pytest.raises(ValueError, match="motion must have shape"):
        fit(x, y, t, p, torch.zeros(5), _warp(), (H, W), (0.1, 1.0))


def test_entry_limits_and_workspace_queries():
    """the queries are the grid flow's timestamp queries, 0 for rejected arguments, and the entries reject bad limits,
    a null motion or tau, a NaN blur sigma and a short workspace with their codes before any CUDA call"""
    from event_utils_b200 import _lib
    L = _lib.load()
    q, qc = L.evk_depth_grid_timestamp_objective_workspace_bytes, L.evk_depth_grid_timestamp_candidates_workspace_bytes
    for args in ((4, 12, 16, 480, 640), (32767, 2, 2, 4, 4)):
        assert q(*args) == L.evk_grid_flow_timestamp_objective_workspace_bytes(*args) > 0
    for args in ((1, 64, 65, 480, 640), (1, 13, 4, 12, 16), (32768, 2, 2, 4, 4), (-1, 2, 2, 4, 4), (1, 1, 4, 12, 16)):
        assert q(*args) == 0
    for args in ((2, 8, 12, 16, 480, 640), (1, 3, 64, 64, 480, 640), (1023, 32, 2, 2, 4, 4)):
        assert qc(*args) == L.evk_grid_flow_timestamp_candidates_workspace_bytes(*args) > 0
    for args in ((1, 4, 64, 64, 480, 640), (1, 33, 2, 2, 480, 640), (1024, 32, 2, 2, 4, 4), (1, 0, 3, 4, 12, 16)):
        assert qc(*args) == 0            # n_cand gh gw <= 12288, n_cand <= 32, batch n_cand <= 32767
    one = ctypes.c_void_p(256)
    ws = ctypes.c_void_p(1 << 20)
    big = 1 << 40
    obj, grad, cand = (L.evk_depth_grid_timestamp_objective_f32, L.evk_depth_grid_timestamp_objective_grad_f32,
                       L.evk_depth_grid_timestamp_candidates_f32)
    ev = (one,) * 6
    assert obj(*ev, 1, 10, one, 1.0, 2.0, one, 64, 65, 480, 640, 1.0, one, one, one, ws, big, None) == -1
    assert b"gh gw <= 4096" in L.evk_last_error()
    assert obj(*ev, 32768, 10, one, 1.0, 2.0, one, 2, 2, 4, 4, 1.0, one, one, one, ws, big, None) == -1
    assert grad(*ev, 1, 10, one, 1.0, 2.0, one, 1, 4, 12, 16, 1.0, one, one, one, one, ws, big, None) == -1
    assert obj(*ev, 1, 10, None, 1.0, 2.0, one, 3, 4, 12, 16, 1.0, one, one, one, ws, big, None) == -1
    assert b"null motion" in L.evk_last_error()
    assert obj(one, one, one, None, one, one, 1, 10, one, 1.0, 2.0, one, 3, 4, 12, 16, 1.0, one, one, one, ws, big,
               None) == -1                                      # no stamps
    assert grad(*ev, 1, 10, one, 1.0, 2.0, one, 3, 4, 12, 16, 1.0, one, one, None, one, ws, big, None) == -1
    assert b"null array" in L.evk_last_error()
    assert cand(*ev, 1, 10, one, 1.0, 2.0, one, 4, 64, 64, 480, 640, 1.0, one, ws, big, None) == -1
    assert cand(*ev, 1, 10, one, 1.0, 2.0, one, 33, 2, 2, 12, 16, 1.0, one, ws, big, None) == -1
    assert cand(*ev, 1024, 10, one, 1.0, 2.0, one, 32, 2, 2, 4, 4, 1.0, one, ws, big, None) == -1
    assert b"batch n_cand <= 32767" in L.evk_last_error()
    assert obj(*ev, 1, 10, one, 1.0, 2.0, one, 3, 4, 12, 16, 1.0, one, one, one, ws, 16, None) == -3   # workspace
    assert cand(*ev, 1, 10, one, 1.0, 2.0, one, 2, 3, 4, 12, 16, 1.0, one, ws, 16, None) == -3
    for entry, args in ((obj, (one, one, one)), (cand, (one,))):
        nj = (2,) if entry is cand else ()
        assert entry(*ev, 1, 10, one, 1.0, 2.0, one, *nj, 3, 4, 12, 16, float("nan"), *args, ws, big, None) == -1
        assert b"blur sigma" in L.evk_last_error()
