"""The depth-grid average-timestamp loss (contrast_max/depth_grid_timestamp.py) on the GPU: f, the T and C images and the
node gradient against the f64 reference of tests/depth_grid_timestamp_reference.py for every grid size, blur and stamp
direction, the identities with the per-event camera-motion timestamp loss and with camera_rotation_warp, the candidates
pass and its limits, chunked and empty windows, host syncs and launch counts, and the fit's recovery of the depth
scenes of tests/test_gpu_depth_grid.py beside the contrast fit."""
import ctypes

import numpy as np
import pytest
import torch

import camera_motion_reference as CM
import depth_grid_timestamp_reference as R
from conftest import assert_close_to_max
from test_gpu_depth_grid import (INTR, MOTION, RANGE, SCENE_INTR, H, W, _cuda, _grids, median_errors, recovery_windows,
                                 safe_stream)

pytestmark = pytest.mark.gpu

# the tolerances of tests/test_gpu_depth_grid.py
F_REL, GRAD_REL = 1e-4, 1e-3


def _warp(intr=INTR):
    from event_utils_b200.contrast_max.warps import camera_motion_warp
    return camera_motion_warp(intr)


def ts_stream(seed, sizes, grids, motion, edge=0.1):
    """safe_stream's windows with every 29th polarity NaN (in neither image)"""
    x, y, d, p, off = safe_stream(seed, sizes, grids, motion, edge)
    p[::29] = np.nan
    return x, y, d, p, off


def torch_loss(x, y, d, p, off, grid, motion, sigma=2.0, reverse=False, intr=INTR):
    from event_utils_b200.contrast_max import depth_grid_timestamp_objective_torch
    g = torch.tensor(np.asarray(grid, np.float64), device="cuda", requires_grad=True)
    f = depth_grid_timestamp_objective_torch(*_cuda(x, y, d, p), g, torch.tensor(np.asarray(motion), device="cuda"),
                                             _warp(intr), (H, W), t0=0.0, blur_sigma=sigma, timestamp_reverse=reverse,
                                             batch_end_indices=torch.from_numpy(off[1:]).cuda())
    return f, g


@pytest.mark.parametrize("reverse", [False, True])
@pytest.mark.parametrize("sigma", [0.0, 1.0, 2.0])
@pytest.mark.parametrize("shape", [(2, 2), (3, 4), (12, 16), (H, W)])
def test_forward_images_and_node_gradient_match_the_reference(shape, sigma, reverse):
    rng = np.random.default_rng(hash(shape) % 1000)
    grids = _grids(rng, 3, *shape)
    x, y, d, p, off = ts_stream(7, [3000, 2500, 3500], grids, MOTION)
    f, g = torch_loss(x, y, d, p, off, grids, MOTION, sigma, reverse)
    T, C = (a.cpu().numpy() for a in f.grad_fn.saved_tensors[-2:])      # the images the forward keeps
    f.sum().backward()
    gr = torch.from_numpy(grids).requires_grad_(True)
    fr, Tr, Cr = R.reference(x, y, d, CM.tau_f32(d, off, reverse), p, off, gr, MOTION, INTR, sigma, img_size=(H, W))
    fr.sum().backward()
    assert_close_to_max(f.detach().cpu().numpy(), fr.detach().numpy(), F_REL, "f")
    assert_close_to_max(T, Tr.detach().numpy(), F_REL, "T")
    assert_close_to_max(C, Cr.detach().numpy(), F_REL, "C")
    assert_close_to_max(g.grad.cpu().numpy(), gr.grad.numpy(), GRAD_REL, "grad")
    assert g.grad.abs().max() > 0


def test_identity_with_the_per_event_loss_where_rho_is_the_node():
    """gh = H, gw = W and integer pixels: f is motion_timestamp_objective_torch's with inv_depth = D[b, y, x]"""
    from event_utils_b200.contrast_max import motion_timestamp_objective_torch
    rng = np.random.default_rng(11)
    sizes = [4000, 3000, 5000]
    x = rng.integers(0, W, sum(sizes)).astype(np.float32)
    y = rng.integers(0, H, sum(sizes)).astype(np.float32)
    d = (-rng.integers(0, 410, sum(sizes)) / 4096.0).astype(np.float32)
    p = (rng.integers(0, 2, sum(sizes)) * 2 - 1).astype(np.float32)
    off = np.cumsum([0] + sizes)
    grids = _grids(rng, 3, H, W).astype(np.float32)
    rho = np.concatenate([grids[b][y[off[b]:off[b + 1]].astype(int), x[off[b]:off[b + 1]].astype(int)] for b in range(3)])
    for reverse in (False, True):
        f, _ = torch_loss(x, y, d, p, off, grids, MOTION, 2.0, reverse)
        fm = motion_timestamp_objective_torch(*_cuda(x, y, d, p), torch.tensor(MOTION, device="cuda"), _warp(), t0=0.0,
                                              blur_sigma=2.0, timestamp_reverse=reverse, img_size=(H, W),
                                              batch_end_indices=torch.from_numpy(off[1:]).cuda(),
                                              inv_depth=torch.from_numpy(rho).cuda())
        np.testing.assert_allclose(f.detach().cpu().numpy(), fm.cpu().numpy(), rtol=1e-6)


def test_identities_with_a_constant_grid_and_without_translation():
    from event_utils_b200.contrast_max import camera_rotation_warp, motion_timestamp_objective_torch
    rng = np.random.default_rng(12)
    grids = np.stack([np.full((3, 4), c) for c in (0.3, 0.7, 0.45)]).astype(np.float32)
    x, y, d, p, off = ts_stream(5, [4000, 3000, 5000], grids, MOTION, edge=0.0)
    ends = torch.from_numpy(off[1:]).cuda()
    sample = np.repeat(np.arange(3), np.diff(off))
    f, _ = torch_loss(x, y, d, p, off, grids, MOTION)
    fm = motion_timestamp_objective_torch(*_cuda(x, y, d, p), torch.tensor(MOTION, device="cuda"), _warp(), t0=0.0,
                                          img_size=(H, W), batch_end_indices=ends,
                                          inv_depth=torch.from_numpy(grids[sample, 0, 0].copy()).cuda())
    np.testing.assert_allclose(f.detach().cpu().numpy(), fm.cpu().numpy(), rtol=1e-5)
    still = [m[:3] + (0.0, 0.0, 0.0) for m in MOTION]
    g = _grids(rng, 3, 6, 8)
    g[g < 0] = 0.2
    f0, g0 = torch_loss(x, y, d, p, off, g, still)
    f0.sum().backward()
    fr = motion_timestamp_objective_torch(*_cuda(x, y, d, p), torch.tensor([m[:3] for m in MOTION], device="cuda"),
                                          camera_rotation_warp(INTR), t0=0.0, img_size=(H, W), batch_end_indices=ends)
    np.testing.assert_allclose(f0.detach().cpu().numpy(), fr.cpu().numpy(), rtol=1e-6)
    assert not g0.grad.any()


@pytest.mark.parametrize("J, shape", [(1, (3, 4)), (32, (6, 8)), (32, (16, 24))])
def test_candidates_are_the_objective(J, shape):
    """f[b, j] is the objective at D[b] = candidates[b, j]; (32, 16 x 24) is the n_cand gh gw limit of one pass"""
    from event_utils_b200.contrast_max import depth_grid_timestamp_candidates_torch
    rng = np.random.default_rng(J)
    cand = rng.uniform(0.125, 1.0, (2, J) + shape).astype(np.float32)
    x, y, d, p, off = ts_stream(9, [3000, 4000], cand, MOTION[:2])
    fc = depth_grid_timestamp_candidates_torch(*_cuda(x, y, d, p), torch.from_numpy(cand).cuda(),
                                               torch.tensor(MOTION[:2], device="cuda"), _warp(), (H, W), t0=0.0,
                                               timestamp_reverse=True, batch_end_indices=torch.from_numpy(off[1:]).cuda())
    assert fc.shape == (2, J) and fc.dtype == torch.float64
    for j in range(0, J, max(1, J // 4)):
        f, _ = torch_loss(x, y, d, p, off, cand[:, j], MOTION[:2], reverse=True)
        np.testing.assert_allclose(fc[:, j].cpu().numpy(), f.detach().cpu().numpy(), rtol=1e-6)


def test_chunked_and_empty_windows_change_nothing(monkeypatch):
    from event_utils_b200.contrast_max import depth_grid_timestamp as DG
    rng = np.random.default_rng(21)
    motion = [MOTION[b % 2] for b in range(4)]
    cand = rng.uniform(0.2, 1.0, (4, 40, 3, 4)).astype(np.float32)
    x, y, d, p, off = ts_stream(3, [3000, 0, 2000, 2500], cand[:, :1], motion, edge=0.0)
    args = _cuda(x, y, d, p)
    kw = dict(t0=0.0, blur_sigma=1.0, batch_end_indices=torch.from_numpy(off[1:]).cuda())
    mt = torch.tensor(motion, device="cuda")
    f_all = DG.depth_grid_timestamp_candidates_torch(*args, torch.from_numpy(cand).cuda(), mt, _warp(), (H, W), **kw)
    fit_all = DG.depth_grid_timestamp_fit_torch(*args, mt, _warp(), (H, W), (0.1, 1.2), grid_shapes=((3, 4),), max_iter=3,
                                                num_samples=5, grid_levels=1, **kw)
    monkeypatch.setattr(DG, "TIMESTAMP_CANDIDATES_WORKSPACE_BYTES", 1)     # one window per call
    monkeypatch.setattr(DG, "FIT_WORKSPACE_BYTES", 1)
    f_one = DG.depth_grid_timestamp_candidates_torch(*args, torch.from_numpy(cand).cuda(), mt, _warp(), (H, W), **kw)
    fit_one = DG.depth_grid_timestamp_fit_torch(*args, mt, _warp(), (H, W), (0.1, 1.2), grid_shapes=((3, 4),), max_iter=3,
                                                num_samples=5, grid_levels=1, **kw)
    # the f32 image sums add the taps in any order: only their rounding differs
    np.testing.assert_allclose(f_all.cpu().numpy(), f_one.cpu().numpy(), rtol=1e-6)
    np.testing.assert_allclose(fit_all.inv_depth.cpu().numpy(), fit_one.inv_depth.cpu().numpy(), rtol=0, atol=1e-4)
    f, g = torch_loss(x, y, d, p, off, cand[:, 0], motion, sigma=1.0)
    f.sum().backward()
    assert f[1].item() == 0.0 and not g.grad[1].any() and torch.isfinite(g.grad).all()


def test_candidates_past_the_window_limit_of_one_call():
    """1100 windows of 32 candidates: batch n_cand > 32767, so the windows run in several calls"""
    from event_utils_b200.contrast_max import depth_grid_timestamp_candidates_torch
    B, J, n = 1100, 32, 40
    rng = np.random.default_rng(5)
    x, y = (rng.random(B * n) * (W - 1)).astype(np.float32), (rng.random(B * n) * (H - 1)).astype(np.float32)
    d, p = (-rng.random(B * n) * 0.1).astype(np.float32), (rng.integers(0, 2, B * n) * 2 - 1).astype(np.float32)
    off = np.arange(B + 1) * n
    motion = [MOTION[b % 2] for b in range(B)]
    cand = rng.uniform(0.2, 1.0, (B, J, 2, 2)).astype(np.float32)
    fc = depth_grid_timestamp_candidates_torch(*_cuda(x, y, d, p), torch.from_numpy(cand).cuda(),
                                               torch.tensor(motion, device="cuda"), _warp(), (H, W), t0=0.0,
                                               batch_end_indices=torch.from_numpy(off[1:]).cuda())
    for j in (0, J - 1):
        f, _ = torch_loss(x, y, d, p, off, cand[:, j], motion)
        np.testing.assert_allclose(fc[:, j].cpu().numpy(), f.detach().cpu().numpy(), rtol=1e-6)


def test_no_host_round_trips_and_constant_launch_count():
    from event_utils_b200 import _lib
    from event_utils_b200.contrast_max import depth_grid_timestamp_candidates_torch, depth_grid_timestamp_objective_torch
    L = _lib.lib()
    counts = []
    for sizes in ([40000], [2500] * 16):
        B = len(sizes)
        rng = np.random.default_rng(B)
        grids = rng.uniform(0.2, 1.0, (B, 6, 8))
        motion = torch.tensor([MOTION[b % 2] for b in range(B)], device="cuda")
        n = sum(sizes)
        x, y = (rng.random(n) * (W - 1)).astype(np.float32), (rng.random(n) * (H - 1)).astype(np.float32)
        d, p = (-rng.random(n) * 0.1).astype(np.float32), (rng.integers(0, 2, n) * 2 - 1).astype(np.float32)
        ev = _cuda(x, y, d, p)
        ends = torch.from_numpy(np.cumsum(sizes)).cuda()
        gt = torch.from_numpy(grids).cuda().requires_grad_(True)
        cand = torch.from_numpy(grids).cuda().unsqueeze(1).repeat(1, 5, 1, 1)
        kw = dict(batch_end_indices=ends)
        depth_grid_timestamp_objective_torch(*ev, gt, motion, _warp(), (H, W), **kw).sum().backward()   # warm-up
        depth_grid_timestamp_candidates_torch(*ev, cand, motion, _warp(), (H, W), **kw)
        torch.cuda.synchronize()
        L.evk_prof_enable(1)
        torch.cuda.set_sync_debug_mode("error")
        try:
            f = depth_grid_timestamp_objective_torch(*ev, gt, motion, _warp(), (H, W), **kw)
            f.sum().backward()
            depth_grid_timestamp_candidates_torch(*ev, cand, motion, _warp(), (H, W), **kw)
        finally:
            torch.cuda.set_sync_debug_mode(0)
        ms, timed, launches = ctypes.c_double(), ctypes.c_longlong(), ctypes.c_longlong()
        _lib.check(L.evk_prof_collect(ctypes.byref(ms), ctypes.byref(timed), ctypes.byref(launches)))
        L.evk_prof_enable(0)
        assert torch.isfinite(gt.grad).all()
        counts.append(launches.value)
    assert counts[0] == counts[1] and counts[0] > 0, counts


# the median relative error of the fitted rho at the scenes' points: the largest of three H100 runs, with margin
RECOVERY_TOL = (0.02, 0.025, 0.03)


def test_fit_recovers_depth_from_a_known_motion():
    from event_utils_b200.contrast_max import (depth_grid_fit_torch, depth_grid_timestamp_candidates_torch,
                                              depth_grid_timestamp_fit_torch)
    (x, y, t, p), ends, motion, truth = recovery_windows()
    ev = _cuda(x, y, t, p)
    kw = dict(batch_end_indices=torch.from_numpy(ends).cuda())
    mt = torch.from_numpy(motion).cuda()
    fit = depth_grid_timestamp_fit_torch(*ev, mt, _warp(SCENE_INTR), (180, 240), RANGE, **kw)
    D = fit.inv_depth.cpu().numpy()
    assert D.shape == (3, 12, 16) and (D >= RANGE[0]).all() and (D <= RANGE[1]).all()
    err = median_errors(D, truth)
    # the best constant inverse depth of every window, from a fine scan of the box
    consts = np.linspace(RANGE[0], RANGE[1], 32)
    fc = depth_grid_timestamp_candidates_torch(*ev, torch.from_numpy(np.broadcast_to(consts[None, :, None, None],
                                                                                       (3, 32, 3, 4)).copy()).cuda(),
                                               mt, _warp(SCENE_INTR), (180, 240), **kw).cpu().numpy()
    best = consts[fc.argmin(1)]
    err_const = [float(np.median(np.abs(best[b] - r) / r)) for b, (_, _, r) in enumerate(truth)]
    contrast = depth_grid_fit_torch(*ev, mt, _warp(SCENE_INTR), (180, 240), RANGE, **kw).inv_depth.cpu().numpy()
    contrast = median_errors(contrast, truth)
    print("median relative rho error: timestamp fit %s, contrast fit %s, best constant %s"
          % (np.round(err, 4), np.round(contrast, 4), np.round(err_const, 4)))
    assert all(e <= tol for e, tol in zip(err, RECOVERY_TOL)), err
    assert all(e <= 0.5 * c for e, c in zip(err, err_const)), (err, err_const)
