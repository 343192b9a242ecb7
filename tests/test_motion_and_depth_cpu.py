"""No-GPU checks of the joint motion-and-depth loss and fit (contrast_max/motion_and_depth.py): the f64 reference's
gradient in all six motion components and in a sample of nodes against central differences, the direction chart of
the fit and its chain rule, and every argument error raised before the library is loaded."""
import numpy as np
import pytest
import torch

import motion_and_depth_reference as MR

H, W = 24, 32
INTR = (28.3, 25.9, 17.4, 10.2)
MOTION = [(2.0, -3.0, 4.0, 1.0, -0.8, 1.5), (-1.5, 1.5, -2.0, -1.5, 0.5, -1.0)]


def _events(seed, sizes):
    rng = np.random.default_rng(seed)
    n = sum(sizes)
    x = (rng.random(n) * (W - 1)).astype(np.float32)
    y = (rng.random(n) * (H - 1)).astype(np.float32)
    d = (-rng.random(n) * 0.1).astype(np.float32)
    p = (rng.integers(0, 2, n) * 2 - 1).astype(np.float32)
    return x, y, d, p, np.cumsum([0] + sizes)


@pytest.mark.parametrize("name", ["variance", "sos", "soe", "sosa"])
def test_reference_gradient_matches_central_differences(name):
    x, y, d, p, off = _events(1, [600, 500])
    rng = np.random.default_rng(2)
    grid0 = rng.uniform(0.3, 1.0, (2, 3, 4))
    m0 = np.array(MOTION)

    def f(grid, motion):
        return MR.contrast(x, y, d, p, off, torch.from_numpy(grid), torch.from_numpy(motion), INTR, 1.0, name,
                           img_size=(H, W), exact=True).numpy()
    g = torch.from_numpy(grid0).requires_grad_(True)
    m = torch.from_numpy(m0).requires_grad_(True)
    MR.contrast(x, y, d, p, off, g, m, INTR, 1.0, name, img_size=(H, W), exact=True).sum().backward()
    h = 1e-6
    for k in range(6):
        e = np.zeros_like(m0)
        e[:, k] = h
        fd = (f(grid0, m0 + e) - f(grid0, m0 - e)) / (2 * h)
        np.testing.assert_allclose(m.grad[:, k].numpy(), fd, rtol=1e-4, atol=1e-6 * np.abs(fd).max() + 1e-12)
    for b, i, j in [(0, 0, 0), (0, 1, 2), (1, 2, 3), (1, 0, 1)]:
        e = np.zeros_like(grid0)
        e[b, i, j] = h
        fd = (f(grid0 + e, m0) - f(grid0 - e, m0)) / (2 * h)
        np.testing.assert_allclose(g.grad[b, i, j].item(), fd[b], rtol=1e-4, atol=1e-6 * abs(fd[b]) + 1e-12)


def test_chart_round_trips():
    from event_utils_b200.contrast_max.motion_and_depth import _chart_frame, _chart_gradient, _chart_velocity
    rng = np.random.default_rng(3)
    v0 = torch.from_numpy(np.vstack([rng.normal(size=(5, 3)), [[0.0, 0.0, 2.0], [1e-3, 0.0, 0.0]]]))
    frame = _chart_frame(v0)
    vh, e1, e2, speed = frame
    eye = torch.stack((vh, e1, e2), 1)
    np.testing.assert_allclose((eye @ eye.transpose(1, 2)).numpy(), np.broadcast_to(np.eye(3), (7, 3, 3)), atol=1e-12)
    np.testing.assert_allclose(_chart_velocity(torch.zeros(7, 2, dtype=torch.float64), frame).numpy(), v0.numpy(),
                               rtol=1e-12, atol=1e-15)
    ab = torch.from_numpy(rng.uniform(-1, 1, (7, 2)))
    v = _chart_velocity(ab, frame)
    np.testing.assert_allclose(v.norm(dim=1).numpy(), v0.norm(dim=1).numpy(), rtol=1e-12)
    gv = torch.from_numpy(rng.normal(size=(7, 3)))
    g = _chart_gradient(ab, frame, gv).numpy()
    h = 1e-6
    for k in range(2):
        e = torch.zeros_like(ab)
        e[:, k] = h
        fd = ((_chart_velocity(ab + e, frame) - _chart_velocity(ab - e, frame)) * gv).sum(1) / (2 * h)
        np.testing.assert_allclose(g[:, k], fd.numpy(), rtol=1e-6, atol=1e-9)


@pytest.fixture
def no_library(monkeypatch):
    from event_utils_b200 import _lib

    def touched():
        raise AssertionError("the library was loaded before the argument check")
    monkeypatch.setattr(_lib, "lib", touched)


def _warp():
    from event_utils_b200.contrast_max.warps import camera_motion_warp
    return camera_motion_warp(INTR)


def test_argument_errors_come_before_the_library(no_library):
    from event_utils_b200.contrast_max import (camera_rotation_warp, motion_and_depth_contrast_candidates_torch,
                                               motion_and_depth_contrast_objective_torch, motion_and_depth_fit_torch)
    x = torch.zeros(10)
    grid = torch.ones(2, 3, 4)
    ends = [5, 10]
    obj = motion_and_depth_contrast_objective_torch
    cand = motion_and_depth_contrast_candidates_torch
    fit = motion_and_depth_fit_torch
    ok_motion = torch.tensor(MOTION)
    bad = [
        lambda: obj(x, x, x, x, grid, ok_motion, camera_rotation_warp(INTR), (H, W), batch_end_indices=ends),
        lambda: obj(x, x, x, x, grid, ok_motion, _warp(), (H, W), objective="moa", batch_end_indices=ends),
        lambda: obj(x, x, x, x, grid, ok_motion, _warp(), (H, W), objective="isoa", batch_end_indices=ends),
        lambda: obj(x, x, x, x, grid, ok_motion[:, :5], _warp(), (H, W), batch_end_indices=ends),
        lambda: obj(x, x, x, x, grid, ok_motion[0, :5], _warp(), (H, W), batch_end_indices=ends),
        lambda: obj(x, x, x, x, grid, torch.zeros(3, 6), _warp(), (H, W), batch_end_indices=ends),
        lambda: obj(x, x, x, x, torch.ones(2, 1, 4), ok_motion, _warp(), (H, W), batch_end_indices=ends),
        lambda: obj(x, x, x, x, torch.ones(2, 65, 64), ok_motion, _warp(), (100, 100), batch_end_indices=ends),
        lambda: cand(x, x, x, x, torch.zeros(2, 3, 6), torch.ones(2, 4, 3, 4), _warp(), (H, W), batch_end_indices=ends),
        lambda: cand(x, x, x, x, torch.zeros(2, 0, 6), torch.ones(2, 0, 3, 4), _warp(), (H, W), batch_end_indices=ends),
        lambda: cand(x, x, x, x, torch.zeros(2, 6), torch.ones(2, 1, 3, 4), _warp(), (H, W), batch_end_indices=ends),
        lambda: cand(x, x, x, x, torch.zeros(2, 1, 6), torch.ones(2, 1, 3, 4), _warp(), (H, W), objective="moa",
                     batch_end_indices=ends),
        lambda: cand(x, x, x, x, torch.zeros(2, 1, 6), torch.ones(2, 1, 3, 4), camera_rotation_warp(INTR), (H, W),
                     batch_end_indices=ends),
        lambda: fit(x, x, x, x, _warp(), (H, W), None, (0.1, 1.0), batch_end_indices=ends),
        lambda: fit(x, x, x, x, _warp(), (H, W), (0.1, 0.2, 0.3, 0.0, 0.0, 0.0), (0.1, 1.0), batch_end_indices=ends),
        lambda: fit(x, x, x, x, _warp(), (H, W), [MOTION[0], (0, 0, 0, 0, 0, 0)], (0.1, 1.0), batch_end_indices=ends),
        lambda: fit(x, x, x, x, _warp(), (H, W), ok_motion, None, batch_end_indices=ends),
        lambda: fit(x, x, x, x, _warp(), (H, W), ok_motion, (1.0, 0.5), batch_end_indices=ends),
        lambda: fit(x, x, x, x, _warp(), (H, W), ok_motion, (0.1, 1.0), grid_shapes=((1, 4),), batch_end_indices=ends),
        lambda: fit(x, x, x, x, _warp(), (H, W), ok_motion, (0.1, 1.0), objective="isoa", batch_end_indices=ends),
        lambda: fit(x, x, x, x, camera_rotation_warp(INTR), (H, W), ok_motion, (0.1, 1.0), batch_end_indices=ends),
        lambda: fit(x, x, x, x, _warp(), (H, W), ok_motion[:, :3], (0.1, 1.0), batch_end_indices=ends),
        lambda: fit(x, x, x, x, _warp(), (H, W), ok_motion, (0.1, 1.0), inv_depth0=torch.ones(6, 8),
                    batch_end_indices=ends),
        lambda: fit(x, x, x, x, _warp(), (H, W), ok_motion, (0.1, 1.0), rotation_scale=0.0, batch_end_indices=ends),
        lambda: fit(x, x, x, x, _warp(), (H, W), ok_motion, (0.1, 1.0), line_search_steps=33, batch_end_indices=ends),
        lambda: fit(x, x, x, x, _warp(), (H, W), ok_motion, (0.1, 1.0), num_samples=4, batch_end_indices=ends),
    ]
    for i, call in enumerate(bad):
        with pytest.raises(ValueError):
            call()
            pytest.fail("case %d raised nothing" % i)


def test_fit_rejects_more_than_512_unknowns_by_the_motion_parameters(no_library):
    """K = 5 + gh gw: a 4 x 127 grid (508 nodes, which depth_grid_fit_torch takes) is one unknown too many"""
    from event_utils_b200.contrast_max import motion_and_depth_fit_torch
    x = torch.zeros(10)
    with pytest.raises(ValueError, match="K = 5 \\+ gh gw <= 512"):
        motion_and_depth_fit_torch(x, x, x, x, _warp(), (100, 300), MOTION[0], (0.1, 1.0), grid_shapes=((4, 127),))
