"""The joint motion-and-depth contrast loss (contrast_max/motion_and_depth.py) on the GPU: f against the depth-grid
loss, the node gradient against the depth grid's, the motion gradient against the f64 reference and against the
per-event camera-motion loss at the same rho, the joint candidates pass, window limits, empty and skewed windows, NaN
events, chunked windows, host syncs and launch counts, and the joint fit's recovery of the three depth-grid scenes from
a wrong start motion."""
import ctypes

import numpy as np
import pytest
import torch

import camera_motion_reference as CM
import depth_grid_reference as R
import model_grad_bounds as GB
import motion_and_depth_reference as MR
import test_gpu_depth_grid as DG
from conftest import assert_close_to_max
from grid_flow_reference import node_taps
from motion_objective_reference import contributes

pytestmark = pytest.mark.gpu

H, W, INTR, MOTION, OBJECTIVES = DG.H, DG.W, DG.INTR, DG.MOTION, DG.OBJECTIVES
_cuda, _warp, safe_stream = DG._cuda, DG._warp, DG.safe_stream


def joint_loss(x, y, d, p, off, grid, motion, name="variance", sigma=1.0, intr=INTR, size=(H, W)):
    from event_utils_b200.contrast_max import motion_and_depth_contrast_objective_torch
    g = torch.tensor(np.asarray(grid, np.float64), device="cuda", requires_grad=True)
    m = torch.tensor(np.asarray(motion, np.float64), device="cuda", requires_grad=True)
    f = motion_and_depth_contrast_objective_torch(*_cuda(x, y, d, p), g, m, _warp(intr), size, t0=0.0, objective=name,
                                                  blur_sigma=sigma, batch_end_indices=torch.from_numpy(off[1:]).cuda())
    return f, g, m


def event_rho(x, y, off, grids):
    return np.concatenate([R.event_rho_f32(x[off[b]:off[b + 1]], y[off[b]:off[b + 1]], grids[b], H, W)
                           for b in range(len(off) - 1)])


def check_motion_bounds(x, y, d, p, off, grids, motion, name, got, what):
    """every window's every motion component within the f32 rounding bound of tests/model_grad_bounds.py for the
    camera-motion contrast gradient at the kernel's rho (grad_f = 1)"""
    rho = event_rho(x, y, off, grids)
    rows = np.array([tuple(m) + INTR[:2] for m in motion], np.float64)
    p64 = torch.tensor(rows, requires_grad=True)
    f, iwe = CM.contrast(x, y, d, p, rho, off, p64, 1.0, name, INTR[2:], img_size=(H, W))
    f.sum().backward()
    M, c, E = GB.param_contrast_bound("camera_motion", x, y, d, p, off, rows, 1.0, name, 3.0, np.ones(len(rows)),
                                      iwe.detach().numpy(), INTR[2:], (H, W), rho)
    GB.check(got, p64.grad.numpy()[:, :6], M[:, :6], c[:, :6], E[:, :6], what)


@pytest.mark.parametrize("shape", [(3, 4), (12, 16)])
@pytest.mark.parametrize("name", OBJECTIVES)
def test_forward_and_both_gradients(shape, name):
    rng = np.random.default_rng(hash(shape) % 1000 + 7)
    grids = DG._grids(rng, 3, *shape)
    x, y, d, p, off = safe_stream(7, [3000, 2500, 3500], grids, MOTION)
    f, g, m = joint_loss(x, y, d, p, off, grids, MOTION, name)
    f.sum().backward()
    f0, g0 = DG.torch_loss(x, y, d, p, off, grids, MOTION, name)
    f0.sum().backward()
    # the same forward entry; the f32 image sums add the taps in any order, so two calls agree to their rounding
    np.testing.assert_allclose(f.detach().cpu().numpy(), f0.detach().cpu().numpy(), rtol=1e-6)
    assert_close_to_max(g.grad.cpu().numpy(), g0.grad.cpu().numpy(), 1e-5, "node gradient against the depth grid's")
    gr = torch.from_numpy(grids).requires_grad_(True)
    mr = torch.tensor(MOTION, dtype=torch.float64, requires_grad=True)
    MR.contrast(x, y, d, p, off, gr, mr, INTR, 1.0, name, img_size=(H, W)).sum().backward()
    for k in range(6):
        assert_close_to_max(m.grad[:, k].cpu().numpy(), mr.grad[:, k].numpy(), DG.GRAD_REL, "motion component %d" % k)
    assert_close_to_max(g.grad.cpu().numpy(), gr.grad.numpy(), DG.GRAD_REL, "node gradient against the reference")
    check_motion_bounds(x, y, d, p, off, grids, MOTION, name, m.grad.cpu().numpy(), "motion %s %s" % (shape, name))


def outside_stream(seed, sizes, grids, motion):
    """Windows of events half on the sensor and half in a band up to 8 px around it, beyond the outer node row or
    column (no node cell: rho = 0, the rotation-only warp), with safe_stream's rule against f32 tap and keep flips"""
    rng = np.random.default_rng(seed)
    out, ends = [[] for _ in range(4)], []
    for b, n in enumerate(sizes):
        gh, gw = grids[b].shape
        x = (rng.random(4 * n) * (W - 1 + 16) - 8).astype(np.float32)
        y = (rng.random(4 * n) * (H - 1 + 16) - 8).astype(np.float32)
        none = ~node_taps(x, y, gh, gw, H, W)[3].any(1)
        x = np.concatenate([x[none][: n // 2], (rng.random(n - n // 2) * (W - 1)).astype(np.float32)])
        y = np.concatenate([y[none][: n // 2], (rng.random(n - n // 2) * (H - 1)).astype(np.float32)])
        m = x.size
        d = (-rng.integers(0, 410, m) / 4096.0).astype(np.float32)
        p = (rng.integers(0, 2, m) * 2 - 1).astype(np.float32)
        xw, yw = CM.warp(x, y, d, R.event_rho_f32(x, y, grids[b], H, W), motion[b][:3], motion[b][3:], INTR)
        ok = np.ones(m, bool)
        for c in (xw, yw):
            with np.errstate(invalid="ignore"):
                ok &= ~np.isfinite(c) | (np.abs(c - np.round(c)) >= 1e-3)
        for o, a in zip(out, (x, y, d, p)):
            o.append(a[ok])
        ends.append(sum(a.size for a in out[0]))
    return [np.concatenate(o) for o in out] + [np.array([0] + ends, np.int64)]


@pytest.mark.parametrize("name", OBJECTIVES)
def test_events_beyond_the_node_grid_feed_the_motion_gradient(name):
    """an event beyond the outer nodes has rho = 0 in the forward; where its rotation-only warp is kept it counts in f
    and in the motion gradient (and in no node's)"""
    from event_utils_b200.contrast_max import motion_contrast_objective_torch
    rng = np.random.default_rng(17)
    grids = rng.uniform(0.2, 1.0, (2, 12, 16))
    x, y, d, p, off = outside_stream(4, [6000, 5000], grids, MOTION[:2])
    rho = event_rho(x, y, off, grids)
    for b in range(2):
        sl = slice(off[b], off[b + 1])
        xw, yw = CM.warp(x[sl], y[sl], d[sl], rho[sl], MOTION[b][:3], MOTION[b][3:], INTR)
        none = ~node_taps(x[sl], y[sl], 12, 16, H, W)[3].any(1)
        assert (none & contributes(xw, yw, H, W)).sum() > 100     # the case is exercised in both windows
    f, g, m = joint_loss(x, y, d, p, off, grids, MOTION[:2], name)
    f.sum().backward()
    gr = torch.from_numpy(grids).requires_grad_(True)
    mr = torch.tensor(MOTION[:2], dtype=torch.float64, requires_grad=True)
    fr = MR.contrast(x, y, d, p, off, gr, mr, INTR, 1.0, name, img_size=(H, W))
    fr.sum().backward()
    assert_close_to_max(f.detach().cpu().numpy(), fr.detach().numpy(), DG.F_REL, "f")
    for k in range(6):
        assert_close_to_max(m.grad[:, k].cpu().numpy(), mr.grad[:, k].numpy(), DG.GRAD_REL, "motion component %d" % k)
    assert_close_to_max(g.grad.cpu().numpy(), gr.grad.numpy(), DG.GRAD_REL, "nodes")
    check_motion_bounds(x, y, d, p, off, grids, MOTION[:2], name, m.grad.cpu().numpy(), "outside " + name)
    prm = torch.tensor(MOTION[:2], dtype=torch.float64, device="cuda", requires_grad=True)
    fm = motion_contrast_objective_torch(*_cuda(x, y, d, p), prm, _warp(), t0=0.0, objective=name, blur_sigma=1.0,
                                         img_size=(H, W), batch_end_indices=torch.from_numpy(off[1:]).cuda(),
                                         inv_depth=torch.from_numpy(rho).cuda())
    fm.sum().backward()
    np.testing.assert_allclose(f.detach().cpu().numpy(), fm.detach().cpu().numpy(), rtol=1e-6)
    for k in range(6):
        assert_close_to_max(m.grad[:, k].cpu().numpy(), prm.grad[:, k].cpu().numpy(), 1e-5, "component %d" % k)


@pytest.mark.parametrize("name", OBJECTIVES)
def test_motion_gradient_is_the_per_event_losses(name):
    """the first six components of motion_contrast_objective_torch's gradient with inv_depth = the kernel's rho"""
    from event_utils_b200.contrast_max import motion_contrast_objective_torch
    rng = np.random.default_rng(5)
    grids = DG._grids(rng, 3, 6, 8)
    x, y, d, p, off = safe_stream(8, [4000, 3000, 5000], grids, MOTION)
    f, g, m = joint_loss(x, y, d, p, off, grids, MOTION, name)
    f.sum().backward()
    rho = np.concatenate([R.event_rho_f32(x[off[b]:off[b + 1]], y[off[b]:off[b + 1]], grids[b], H, W) for b in range(3)])
    prm = torch.tensor(MOTION, dtype=torch.float64, device="cuda", requires_grad=True)
    fm = motion_contrast_objective_torch(*_cuda(x, y, d, p), prm, _warp(), t0=0.0, objective=name, blur_sigma=1.0,
                                         img_size=(H, W), batch_end_indices=torch.from_numpy(off[1:]).cuda(),
                                         inv_depth=torch.from_numpy(rho.astype(np.float32)).cuda())
    fm.sum().backward()
    np.testing.assert_allclose(f.detach().cpu().numpy(), fm.detach().cpu().numpy(), rtol=1e-6)
    for k in range(6):
        assert_close_to_max(m.grad[:, k].cpu().numpy(), prm.grad[:, k].cpu().numpy(), 1e-5, "component %d" % k)


def test_a_shared_motion_broadcasts_and_gets_the_summed_gradient():
    rng = np.random.default_rng(6)
    grids = DG._grids(rng, 2, 3, 4)
    x, y, d, p, off = safe_stream(4, [3000, 2000], grids, [MOTION[0]] * 2)
    from event_utils_b200.contrast_max import motion_and_depth_contrast_objective_torch
    m = torch.tensor(MOTION[0], dtype=torch.float64, device="cuda", requires_grad=True)
    f = motion_and_depth_contrast_objective_torch(*_cuda(x, y, d, p), torch.from_numpy(grids).cuda(), m, _warp(), (H, W),
                                                  t0=0.0, batch_end_indices=torch.from_numpy(off[1:]).cuda())
    f.sum().backward()
    f2, _, m2 = joint_loss(x, y, d, p, off, grids, [MOTION[0]] * 2)
    f2.sum().backward()
    assert m.grad.shape == (6,)
    assert_close_to_max(m.grad.cpu().numpy(), m2.grad.sum(0).cpu().numpy(), 1e-5, "shared motion")


@pytest.mark.parametrize("J, shape", [(1, (3, 4)), (32, (6, 8)), (32, (16, 24)), (40, (3, 4))])
def test_candidates_are_the_objective_at_each_pair(J, shape):
    """f[b, j] is the forward at (motion_j, grid_j); (32, 16 x 24) is the limit of one pass and J = 40 takes two"""
    from event_utils_b200.contrast_max import motion_and_depth_contrast_candidates_torch
    rng = np.random.default_rng(J)
    cand = rng.uniform(0.125, 1.0, (2, J) + shape).astype(np.float32)
    mot = np.array(MOTION[:2])[:, None, :] + rng.normal(0, 0.2, (2, J, 6))
    x, y, d, p, off = safe_stream(9, [3000, 4000], cand[:, :1], MOTION[:2])
    fc = motion_and_depth_contrast_candidates_torch(*_cuda(x, y, d, p), torch.from_numpy(mot).cuda(),
                                                    torch.from_numpy(cand).cuda(), _warp(), (H, W), t0=0.0,
                                                    objective="soe", batch_end_indices=torch.from_numpy(off[1:]).cuda())
    assert fc.shape == (2, J) and fc.dtype == torch.float64
    for j in range(0, J, max(1, J // 4)):
        f, _, _ = joint_loss(x, y, d, p, off, cand[:, j], mot[:, j], "soe")
        np.testing.assert_allclose(fc[:, j].cpu().numpy(), f.detach().cpu().numpy(), rtol=1e-6)


@pytest.mark.parametrize("name", OBJECTIVES)
def test_candidates_with_one_motion_are_the_depth_grids(name):
    from event_utils_b200.contrast_max import (depth_grid_contrast_candidates_torch,
                                               motion_and_depth_contrast_candidates_torch)
    rng = np.random.default_rng(13)
    cand = rng.uniform(0.125, 1.0, (3, 12, 6, 8)).astype(np.float32)
    x, y, d, p, off = safe_stream(10, [3000, 4000, 2500], cand[:, :1], MOTION)
    ev, ends = _cuda(x, y, d, p), torch.from_numpy(off[1:]).cuda()
    mt = torch.tensor(MOTION, device="cuda", dtype=torch.float64)
    fj = motion_and_depth_contrast_candidates_torch(*ev, mt[:, None].expand(3, 12, 6), torch.from_numpy(cand).cuda(),
                                                    _warp(), (H, W), t0=0.0, objective=name, batch_end_indices=ends)
    fd = depth_grid_contrast_candidates_torch(*ev, torch.from_numpy(cand).cuda(), mt, _warp(), (H, W), t0=0.0,
                                              objective=name, batch_end_indices=ends)
    # the same taps; only the order in which the f32 image sums add them can differ
    np.testing.assert_allclose(fj.cpu().numpy(), fd.cpu().numpy(), rtol=1e-6)


def test_empty_skewed_and_nan_windows_and_chunks(monkeypatch):
    from event_utils_b200.contrast_max import motion_and_depth as MD
    rng = np.random.default_rng(21)
    motion = [MOTION[b % 2] for b in range(4)]
    cand = rng.uniform(0.2, 1.0, (4, 40, 3, 4)).astype(np.float32)
    x, y, d, p, off = safe_stream(3, [30000, 0, 200, 2500], cand[:, :1], motion, edge=0.0)
    x[5], y[off[3] + 7], p[off[2] + 1] = np.nan, np.nan, np.nan        # non-finite events contribute nothing
    args = _cuda(x, y, d, p)
    mc = torch.from_numpy(np.array(motion)[:, None, :] + rng.normal(0, 0.1, (4, 40, 6))).cuda()
    kw = dict(t0=0.0, blur_sigma=0.0, batch_end_indices=torch.from_numpy(off[1:]).cuda())
    x0 = torch.tensor(motion, device="cuda", dtype=torch.float64)
    f_all = MD.motion_and_depth_contrast_candidates_torch(*args, mc, torch.from_numpy(cand).cuda(), _warp(), (H, W), **kw)
    fit_all = MD.motion_and_depth_fit_torch(*args, _warp(), (H, W), x0, (0.1, 1.2), grid_shapes=((3, 4),), max_iter=3,
                                            num_samples=5, grid_levels=1, **kw)
    monkeypatch.setattr(MD, "CANDIDATES_WORKSPACE_BYTES", 1)     # one window per call
    monkeypatch.setattr(MD, "FIT_WORKSPACE_BYTES", 1)
    f_one = MD.motion_and_depth_contrast_candidates_torch(*args, mc, torch.from_numpy(cand).cuda(), _warp(), (H, W), **kw)
    fit_one = MD.motion_and_depth_fit_torch(*args, _warp(), (H, W), x0, (0.1, 1.2), grid_shapes=((3, 4),), max_iter=3,
                                            num_samples=5, grid_levels=1, **kw)
    np.testing.assert_allclose(f_all.cpu().numpy(), f_one.cpu().numpy(), rtol=1e-6)
    np.testing.assert_allclose(fit_all.inv_depth.cpu().numpy(), fit_one.inv_depth.cpu().numpy(), rtol=0, atol=1e-4)
    np.testing.assert_allclose(fit_all.motion.cpu().numpy(), fit_one.motion.cpu().numpy(), rtol=0, atol=1e-4)
    # the empty window keeps its start and its speed; every speed is kept
    np.testing.assert_allclose(fit_all.motion[1].cpu().numpy(), motion[1], rtol=1e-12)
    np.testing.assert_allclose(fit_all.motion[:, 3:].norm(dim=1).cpu().numpy(), np.linalg.norm(np.array(motion)[:, 3:], axis=1),
                               rtol=1e-12)
    f, g, m = joint_loss(x, y, d, p, off, cand[:, 0], motion, sigma=0.0)
    f.sum().backward()
    assert torch.isfinite(f).all() and torch.isfinite(g.grad).all() and torch.isfinite(m.grad).all()
    assert not g.grad[1].any() and not m.grad[1].any()
    assert m.grad[0].abs().max() > 0 and m.grad[2].abs().max() > 0


def test_window_limits():
    """65535 windows in one call of the joint backward (its batch limit); 65536 are refused with the entry's message"""
    from event_utils_b200 import _lib
    from event_utils_b200.contrast_max import motion_and_depth_contrast_objective_torch
    B = 65535
    rng = np.random.default_rng(1)
    grids = rng.uniform(0.2, 1.0, (3, 3, 4))
    x, y, d, p, off = safe_stream(2, [2000, 1500, 1000], grids, MOTION, edge=0.0)
    ends = np.concatenate([off[1:2], np.full(B - 3, off[1]), off[2:]])     # windows 0, B-2 and B-1 hold events
    g = torch.from_numpy(np.concatenate([grids[:1], np.full((B - 3, 3, 4), 0.5), grids[1:]])).cuda().requires_grad_(True)
    mt = torch.tensor([MOTION[0]] + [MOTION[1]] * (B - 3) + MOTION[1:], device="cuda", dtype=torch.float64,
                      requires_grad=True)
    f = motion_and_depth_contrast_objective_torch(*_cuda(x, y, d, p), g, mt, _warp(), (H, W), t0=0.0,
                                                  batch_end_indices=torch.from_numpy(ends).cuda())
    f.sum().backward()
    f3, g3, m3 = joint_loss(x, y, d, p, off, grids, MOTION)
    f3.sum().backward()
    idx = [0, B - 2, B - 1]
    np.testing.assert_allclose(f[idx].detach().cpu().numpy(), f3.detach().cpu().numpy(), rtol=1e-6)
    assert_close_to_max(mt.grad[idx].cpu().numpy(), m3.grad.cpu().numpy(), 1e-5, "motion at the cap")
    assert not mt.grad[1:B - 2].any() and not g.grad[1:B - 2].any()
    gb = torch.cat((g.detach(), g.detach()[:1]))
    with pytest.raises(_lib.EvkError, match="batch"):
        motion_and_depth_contrast_objective_torch(*_cuda(x, y, d, p), gb, torch.cat((mt.detach(), mt.detach()[:1])),
                                                  _warp(), (H, W), t0=0.0,
                                                  batch_end_indices=torch.from_numpy(np.append(ends, ends[-1])).cuda())


def test_no_host_round_trips_and_constant_launch_count():
    from event_utils_b200 import _lib
    from event_utils_b200.contrast_max import (motion_and_depth_contrast_candidates_torch,
                                               motion_and_depth_contrast_objective_torch, motion_and_depth_fit_torch)
    L = _lib.lib()
    counts = []
    for sizes in ([40000], [2500] * 16):
        B = len(sizes)
        rng = np.random.default_rng(B)
        grids = rng.uniform(0.2, 1.0, (B, 6, 8))
        motion = torch.tensor([MOTION[b % 2] for b in range(B)], device="cuda", dtype=torch.float64)
        n = sum(sizes)
        x, y = (rng.random(n) * (W - 1)).astype(np.float32), (rng.random(n) * (H - 1)).astype(np.float32)
        d, p = (-rng.random(n) * 0.1).astype(np.float32), (rng.integers(0, 2, n) * 2 - 1).astype(np.float32)
        ev = _cuda(x, y, d, p)
        ends = torch.from_numpy(np.cumsum(sizes)).cuda()
        gt = torch.from_numpy(grids).cuda().requires_grad_(True)
        mt = motion.clone().requires_grad_(True)
        cand = torch.from_numpy(grids).cuda().unsqueeze(1).repeat(1, 5, 1, 1)
        mc = motion.unsqueeze(1).repeat(1, 5, 1)
        rng_t = torch.tensor((0.1, 1.5), device="cuda", dtype=torch.float64)
        kw = dict(objective="soe", batch_end_indices=ends)

        def run():
            motion_and_depth_contrast_objective_torch(*ev, gt, mt, _warp(), (H, W), **kw).sum().backward()
            motion_and_depth_contrast_candidates_torch(*ev, mc, cand, _warp(), (H, W), **kw)
            motion_and_depth_fit_torch(*ev, _warp(), (H, W), motion, rng_t, grid_shapes=((3, 4), (6, 8)), max_iter=2,
                                       num_samples=5, grid_levels=1, **kw)
        run()   # warm-up
        torch.cuda.synchronize()
        L.evk_prof_enable(1)
        torch.cuda.set_sync_debug_mode("error")
        try:
            run()
        finally:
            torch.cuda.set_sync_debug_mode(0)
        ms, timed, launches = ctypes.c_double(), ctypes.c_longlong(), ctypes.c_longlong()
        _lib.check(L.evk_prof_collect(ctypes.byref(ms), ctypes.byref(timed), ctypes.byref(launches)))
        L.evk_prof_enable(0)
        assert torch.isfinite(gt.grad).all() and torch.isfinite(mt.grad).all()
        counts.append(launches.value)
    assert counts[0] == counts[1] and counts[0] > 0, counts


# ---- recovery of the depth-grid scenes from a wrong start motion ------------------------------------------------
W_OFF, HEADING_OFF = 0.1, 10.0     # rad/s per axis of w, degrees of v at the true speed
# the largest of three H100 runs with margin: |w - w_true| / |start error| and heading error / start heading error
# (eight runs: w 0.32-0.47 / 0.25-0.31 / 0.45-0.47, heading 0.70-0.79 / 0.16 / 0.78-0.84).  The slanted plane and the
# plane seen with forward v keep most of their heading error: DESIGN.md section 6.
RECOVERY_TOL = dict(w=(0.6, 0.4, 0.6), heading=(0.9, 0.25, 0.9))


def _turn(v, degrees, rng):
    """v turned by `degrees` about an axis normal to it, at the same speed"""
    a = rng.normal(size=3)
    a -= a.dot(v) / v.dot(v) * v
    a /= np.linalg.norm(a)
    t = np.radians(degrees)
    return np.cos(t) * v + np.sin(t) * np.linalg.norm(v) * a


def wrong_start(motion, seed=0):
    rng = np.random.default_rng(seed)
    return np.array([np.concatenate((m[:3] + W_OFF, _turn(m[3:], HEADING_OFF, rng))) for m in motion])


def heading_error(v, v_true):
    c = (v * v_true).sum(-1) / (np.linalg.norm(v, axis=-1) * np.linalg.norm(v_true, axis=-1))
    return np.degrees(np.arccos(np.clip(c, -1, 1)))


def recovery(seed=0, opts=None):
    """the joint fit (with the extra arguments opts) and depth_grid_fit_torch at the wrong start and at the truth on
    the three scenes: a dict of their errors and objectives"""
    from event_utils_b200.contrast_max import (depth_grid_contrast_objective_torch, depth_grid_fit_torch,
                                               motion_and_depth_fit_torch)
    (x, y, t, p), ends, motion, truth = DG.recovery_windows()
    ev = _cuda(x, y, t, p)
    kw = dict(batch_end_indices=torch.from_numpy(ends).cuda())
    x0 = wrong_start(motion, seed)
    warp = _warp(DG.SCENE_INTR)
    fit = motion_and_depth_fit_torch(*ev, warp, (180, 240), torch.from_numpy(x0).cuda(), DG.RANGE, **kw, **(opts or {}))
    at_wrong = depth_grid_fit_torch(*ev, torch.from_numpy(x0).cuda(), warp, (180, 240), DG.RANGE, **kw)
    at_truth = depth_grid_fit_torch(*ev, torch.from_numpy(motion).cuda(), warp, (180, 240), DG.RANGE, **kw)
    m = fit.motion.cpu().numpy()
    return dict(w=np.linalg.norm(m[:, :3] - motion[:, :3], axis=1) / np.linalg.norm(x0[:, :3] - motion[:, :3], axis=1),
                heading=heading_error(m[:, 3:], motion[:, 3:]) / heading_error(x0[:, 3:], motion[:, 3:]),
                speed=np.linalg.norm(m[:, 3:], axis=1) / np.linalg.norm(motion[:, 3:], axis=1),
                rho=np.array(DG.median_errors(fit.inv_depth.cpu().numpy(), truth)),
                rho_wrong=np.array(DG.median_errors(at_wrong.inv_depth.cpu().numpy(), truth)),
                rho_truth=np.array(DG.median_errors(at_truth.inv_depth.cpu().numpy(), truth)),
                F=fit.f.cpu().numpy(), F_truth=at_truth.f.cpu().numpy(), status=fit.status.cpu().numpy())


def test_joint_fit_recovers_motion_and_depth():
    r = recovery()
    print({k: np.round(v, 5) for k, v in r.items()})
    np.testing.assert_allclose(r["speed"], 1.0, rtol=1e-12)
    assert (r["w"] <= RECOVERY_TOL["w"]).all(), r["w"]
    assert (r["heading"] <= RECOVERY_TOL["heading"]).all(), r["heading"]
    assert (r["rho"] < r["rho_wrong"]).all(), (r["rho"], r["rho_wrong"])
    # F at or below the F of depth_grid_fit_torch at the true motion, but for the f32 noise of F
    assert (r["F"] <= r["F_truth"] + 1e-5 * np.abs(r["F_truth"])).all(), (r["F"], r["F_truth"])
