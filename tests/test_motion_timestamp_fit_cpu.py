"""No-GPU checks of the batched fit of the average-timestamp loss: the candidates entry's workspace query and argument
errors, the fit's argument errors, the bounded BFGS core, and the premise of the GPU recovery tests (the f64 reference's
level-0 grid minimum is the grid point nearest the truth)."""
import ctypes

import numpy as np
import pytest
import torch

import motion_timestamp_reference as R
from flow_objective_reference import blur_matrix
from event_utils_b200.contrast_max import motion_fit as MF
from test_gpu_motion_timestamp_fit import FIT_BLURS, FIT_CENTRE, FIT_RANGES, FIT_SEEDS, FIT_WINDOW, host_windows

E_ARG, E_WORKSPACE, E_UNSUPPORTED = -1, -3, -5


def _lib():
    from event_utils_b200 import _lib
    return _lib.load()


def _aligned(nbytes):
    return (nbytes + 255) // 256 * 256


def test_candidates_workspace_query():
    L = _lib()
    for B, J, H, W in ((1, 1, 2, 2), (5, 7, 180, 240), (64, 32, 60, 80), (0, 3, 10, 10)):
        I, npix = 2 * B * J, (H + 1) * (W + 1)
        # counters, gsums, gmax, the 32-byte blocks, tmp / G / T, then the C images
        want = (_aligned(4 * I) + _aligned(64 * I) + _aligned(4 * I) + _aligned(32 * I * npix) + 3 * _aligned(4 * I * npix)
                + _aligned(4 * I * npix))
        assert L.evk_motion_timestamp_candidates_workspace_bytes(B, J, H, W) == want
    per = L.evk_motion_timestamp_candidates_workspace_bytes(1, 32, 180, 240) / (32 * 181 * 241)
    assert 96 <= per < 96.1
    for bad in ((-1, 4, 10, 10), (2, 0, 10, 10), (2, 33, 10, 10), (2, 4, 1, 10), (2, 4, 10, 1)):
        assert L.evk_motion_timestamp_candidates_workspace_bytes(*bad) == 0, bad


def _call(**kw):
    """evk_motion_timestamp_candidates_f32 with fake, aligned, never dereferenced pointers and a plausible argument list"""
    L = _lib()
    fake = ctypes.c_void_p(1 << 20)
    a = dict(batch=4, n=1000, warp=1, n_cand=8, K=3, H=60, W=80, sigma=1.0, f_out=fake, ws_bytes=1 << 40)
    a.update(kw)
    rc = L.evk_motion_timestamp_candidates_f32(fake, fake, fake, fake, fake, fake, a["batch"], a["n"], a["warp"], fake,
                                               a["n_cand"], a["K"], 40.0, 30.0, a["H"], a["W"], a["sigma"], a["f_out"], fake,
                                               a["ws_bytes"], None)
    return rc, L.evk_last_error()


def test_candidates_argument_errors_without_a_gpu():
    assert _call(K=2)[0] == E_ARG                          # rotation has K = 3
    assert _call(warp=3, K=3)[0] == E_ARG                  # linvel has K = 2
    assert _call(warp=7)[0] == E_ARG
    for J in (0, 33, -1):
        rc, msg = _call(n_cand=J)
        assert rc == E_ARG and b"n_cand" in msg, (J, msg)
    rc, msg = _call(batch=1024, n_cand=32)                 # 32768 image pairs
    assert rc == E_ARG and b"32767" in msg
    assert _call(batch=1023, n_cand=32, f_out=None)[0] == E_ARG
    assert _call(f_out=None)[0] == E_ARG
    assert _call(batch=-1)[0] == E_ARG
    assert _call(H=1)[0] == E_ARG
    for sigma, want in ((float("nan"), E_ARG), (16.125, E_UNSUPPORTED), (1e9, E_UNSUPPORTED), (float("inf"), E_UNSUPPORTED)):
        rc, msg = _call(sigma=sigma)
        assert rc == want and b"blur sigma" in msg, (sigma, rc, msg)
    need = _lib().evk_motion_timestamp_candidates_workspace_bytes(4, 8, 60, 80)
    rc, msg = _call(ws_bytes=need - 1)
    assert rc == E_WORKSPACE and b"workspace" in msg


def test_fit_and_candidates_argument_errors():
    from event_utils_b200.contrast_max import (linvel_warp, motion_timestamp_candidates_torch, motion_timestamp_fit_torch,
                                               pure_rotation_warp, variance_objective)
    e = np.zeros(4, np.float32)
    with pytest.raises(ValueError, match="linvel_warp, pure_rotation_warp and xyztheta_warp"):
        motion_timestamp_fit_torch(e, e, e, e, variance_objective(), x0=[0.0, 0.0])
    with pytest.raises(ValueError, match="linvel_warp, pure_rotation_warp and xyztheta_warp"):
        motion_timestamp_candidates_torch(e, e, e, e, np.zeros((1, 1, 2)), variance_objective())
    with pytest.raises(ValueError, match="x0 or param_ranges"):
        motion_timestamp_fit_torch(e, e, e, e, pure_rotation_warp())
    for steps in (0, 33):
        with pytest.raises(ValueError, match="line_search_steps"):
            motion_timestamp_fit_torch(e, e, e, e, linvel_warp(), x0=[0.0, 0.0], line_search_steps=steps)
    with pytest.raises(ValueError, match="blur_sigma"):
        motion_timestamp_fit_torch(e, e, e, e, linvel_warp(), x0=[0.0, 0.0], blur_sigma=())
    for bounds in ([0.0, 1.0], [[0.0, 1.0]], np.zeros((2, 2, 2)), np.zeros((2, 3))):
        with pytest.raises(ValueError, match="bounds must have shape"):
            motion_timestamp_fit_torch(e, e, e, e, linvel_warp(), x0=[0.0, 0.0], bounds=bounds)


# ---- the bounded BFGS core ----------------------------------------------------------------------------------------------
def _cliff():
    """f = (x - 1)^2 + 1 inside |x| < 10 and 0 outside: the timestamp loss's shape, whose global minimum 0 lies where
    every event has left the canvas"""
    def f(x):
        return torch.where(x.abs() < 10, (x - 1) ** 2 + 1, torch.zeros_like(x)).sum(-1)

    def fg(x):
        inside = x.abs() < 10
        return f(x), torch.where(inside, 2 * (x - 1), torch.zeros_like(x))
    return fg, f


def test_bounds_keep_the_line_search_off_the_cliff():
    fg, f = _cliff()
    x0 = torch.tensor([[3.0]], dtype=torch.float64)
    scale = torch.tensor([[5.0]], dtype=torch.float64)
    # the first step, H g = 25 * 4 = 100 long, lands outside; 2^-4 .. 2^-7 of it land inside [-5, 5]
    steps = x0 - 100.0 * torch.pow(2.0, -torch.arange(8, dtype=torch.float64))
    assert steps[0, 0] < -10 and ((steps.abs() <= 5).sum() >= 3)
    x, fx, status, _ = MF._batched_bfgs(fg, f, x0, scale, max_iter=30, line_search_steps=8)
    assert fx.item() == 0.0 and x.abs().item() >= 10                   # unbounded: off the cliff, "converged"
    bounds = torch.tensor([[[-5.0, 5.0]]], dtype=torch.float64)
    seen = []

    def cand(pts):
        seen.append(pts.clone())
        return f(pts)
    for n in range(0, 31):
        x, fx, status, _ = MF._batched_bfgs(fg, cand, x0, scale, max_iter=n, line_search_steps=8, bounds=bounds)
        assert -5.0 <= x.item() <= 5.0, (n, x)
    assert abs(x.item() - 1.0) <= 1e-6 and abs(fx.item() - 1.0) <= 1e-12, (x, fx, status)
    assert any(((p < -5) | (p > 5)).any() for p in seen)              # points outside were scored, and none was taken


def _quadratics(seed=0, B=6, K=3):
    rng = np.random.default_rng(seed)
    a = torch.tensor(10.0 ** rng.uniform(-4, 4, (B, K)))
    m = torch.tensor(rng.uniform(-100, 100, (B, K)))
    scale = torch.tensor(rng.uniform(0.5, 2.0, (B, K))) / a.sqrt()
    x0 = m + scale * torch.tensor(rng.uniform(-20, 20, (B, K)))
    fg = lambda x: (0.5 * (a * (x - m) ** 2).sum(1) - 5.0, a * (x - m))
    cand = lambda pts: 0.5 * (a.unsqueeze(1) * (pts - m.unsqueeze(1)) ** 2).sum(2) - 5.0
    return fg, cand, x0, scale


def _rosenbrock_fg(x):
    xr = x.detach().clone().requires_grad_(True)
    v = _rosenbrock(xr)
    v.sum().backward()
    return v.detach(), xr.grad


def _rosenbrock(x):
    return 1.0 + (100.0 * (x[..., 1:] - x[..., :-1] ** 2) ** 2 + (1.0 - x[..., :-1]) ** 2).sum(-1)


def test_no_bounds_and_an_unbinding_box_change_nothing():
    """bounds=None is the unbounded core; an infinite box gives bit-identical results"""
    fg, cand, x0, scale = _quadratics()
    starts = torch.tensor([[0.0, 0.0, 0.0], [1.5, 1.5, 1.5], [-0.5, 2.0, -1.0]], dtype=torch.float64)
    cases = [(fg, cand, x0, scale, dict(max_iter=60, ftol=1e-12, gtol=1e-10)),
             (_rosenbrock_fg, _rosenbrock, starts, torch.ones(3, 3, dtype=torch.float64),
              dict(max_iter=300, line_search_steps=16, ftol=1e-15, gtol=1e-12))]
    for fgi, ci, xi, si, kw in cases:
        plain = MF._batched_bfgs(fgi, ci, xi, si, **kw)
        none = MF._batched_bfgs(fgi, ci, xi, si, bounds=None, **kw)
        box = torch.tensor([-np.inf, np.inf], dtype=torch.float64).expand(xi.shape[0], xi.shape[1], 2)
        inf = MF._batched_bfgs(fgi, ci, xi, si, bounds=box, **kw)
        for a, b, c in zip(plain, none, inf):
            assert torch.equal(a, b) and torch.equal(a, c)


# ---- the premise of the GPU recovery tests ------------------------------------------------------------------------------
def _level0_values(kind, x, y, d, tau, p, pts, sigmas, H=180, W=240):
    """f of the f64 reference (motion_timestamp_reference.reference, restated with bincount for speed) at every point,
    for every blur: (len(sigmas), P)"""
    Hc, Wc = H + 1, W + 1
    mats = [(blur_matrix(Hc, s), blur_matrix(Wc, s)) for s in sigmas]
    x64, y64, d64 = (torch.from_numpy(a.astype(np.float64)) for a in (x, y, d))
    out = np.empty((len(sigmas), len(pts)))
    for i, prm in enumerate(pts):
        xw32, yw32 = R.warp_f32(kind, x, y, d, prm, FIT_CENTRE)
        keep = R.contributes(xw32, yw32, H, W)
        xw, yw = (a.numpy() for a in R.warp_f64(kind, x64, y64, d64, torch.tensor(prm), FIT_CENTRE))
        T = []
        for sel in (p > 0, p <= 0):
            k = np.flatnonzero(keep & sel)
            px, py = np.floor(xw32[k]).astype(np.int64), np.floor(yw32[k]).astype(np.int64)
            dx, dy = xw[k] - px, yw[k] - py
            S, C = np.zeros(Hc * Wc), np.ones(Hc * Wc)
            for oy, ox, wt in ((0, 0, (1 - dx) * (1 - dy)), (0, 1, dx * (1 - dy)), (1, 0, (1 - dx) * dy), (1, 1, dx * dy)):
                cell = (py + oy) * Wc + px + ox
                S += np.bincount(cell, tau[k] * wt, Hc * Wc)
                C += np.bincount(cell, wt, Hc * Wc)
            T.append((S / C).reshape(Hc, Wc))
        for s, (My, Mx) in enumerate(mats):
            out[s, i] = sum(float(((My @ Ti @ Mx.T) ** 2).sum()) for Ti in T)
    return out


@pytest.mark.parametrize("kind", ["linvel", "rotation"])
def test_reference_level0_grid_minimum_is_nearest_the_truth(kind):
    _, truths, (x, y, t, p), ends = host_windows(kind, 64, FIT_SEEDS[kind], **FIT_WINDOW)
    off = np.concatenate(([0], ends)).astype(np.int64)
    tau = R.tau_f32(t, off).astype(np.float64)
    ranges = torch.tensor(FIT_RANGES[kind], dtype=torch.float64).expand(1, -1, -1)
    axes = MF._grid_axes(ranges, 5, False)
    pts = MF._grid_points(axes)[0].numpy()
    near = np.array([[np.abs(axes[0, k].numpy() - tr[k]).argmin() for k in range(len(tr))] for tr in truths])
    for b in range(len(truths)):
        sl = slice(off[b], off[b + 1])
        d = (t[sl] - t[sl][-1]).astype(np.float32)
        xb, yb, pb = (a[sl].astype(np.float32) for a in (x, y, p))
        f = _level0_values(kind, xb, yb, d, tau[sl], pb, pts, FIT_BLURS)
        want = np.array([axes[0, k, near[b, k]].item() for k in range(pts.shape[1])])
        for s, sigma in enumerate(FIT_BLURS):
            got = pts[f[s].argmin()]
            if kind == "linvel":
                assert np.array_equal(got, want), (kind, b, sigma, got, want, truths[b])
            else:
                # the centre and the rate trade off against each other on the 5-sample grid: within one step per axis
                step = (axes[0, :, 1] - axes[0, :, 0]).numpy()
                assert (np.abs(got - want) <= step * 1.001).all(), (kind, b, sigma, got, want, truths[b])
