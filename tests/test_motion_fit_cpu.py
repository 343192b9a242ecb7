"""No-GPU checks of the batched motion fit: the candidates entry's workspace query and argument errors, the device grid
against grid_search_initial / find_new_range, and the batched BFGS core on analytic functions."""
import ctypes

import numpy as np
import pytest
import torch

from event_utils_b200.contrast_max import events_cmax
from event_utils_b200.contrast_max import motion_fit as MF

E_ARG, E_WORKSPACE, E_UNSUPPORTED = -1, -3, -5


def _lib():
    from event_utils_b200 import _lib
    return _lib.load()


def _aligned(nbytes):
    return (nbytes + 255) // 256 * 256


def test_candidates_workspace_query():
    L = _lib()
    for B, J, H, W in ((1, 1, 2, 2), (5, 7, 180, 240), (64, 32, 60, 80), (0, 3, 10, 10)):
        C, npix = B * J, (H + 1) * (W + 1)
        want = (_aligned(4 * C) + _aligned(64 * C) + _aligned(4 * C) + _aligned(16 * C * npix) + 3 * _aligned(4 * C * npix))
        assert L.evk_cmax_motion_candidates_workspace_bytes(B, J, H, W) == want
    # a forward-only canvas: about 28 bytes per pixel, against the 44 of the differentiable entry
    per = L.evk_cmax_motion_candidates_workspace_bytes(1, 32, 180, 240) / (32 * 181 * 241)
    assert 28 <= per < 28.1
    assert L.evk_cmax_motion_objective_workspace_bytes(32, 180, 240) / (32 * 181 * 241) >= 44
    for bad in ((-1, 4, 10, 10), (2, 0, 10, 10), (2, 33, 10, 10), (2, 4, 1, 10), (2, 4, 10, 1)):
        assert L.evk_cmax_motion_candidates_workspace_bytes(*bad) == 0, bad


def _call(**kw):
    """evk_cmax_motion_candidates_f32 with fake, aligned, never dereferenced pointers and a plausible argument list"""
    L = _lib()
    fake = ctypes.c_void_p(1 << 20)
    a = dict(batch=4, n=1000, warp=1, n_cand=8, K=3, H=60, W=80, sigma=1.0, objective=0, ws_bytes=1 << 40)
    a.update(kw)
    rc = L.evk_cmax_motion_candidates_f32(fake, fake, fake, fake, fake, a["batch"], a["n"], a["warp"], fake, a["n_cand"], a["K"],
                                          40.0, 30.0, a["H"], a["W"], a["sigma"], a["objective"], 3.0, fake, fake, a["ws_bytes"],
                                          None)
    return rc, L.evk_last_error()


def test_candidates_argument_errors_without_a_gpu():
    assert _call(K=2)[0] == E_ARG                          # rotation has K = 3
    assert _call(warp=3, K=3)[0] == E_ARG                  # linvel has K = 2
    assert _call(warp=7)[0] == E_ARG
    for J in (0, 33, -1):
        rc, msg = _call(n_cand=J)
        assert rc == E_ARG and b"n_cand" in msg, (J, msg)
    rc, msg = _call(batch=2048, n_cand=32)                 # 65536 canvases
    assert rc == E_ARG and b"65535" in msg
    assert _call(batch=-1)[0] == E_ARG
    assert _call(H=1)[0] == E_ARG
    for obj in (3, 4):                                     # moa, isoa
        rc, msg = _call(objective=obj)
        assert rc == E_UNSUPPORTED and b"piecewise constant" in msg
    assert _call(objective=9)[0] == E_ARG
    for sigma, want in ((float("nan"), E_ARG), (16.125, E_UNSUPPORTED), (1e9, E_UNSUPPORTED), (float("inf"), E_UNSUPPORTED)):
        rc, msg = _call(sigma=sigma)
        assert rc == want and b"blur sigma" in msg, (sigma, rc, msg)
    need = _lib().evk_cmax_motion_candidates_workspace_bytes(4, 8, 60, 80)
    rc, msg = _call(ws_bytes=need - 1)
    assert rc == E_WORKSPACE and b"workspace" in msg


# ---- the device grid against grid_search_initial and find_new_range ----------------------------------------------------
class _Rot:
    dims = 3


def _reference_grid(monkeypatch, ranges, num, log_scale):
    """grid_search_initial's axes and points, its evaluation replaced by zeros (it needs no GPU then)"""
    monkeypatch.setattr(events_cmax, "evaluate_candidates", lambda obj, pts, *a, **k: (np.zeros(len(pts)), None))
    out = events_cmax.grid_search_initial(None, None, None, None, _Rot(), None, None, param_ranges=ranges, log_scale=log_scale,
                                          num_samples_per_param=num)
    return out["search_axes"], np.array(out["params"])


@pytest.mark.parametrize("log_scale", [False, True])
@pytest.mark.parametrize("num", [3, 5, 7])
def test_grid_axes_and_points_equal_grid_search_initial(monkeypatch, log_scale, num):
    windows = [[[-150, 150], [-150, 150], [-150, 150]], [[0.5, 7.25], [-3.0, 11.0], [100.0, 100.0]],
               [[-1e-3, 2e-3], [1e5, 3e5], [-7.3, -2.1]]]
    ranges = torch.tensor(windows, dtype=torch.float64)
    axes = MF._grid_axes(ranges, num, log_scale)
    pts = MF._grid_points(axes)
    assert axes.shape == (3, 3, num) and pts.shape == (3, num ** 3, 3)
    for b, r in enumerate(windows):
        ref_axes, ref_pts = _reference_grid(monkeypatch, r, num, log_scale)
        for k in range(3):
            assert np.array_equal(axes[b, k].numpy(), ref_axes[k]), (b, k)
        assert np.array_equal(pts[b].numpy(), ref_pts), b


@pytest.mark.parametrize("log_scale", [False, True])
def test_recentring_equals_find_new_range(log_scale):
    """every sample of every axis as the best point (index 0 takes the distance to the LAST sample, the last index the
    outermost spacing), plus points off the axis and beyond both ends"""
    ranges = torch.tensor([[[-150, 150], [2.0, 9.0]], [[-1.0, 3.0], [40.0, 41.0]]], dtype=torch.float64)
    axes = MF._grid_axes(ranges, 5, log_scale)
    a = axes.numpy()
    for extra in range(5 + 3):
        if extra < 5:
            best = axes[..., extra]
        else:
            off = {5: -1.0, 6: 0.37, 7: 1e3}[extra]
            best = axes[..., 2] + off * (axes[..., 4] - axes[..., 0])
        got = MF._new_ranges(axes, best).numpy()
        for b in range(2):
            for k in range(2):
                ref = events_cmax.find_new_range(a[b, k], float(best[b, k]))
                assert got[b, k].tolist() == [float(v) for v in ref], (extra, b, k, got[b, k], ref)


def test_grid_search_levels_and_ties():
    """two levels on a separable quadratic with its minimum off the grid; equal values take the first point"""
    m = torch.tensor([[3.3, -7.1], [40.0, 2.0]], dtype=torch.float64)
    ranges = torch.tensor([[-50.0, 50.0]], dtype=torch.float64).expand(2, 2, 2).contiguous()
    f = lambda pts: ((pts - m.unsqueeze(1)) ** 2).sum(2)
    one = MF._grid_search(f, ranges, 5, 1)
    two = MF._grid_search(f, ranges, 5, 2)
    three = MF._grid_search(f, ranges, 5, 3)
    for lo, hi in ((one, two), (two, three)):
        assert ((hi - m).norm(dim=1) <= (lo - m).norm(dim=1)).all()
    assert (three - m).abs().max() < 3.2
    flat = MF._grid_search(lambda pts: torch.zeros(pts.shape[:2], dtype=torch.float64), ranges, 5, 1)
    assert flat.tolist() == [[-50.0, -50.0]] * 2                    # the first meshgrid point
    nan_first = MF._grid_search(lambda pts: torch.where(pts[..., 0] < -40, float("nan"), 0.0), ranges, 5, 1)
    assert (nan_first[:, 1] == -50.0).all() and (nan_first[:, 0] > -40).all()


# ---- the BFGS core on batched analytic functions -----------------------------------------------------------------------
def _quadratics(seed=0, B=6, K=3):
    """f_b(x) = 0.5 sum_k a_bk (x_k - m_bk)^2 - 5, curvatures over eight decades, and a scale within 2x of 1/sqrt(a)"""
    rng = np.random.default_rng(seed)
    a = torch.tensor(10.0 ** rng.uniform(-4, 4, (B, K)))
    m = torch.tensor(rng.uniform(-100, 100, (B, K)))
    scale = torch.tensor(rng.uniform(0.5, 2.0, (B, K))) / a.sqrt()
    x0 = m + scale * torch.tensor(rng.uniform(-20, 20, (B, K)))

    def fg(x):
        r = x - m
        return 0.5 * (a * r * r).sum(1) - 5.0, a * r

    def cand(pts):
        r = pts - m.unsqueeze(1)
        return 0.5 * (a.unsqueeze(1) * r * r).sum(2) - 5.0
    return fg, cand, x0, scale, m


def _rosenbrock(K):
    """1 + the K-D Rosenbrock function, minimum 1 at ones"""
    def f(x):
        return 1.0 + (100.0 * (x[..., 1:] - x[..., :-1] ** 2) ** 2 + (1.0 - x[..., :-1]) ** 2).sum(-1)

    def fg(x):
        xr = x.detach().clone().requires_grad_(True)
        v = f(xr)
        v.sum().backward()
        return v.detach(), xr.grad
    return fg, f


def test_bfgs_reaches_every_quadratic_minimum():
    fg, cand, x0, scale, m = _quadratics()
    x, f, status, iters = MF._batched_bfgs(fg, cand, x0, scale, max_iter=60, ftol=1e-12, gtol=1e-10)
    assert (status == MF.CONVERGED).all(), status
    assert ((x - m).abs() <= 1e-5 * scale).all(), (x - m) / scale
    assert (f - (-5.0)).abs().max() < 1e-9
    assert (iters > 0).all() and (iters <= 60).all()


@pytest.mark.parametrize("K", [2, 3, 4])
def test_bfgs_reaches_the_rosenbrock_minimum(K):
    fg, f = _rosenbrock(K)
    # (from (-1.2, 1, 0.8, 1.9) the 4-D function leads to its second, local minimum near (-0.78, 0.61, 0.38, 0.15))
    starts = [[0.0] * K, [1.5] * K, [-0.5, 2.0, -1.0, 0.5][:K], [2.0, -1.0, 1.5, 0.3][:K]] + ([[-1.2, 1.0, 0.8][:K]] if K < 4 else [])
    starts = torch.tensor(starts, dtype=torch.float64)
    x, fx, status, iters = MF._batched_bfgs(fg, f, starts, torch.ones(len(starts), K, dtype=torch.float64), max_iter=300,
                                            line_search_steps=16, ftol=1e-15, gtol=1e-12)
    assert (status != MF.ITERATION_LIMIT).all() and (status != MF.NONFINITE_START).all(), status
    assert ((x - 1.0).abs() <= 1e-4).all(), x
    assert ((fx - 1.0).abs() <= 1e-10).all(), fx


def test_bfgs_never_increases_f_and_freezes_stopped_windows():
    """f after n iterations is non-increasing in n for every window; a window stopped after n iterations has exactly the
    same x, f, status and iteration count at n + 10"""
    fg_q, cand_q, x0, scale, _ = _quadratics(seed=3, B=4, K=2)
    fg_r, f_r = _rosenbrock(2)

    def fg(x):          # windows 0-3 quadratics, 4-5 Rosenbrock
        fq, gq = fg_q(x[:4])
        fr, gr = fg_r(x[4:])
        return torch.cat((fq, fr)), torch.cat((gq, gr))

    def cand(pts):
        return torch.cat((cand_q(pts[:4]), f_r(pts[4:])))
    starts = torch.cat((x0, torch.tensor([[-1.2, 1.0], [2.0, -1.0]], dtype=torch.float64)))
    sc = torch.cat((scale, torch.ones(2, 2, dtype=torch.float64)))
    runs = [MF._batched_bfgs(fg, cand, starts, sc, max_iter=n, ftol=1e-10, gtol=1e-9) for n in range(0, 41)]
    f_start = fg(starts)[0]
    for n in range(1, 41):
        assert (runs[n][1] <= runs[n - 1][1]).all(), n
        assert (runs[n][1] <= f_start).all()
    for n in range(0, 31):
        x, f, st, it = runs[n]
        x2, f2, st2, it2 = runs[n + 10]
        done = st != MF.ITERATION_LIMIT
        assert torch.equal(x[done], x2[done]) and torch.equal(f[done], f2[done]), n
        assert torch.equal(st[done], st2[done]) and torch.equal(it[done], it2[done]), n
    assert (runs[40][2][:4] == MF.CONVERGED).all()


def test_bfgs_statuses():
    fg_q, cand_q, x0, scale, m = _quadratics(seed=5, B=5, K=2)
    # window 2 starts at NaN; window 3's f is NaN everywhere; window 4's gradient points uphill (no candidate descends)

    def fg(x):
        f, g = fg_q(x)
        f = torch.where(torch.arange(5) == 3, float("nan"), f)
        g = torch.where((torch.arange(5) == 4).unsqueeze(1), -g, g)
        return f, g

    def cand(pts):
        f = cand_q(pts)
        return torch.where((torch.arange(5) == 3).unsqueeze(1), float("nan"), f)
    start = x0.clone()
    start[2, 1] = float("nan")
    x, f, status, iters = MF._batched_bfgs(fg, cand, start, scale, max_iter=40, ftol=1e-12, gtol=1e-10)
    assert status.tolist() == [MF.CONVERGED, MF.CONVERGED, MF.NONFINITE_START, MF.NONFINITE_START, MF.NO_DESCENT], status
    assert torch.equal(x[2:], start[2:]) or (torch.isnan(x[2, 1]) and torch.equal(x[3:], start[3:]))
    assert iters[2:].tolist() == [0, 0, 0]
    # the iteration limit, and a start at the minimum (g = 0): converged with no iteration
    x, f, status, iters = MF._batched_bfgs(fg_q, cand_q, x0, scale, max_iter=1, ftol=0.0, gtol=0.0)
    assert (status == MF.ITERATION_LIMIT).all() and (iters == 1).all()
    x, f, status, iters = MF._batched_bfgs(fg_q, cand_q, m, scale, max_iter=5)
    assert (status == MF.CONVERGED).all() and (iters == 0).all() and torch.equal(x, m)


def test_fit_argument_errors():
    from event_utils_b200.contrast_max import motion_contrast_fit_torch, pure_rotation_warp, linvel_warp
    e = np.zeros(4, np.float32)
    with pytest.raises(ValueError, match="x0 or param_ranges"):
        motion_contrast_fit_torch(e, e, e, e, pure_rotation_warp())
    with pytest.raises(ValueError, match="piecewise constant"):
        motion_contrast_fit_torch(e, e, e, e, linvel_warp(), objective="moa", x0=[0.0, 0.0])
    with pytest.raises(ValueError, match="line_search_steps"):
        motion_contrast_fit_torch(e, e, e, e, linvel_warp(), x0=[0.0, 0.0], line_search_steps=33)
