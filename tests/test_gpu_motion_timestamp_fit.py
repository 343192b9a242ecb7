"""The multi-candidate pass of the average-timestamp loss (evk_motion_timestamp_candidates_f32,
motion_timestamp_candidates_torch) against the batched forward it restates per candidate and the f64 reference, and the
batched fit (motion_timestamp_fit_torch): recovery of known motions inside its bounds, scipy's BFGS per window, NaN
isolation and no host synchronisation."""
import ctypes

import numpy as np
import pytest
import torch

import motion_timestamp_reference as R
from edge_cases import exact_streams
from test_gpu_motion_fit import recovered, truths_of, windows

pytestmark = pytest.mark.gpu

WARP = {"linvel": 3, "rotation": 1, "xyztheta": 2}
H, W = 60, 80
CENTRE = (40.0, 30.0)
BASE = {"linvel": [(30.0, -20.0), (-55.0, 12.5), (5.0, 8.0), (900.0, -700.0), (0.0, 0.0)],
        "rotation": [(40.0, 30.0, 4.0), (35.0, 28.0, -6.0), (45.0, 33.0, 1.5), (10.0, 10.0, 40.0), (40.0, 30.0, 0.0)],
        "xyztheta": [(20.0, -10.0, 3.0, 2.0), (-30.0, 15.0, -2.0, 4.0), (5.0, 5.0, 0.5, -3.0), (600.0, -500.0, 30.0, 9.0),
                     (0.0, 0.0, 0.0, 0.0)]}
# a candidate that sends every event off the canvas
GONE = {"linvel": (1e6, -1e6), "rotation": (1e5, 1e5, 50.0), "xyztheta": (1e6, 1e6, 0.0, 0.0)}

# the recovery tests' scenes (180x240, scene centre (120, 90)): seeds, grid ranges and blur stages; the CPU test
# test_motion_timestamp_fit_cpu.py checks that the f64 reference's level-0 grid minimum is the grid point nearest the
# truth in every window, at every blur
FIT_SEEDS = {"linvel": 161, "rotation": 162}
FIT_RANGES = {"linvel": [[-80.0, 80.0], [-80.0, 80.0]], "rotation": [[110.0, 130.0], [80.0, 100.0], [-10.0, 10.0]]}
FIT_BLURS = (2.0,)
FIT_WINDOW = dict(n_pts=300, per_pt=50)
FIT_CENTRE = (120.0, 90.0)


def _warp(kind, centre=CENTRE):
    from event_utils_b200.contrast_max import linvel_warp, pure_rotation_warp, xyztheta_warp
    return {"linvel": linvel_warp, "rotation": pure_rotation_warp, "xyztheta": lambda: xyztheta_warp(center=centre)}[kind]()


def batch_stream(seed, sizes, h=H, w=W):
    """concatenated windows; events in the sensor, sorted stamps over 0.1 time units per window, d = t - the window's
    last stamp"""
    rng = np.random.default_rng(seed)
    n = sum(sizes)
    x = (rng.random(n) * (w - 1)).astype(np.float32)
    y = (rng.random(n) * (h - 1)).astype(np.float32)
    p = (rng.integers(0, 2, n) * 2 - 1).astype(np.float32)
    t = np.empty(n, np.float32)
    d = np.empty(n, np.float32)
    off = np.concatenate(([0], np.cumsum(sizes))).astype(np.int64)
    for b in range(len(sizes)):
        t[off[b]:off[b + 1]] = np.sort(rng.random(sizes[b])) * 0.1 + b
        if sizes[b]:
            d[off[b]:off[b + 1]] = t[off[b]:off[b + 1]] - t[off[b + 1] - 1]
    return x, y, t, d, p, off


def candidate_sets(kind, B, J, seed):
    """(B,J,K): per window its base parameters perturbed by up to 20 %, the first candidate the base itself and the
    second one that sends every event off the canvas"""
    rng = np.random.default_rng(seed)
    base = np.array(BASE[kind][:B], np.float64)
    c = base[:, None, :] * (1 + rng.uniform(-0.2, 0.2, (B, J, base.shape[1]))) + rng.uniform(-1, 1, (B, J, base.shape[1]))
    c[:, 0] = base
    if J > 1:
        c[:, 1] = GONE[kind]
    return c


def _ev(x, y, t, p):
    return [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (x, y, t, p)]


def candidates(kind, x, y, t, p, off, cand, sigma, reverse=False, t0=None):
    from event_utils_b200.contrast_max import motion_timestamp_candidates_torch
    return motion_timestamp_candidates_torch(*_ev(x, y, t, p), torch.tensor(cand, device="cuda"), _warp(kind), t0=t0,
                                             blur_sigma=sigma, timestamp_reverse=reverse, img_size=(H, W),
                                             batch_end_indices=torch.from_numpy(off[1:]).cuda()).cpu().numpy()


def per_candidate(kind, x, y, t, p, off, cand, sigma, reverse=False, t0=None):
    """motion_timestamp_objective_torch once per candidate index j: (B,J)"""
    from event_utils_b200.contrast_max import motion_timestamp_objective_torch
    ev = _ev(x, y, t, p)
    ends = torch.from_numpy(off[1:]).cuda()
    out = np.empty(cand.shape[:2])
    for j in range(cand.shape[1]):
        out[:, j] = motion_timestamp_objective_torch(*ev, torch.tensor(cand[:, j], device="cuda"), _warp(kind), t0=t0,
                                                     blur_sigma=sigma, timestamp_reverse=reverse, img_size=(H, W),
                                                     batch_end_indices=ends).cpu().numpy()
    return out


@pytest.mark.parametrize("kind", ["linvel", "rotation", "xyztheta"])
@pytest.mark.parametrize("sigma", [0.0, 1.0, 2.0, 3.0])
@pytest.mark.parametrize("reverse", [False, True])
@pytest.mark.parametrize("batch", [1, 5])
def test_candidates_against_the_forward_and_the_reference(kind, sigma, reverse, batch):
    sizes = [20000] if batch == 1 else [15000, 0, 9000, 20000, 1]      # an empty and a one-event window
    x, y, t, _, p, off = batch_stream(7 + batch, sizes)
    # t0 0.01 after each window's last stamp: no event has d = 0, where every motion is the identity, so that a fast
    # enough motion sends every event off the canvas
    t0 = np.array([t[off[b + 1] - 1] + np.float32(0.01) if sizes[b] else 0 for b in range(batch)], np.float32)
    d = np.concatenate([t[off[b]:off[b + 1]] - t0[b] for b in range(batch)]).astype(np.float32)
    for J in (1, 7, 32, 70):
        cand = candidate_sets(kind, batch, J, seed=J)
        if J >= 32:
            cand[0, 3] = np.nan                                        # contributes no event, and only to its own entry
        f = candidates(kind, x, y, t, p, off, cand, sigma, reverse, t0)
        ref = per_candidate(kind, x, y, t, p, off, cand, sigma, reverse, t0)
        assert np.isfinite(f).all()
        np.testing.assert_allclose(f, ref, rtol=1e-6, atol=0, err_msg="%s %g %s J=%d" % (kind, sigma, reverse, J))
        if batch == 5:
            assert (f[1] == 0).all() and (f[4] == 0).all()             # no event; a lone event has tau = 0
        if J > 1:
            assert (f[:, 1] == 0).all()                                # every event off the canvas
        if J >= 32:
            assert f[0, 3] == 0                                        # the NaN candidate: no event
            c2 = cand.copy()
            c2[0, 3] = cand[0, 2]
            f2 = candidates(kind, x, y, t, p, off, c2, sigma, reverse, t0)
            others = np.ones(f.shape, bool)
            others[0, 3] = False
            np.testing.assert_allclose(f2[others], f[others], rtol=1e-6, atol=0)
        if J == 7:
            tau = R.tau_f32(t, off, reverse)
            fr = np.stack([R.reference(kind, x, y, d, tau, p, off, torch.tensor(cand[:, j]), sigma, (H, W), CENTRE)[0]
                           .detach().numpy() for j in range(J)], axis=1)
            np.testing.assert_allclose(f, fr, rtol=1e-5, atol=1e-30)


def _entry(L, name, *args):
    from event_utils_b200 import _lib
    _lib.check(getattr(L, name)(*args))


def test_exactly_summable_streams_bit_for_bit():
    """quarter-pixel warped coordinates (tests/edge_cases.py) and stamps tau on a 1/16 grid: every tap and pixel sum is
    exact in f32, so each candidate's T images equal those of evk_motion_timestamp_objective_f32 at that candidate bit
    for bit -- also when the windows are split into chunks.  f is then the same f64 sum of the same G^2 terms, whose
    per-CTA partial sums both entries add with atomics in no fixed order: equal to 1e-13, far below what one tap of
    1/256 moved to another pixel changes"""
    from event_utils_b200 import _lib
    from event_utils_b200.contrast_max import motion_timestamp_objective as MT
    L = _lib.lib()
    c = exact_streams(3, "cmax", 300001)
    h, w = c["Hs"], c["Ws"]
    x, y, d, p = (np.asarray(c[k], np.float32) for k in ("x", "y", "t", "p"))
    n = x.shape[0]
    tau = (np.random.default_rng(8).integers(0, 17, n) / 16.0).astype(np.float32)
    off = np.array([0, 100000, 100000, n], np.int64)
    centre = (20.0, 12.0)
    X, Y, D, U, P, O = (torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (x, y, d, tau, p, off))
    models = {"linvel": [(c["vx"], c["vy"]), (c["vx"], 0.0)], "xyztheta": [(c["vx"], c["vy"], 0.0, 0.0)],
              "rotation": [(20.0, 12.0, 0.0), (21.0, 13.5, 0.0), (22.25, 10.0, 0.0), (-3.0, 40.0, 0.0)]}
    for kind, prm in models.items():
        cand = torch.tensor([[prm[(b + j) % len(prm)] for j in range(5)] for b in range(3)], dtype=torch.float64,
                            device="cuda")
        opts = (WARP[kind], centre, h, w, 0.0)
        f = MT._ts_candidates(X, Y, D, U, P, O, cand, opts).cpu().numpy()
        saved = MT.TIMESTAMP_CANDIDATES_WORKSPACE_BYTES
        try:
            MT.TIMESTAMP_CANDIDATES_WORKSPACE_BYTES = 1            # one window per chunk
            fc = MT._ts_candidates(X, Y, D, U, P, O, cand, opts).cpu().numpy()
        finally:
            MT.TIMESTAMP_CANDIDATES_WORKSPACE_BYTES = saved
        ref = np.empty((3, 5))
        ws = torch.empty(L.evk_motion_timestamp_objective_workspace_bytes(3, h, w), dtype=torch.uint8, device="cuda")
        for j in range(5):
            prm_j = cand[:, j].contiguous()
            fj = torch.empty(3, dtype=torch.float64, device="cuda")
            T = torch.empty((3, 2, h + 1, w + 1), device="cuda")
            C = torch.empty_like(T)
            _entry(L, "evk_motion_timestamp_objective_f32", X.data_ptr(), Y.data_ptr(), D.data_ptr(), U.data_ptr(), P.data_ptr(),
                   O.data_ptr(), 3, n, WARP[kind], prm_j.data_ptr(), cand.shape[2], centre[0], centre[1],
                   h, w, 0.0, fj.data_ptr(), T.data_ptr(), C.data_ptr(), ws.data_ptr(), ws.numel(), None)
            ref[:, j] = fj.cpu().numpy()
        np.testing.assert_allclose(f, ref, rtol=1e-13, atol=0, err_msg=kind)
        np.testing.assert_allclose(fc, ref, rtol=1e-13, atol=0, err_msg=kind)
        assert (f[1] == 0).all() and (f[[0, 2]] > 0).all()


# ---- the fit ------------------------------------------------------------------------------------------------------------
def host_windows(kind, B, seed, n_pts=300, per_pt=50):
    """(truths (B,K), (x, y, t, p) f64, ends): one window per true motion, test_gpu_motion_fit.windows' scenes"""
    rng = np.random.default_rng(seed)
    truths, duration = truths_of(kind, rng, B)
    (x, y, t, p), ends = windows(kind, truths, duration, rng, n_pts=n_pts, per_pt=per_pt)
    return rng, truths, (x, y, t, p), ends


def _device_windows(kind, B, seed, **kw):
    rng, truths, (x, y, t, p), ends = host_windows(kind, B, seed, **kw)
    ev = [torch.from_numpy(a).float().cuda() for a in (x, y, p)]
    return rng, truths, (ev[0], ev[1], torch.from_numpy(t).cuda(), ev[2]), torch.tensor(ends, device="cuda")


def _f_at(kind, ev, ends, params, sigma):
    from event_utils_b200.contrast_max import motion_timestamp_objective_torch
    return motion_timestamp_objective_torch(*ev, torch.as_tensor(params, device="cuda"), _warp(kind, FIT_CENTRE),
                                            blur_sigma=sigma, batch_end_indices=ends).cpu().numpy()


def _assert_recovered(kind, fit, truths, ev, ends, sigma):
    """every window within the contrast fit test's tolerance of its true motion -- or, for at most 2 of 64, at an f below
    the loss's value at the true motion (the loss's own minimum of such a window lies outside the tolerance)"""
    got = fit.params.cpu().numpy()
    ok = recovered(kind, got, truths)
    f_true = _f_at(kind, ev, ends, truths, sigma)
    beyond = ~ok & (fit.f.cpu().numpy() < f_true)
    assert (ok | beyond).all() and beyond.sum() <= 2, (np.flatnonzero(~ok), got[~ok], truths[~ok], fit.status.cpu().numpy()[~ok],
                                                      fit.f.cpu().numpy()[~ok], f_true[~ok])


def _assert_inside(params, bounds):
    assert ((params >= bounds[..., 0]) & (params <= bounds[..., 1])).all()


@pytest.mark.parametrize("kind", ["linvel", "rotation"])
def test_grid_start_recovers_every_window(kind):
    from event_utils_b200.contrast_max import motion_timestamp_fit_torch
    rng, truths, ev, ends = _device_windows(kind, 64, FIT_SEEDS[kind], **FIT_WINDOW)
    ranges = torch.tensor(FIT_RANGES[kind], device="cuda", dtype=torch.float64)
    fit = motion_timestamp_fit_torch(*ev, _warp(kind, FIT_CENTRE), batch_end_indices=ends, blur_sigma=FIT_BLURS,
                                     param_ranges=ranges, max_iter=40)
    _assert_recovered(kind, fit, truths, ev, ends, FIT_BLURS[-1])
    step = (ranges[:, 1] - ranges[:, 0]) / 4
    _assert_inside(fit.params, torch.stack((ranges[:, 0] - step, ranges[:, 1] + step), -1))
    np.testing.assert_allclose(fit.f.cpu().numpy(), _f_at(kind, ev, ends, fit.params, FIT_BLURS[-1]), rtol=1e-6, atol=0)
    assert fit.params.dtype == torch.float64 and fit.status.dtype == torch.int8 and fit.iterations.dtype == torch.int32


def _start_near(kind, truths, rng):
    if kind == "rotation":
        return np.column_stack((truths[:, :2] + rng.uniform(-2, 2, (len(truths), 2)),
                                truths[:, 2] * rng.uniform(0.85, 1.15, len(truths))))
    return truths * (1 + rng.uniform(-0.15, 0.15, truths.shape))


def _near_bounds(start):
    """a box of +-30 % (and at least 1) around each start"""
    half = np.maximum(0.3 * np.abs(start), 1.0)
    return np.stack((start - half, start + half), axis=-1)


def test_4dof_from_a_near_start_recovers_every_window():
    from event_utils_b200.contrast_max import motion_timestamp_fit_torch
    rng, truths, ev, ends = _device_windows("xyztheta", 64, 163, **FIT_WINDOW)
    x0 = _start_near("xyztheta", truths, rng)
    bounds = torch.tensor(_near_bounds(x0), device="cuda")
    fit = motion_timestamp_fit_torch(*ev, _warp("xyztheta", FIT_CENTRE), batch_end_indices=ends, blur_sigma=1.0,
                                     x0=torch.tensor(x0, device="cuda"), bounds=bounds, param_scale=[1.0, 1.0, 0.1, 0.1],
                                     max_iter=60)
    _assert_recovered("xyztheta", fit, truths, ev, ends, 1.0)
    _assert_inside(fit.params, bounds)


@pytest.mark.parametrize("kind", ["linvel", "rotation", "xyztheta"])
def test_no_worse_than_scipy_and_f_is_the_objective_at_params(kind):
    """per window scipy BFGS (jac=True) on motion_timestamp_objective_torch from the same start: the fit's f is no worse
    (see below), equals the loss at its params, and no window ends above its start"""
    import scipy.optimize as opt
    from event_utils_b200.contrast_max import motion_timestamp_fit_torch, motion_timestamp_objective_torch
    rng, truths, ev, ends = _device_windows(kind, 8, {"linvel": 171, "rotation": 172, "xyztheta": 173}[kind], n_pts=200,
                                            per_pt=100)
    x0 = _start_near(kind, truths, rng)
    warp = _warp(kind, FIT_CENTRE)
    scale = {"linvel": [1.0, 1.0], "rotation": [0.5, 0.5, 0.05], "xyztheta": [1.0, 1.0, 0.1, 0.1]}[kind]
    fit = motion_timestamp_fit_torch(*ev, warp, batch_end_indices=ends, x0=torch.tensor(x0, device="cuda"),
                                     bounds=torch.tensor(_near_bounds(x0), device="cuda"), param_scale=scale, max_iter=60)
    f_fit = fit.f.cpu().numpy()
    f_at = motion_timestamp_objective_torch(*ev, fit.params, warp, batch_end_indices=ends).cpu().numpy()
    np.testing.assert_allclose(f_fit, f_at, rtol=1e-6, atol=0)
    f_start = motion_timestamp_objective_torch(*ev, torch.tensor(x0, device="cuda"), warp, batch_end_indices=ends).cpu().numpy()
    assert (f_fit <= f_start + 1e-6 * np.abs(f_start)).all(), (f_fit, f_start)
    e = ends.cpu().numpy()
    f_sp = np.empty(len(x0))
    for b in range(len(x0)):
        sl = slice(0 if b == 0 else e[b - 1], e[b])
        wev = [a[sl] for a in ev]

        def fun(q):
            prm = torch.tensor(q, device="cuda", requires_grad=True)
            f = motion_timestamp_objective_torch(*wev, prm, warp)
            f.sum().backward()
            return f.item(), prm.grad.cpu().numpy()
        f_sp[b] = opt.minimize(fun, x0[b], jac=True, method="BFGS").fun
    res = fit.status.cpu().numpy()
    worse = f_fit - f_sp
    assert (worse <= 1e-4 * np.abs(f_sp)).all(), (worse / np.abs(f_sp), res)
    assert (worse <= 1e-6 * np.abs(f_sp)).sum() >= 6, (worse / np.abs(f_sp), res)


def test_empty_and_nan_windows_change_no_other_window():
    from event_utils_b200.contrast_max import motion_timestamp_fit_torch
    rng, truths, (x, y, t, p), ends = _device_windows("rotation", 4, 181, n_pts=200, per_pt=100)
    x0 = _start_near("rotation", truths, rng)
    e = ends.cpu().numpy()
    # window 1's events are cut out (an empty window); then window 2 gets a NaN event and window 3 a NaN start
    keep = torch.ones(x.shape[0], dtype=torch.bool, device="cuda")
    keep[e[0]:e[1]] = False
    x2, y2, t2, p2 = (a[keep].clone() for a in (x, y, t, p))
    n1 = e[1] - e[0]
    ends2 = torch.tensor([e[0], e[0], e[2] - n1, e[3] - n1], device="cuda")
    warp = _warp("rotation", FIT_CENTRE)
    kw = dict(batch_end_indices=ends2, bounds=torch.tensor(_near_bounds(x0), device="cuda"), param_scale=[0.5, 0.5, 0.05],
              max_iter=30)
    base = motion_timestamp_fit_torch(x2, y2, t2, p2, warp, x0=torch.tensor(x0, device="cuda"), **kw)
    x3 = x2.clone()
    x3[e[0] + 7] = float("nan")                                         # the 8th event of window 2
    start = x0.copy()
    start[3, 2] = np.nan
    bad = motion_timestamp_fit_torch(x3, y2, t2, p2, warp, x0=torch.tensor(start, device="cuda"), **kw)
    assert base.status[1].item() == 0 and base.f[1].item() == 0.0 and base.iterations[1].item() == 0
    assert np.array_equal(base.params[1].cpu().numpy(), x0[1])
    assert bad.status[3].item() == 3 and np.isnan(bad.params[3, 2].item())
    assert np.isfinite(bad.f[:3].cpu().numpy()).all()
    # window 0 is untouched; window 2 sees the same f up to one event of 20000 (a NaN position contributes nothing)
    assert torch.equal(bad.params[0], base.params[0]) or abs(bad.f[0].item() - base.f[0].item()) <= 1e-5 * abs(base.f[0].item())
    assert abs(bad.f[2].item() - base.f[2].item()) <= 1e-3 * abs(base.f[2].item())


def test_no_host_sync_and_constant_launch_count():
    from event_utils_b200 import _lib
    from event_utils_b200.contrast_max import motion_timestamp_fit_torch
    L = _lib.lib()
    counts = []
    for B in (1, 64):
        _, _, ev, ends = _device_windows("rotation", B, 90 + B, n_pts=100, per_pt=50)
        ranges = torch.tensor(FIT_RANGES["rotation"], device="cuda")
        kw = dict(batch_end_indices=ends, blur_sigma=(2.0, 1.0), param_ranges=ranges, grid_levels=2, max_iter=5)
        motion_timestamp_fit_torch(*ev, _warp("rotation", FIT_CENTRE), **kw)     # warm-up: scratch buffers, modules
        torch.cuda.synchronize()
        L.evk_prof_enable(1)
        torch.cuda.set_sync_debug_mode("error")
        try:
            fit = motion_timestamp_fit_torch(*ev, _warp("rotation", FIT_CENTRE), **kw)
        finally:
            torch.cuda.set_sync_debug_mode(0)
        ms, timed, launches = ctypes.c_double(), ctypes.c_longlong(), ctypes.c_longlong()
        _lib.check(L.evk_prof_collect(ctypes.byref(ms), ctypes.byref(timed), ctypes.byref(launches)))
        L.evk_prof_enable(0)
        assert torch.isfinite(fit.f).all()
        counts.append(launches.value)
    assert counts[0] == counts[1] and counts[0] > 0, counts
