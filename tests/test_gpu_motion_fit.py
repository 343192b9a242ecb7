"""The multi-candidate pass (evk_cmax_motion_candidates_f32, motion_contrast_candidates_torch) against the batched
forward it restates per candidate, and the batched fit (motion_contrast_fit_torch): recovery of known motions, scipy's
BFGS per window, monotonicity, and no host synchronisation."""
import ctypes

import numpy as np
import pytest
import torch

import motion_objective_reference as R
from edge_cases import exact_streams

pytestmark = pytest.mark.gpu

H, W = 60, 80
CENTRE = (40.0, 30.0)
BASE = {"linvel": [(30.0, -20.0), (-55.0, 12.5), (5.0, 8.0), (900.0, -700.0), (0.0, 0.0)],
        "rotation": [(40.0, 30.0, 4.0), (35.0, 28.0, -6.0), (45.0, 33.0, 1.5), (10.0, 10.0, 40.0), (40.0, 30.0, 0.0)],
        "xyztheta": [(20.0, -10.0, 3.0, 2.0), (-30.0, 15.0, -2.0, 4.0), (5.0, 5.0, 0.5, -3.0), (600.0, -500.0, 30.0, 9.0),
                     (0.0, 0.0, 0.0, 0.0)]}
# a candidate that sends every event off the canvas
GONE = {"linvel": (1e6, -1e6), "rotation": (1e5, 1e5, 50.0), "xyztheta": (1e6, 1e6, 0.0, 0.0)}


def _warp(kind, centre=CENTRE):
    from event_utils_b200.contrast_max import linvel_warp, pure_rotation_warp, xyztheta_warp
    return {"linvel": linvel_warp, "rotation": pure_rotation_warp, "xyztheta": lambda: xyztheta_warp(center=centre)}[kind]()


def batch_stream(seed, sizes, h=H, w=W):
    """concatenated windows; events in the sensor, d = t - t0 in [-0.1, -2^-12] on a 2^-12 grid (no event is at d = 0,
    where every motion is the identity, so that a fast enough motion sends every event off the canvas)"""
    rng = np.random.default_rng(seed)
    n = sum(sizes)
    x = (rng.random(n) * (w - 1)).astype(np.float32)
    y = (rng.random(n) * (h - 1)).astype(np.float32)
    p = (rng.integers(0, 2, n) * 2 - 1).astype(np.float32)
    d = np.empty(n, np.float32)
    off = np.concatenate(([0], np.cumsum(sizes))).astype(np.int64)
    for b in range(len(sizes)):
        d[off[b]:off[b + 1]] = -np.sort(rng.integers(1, 411, sizes[b]))[::-1] / 4096.0
    return x, y, d, p, off


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


def candidates(kind, x, y, d, p, off, cand, sigma, name, param=0.3, img_size=(H, W), centre=CENTRE):
    from event_utils_b200.contrast_max import motion_contrast_candidates_torch
    ev = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (x, y, d, p)]
    return motion_contrast_candidates_torch(*ev, torch.tensor(cand, device="cuda"), _warp(kind, centre), t0=0.0, objective=name,
                                            blur_sigma=sigma, obj_param=param, img_size=img_size,
                                            batch_end_indices=torch.from_numpy(off[1:]).cuda()).cpu().numpy()


def per_candidate(kind, x, y, d, p, off, cand, sigma, name, param=0.3, img_size=(H, W), centre=CENTRE):
    """motion_contrast_objective_torch once per candidate index j: (B,J)"""
    from event_utils_b200.contrast_max import motion_contrast_objective_torch
    ev = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (x, y, d, p)]
    ends = torch.from_numpy(off[1:]).cuda()
    out = np.empty(cand.shape[:2])
    for j in range(cand.shape[1]):
        f = motion_contrast_objective_torch(*ev, torch.tensor(cand[:, j], device="cuda"), _warp(kind, centre), t0=0.0,
                                            objective=name, blur_sigma=sigma, obj_param=param, img_size=img_size,
                                            batch_end_indices=ends)
        out[:, j] = f.cpu().numpy()
    return out


@pytest.mark.parametrize("kind", ["linvel", "rotation", "xyztheta"])
@pytest.mark.parametrize("name", ["variance", "sos", "soe", "sosa"])
@pytest.mark.parametrize("sigma", [0.0, 1.0, 3.0])
@pytest.mark.parametrize("batch", [1, 5])
def test_candidates_against_the_forward_and_the_reference(kind, name, sigma, batch):
    sizes = [20000] if batch == 1 else [15000, 0, 9000, 20000, 1]      # an empty and a one-event window
    x, y, d, p, off = batch_stream(7 + batch, sizes)
    for J in (1, 7, 32, 70):
        cand = candidate_sets(kind, batch, J, seed=J)
        if J >= 32:
            cand[0, 3] = np.nan                                        # contributes no event, and only to its own entry
        f = candidates(kind, x, y, d, p, off, cand, sigma, name)
        ref = per_candidate(kind, x, y, d, p, off, cand, sigma, name)
        assert np.isfinite(f).all()
        np.testing.assert_allclose(f, ref, rtol=1e-6, atol=0, err_msg="%s %s %g J=%d" % (kind, name, sigma, J))
        if batch == 5:
            assert (f[1] == f[1, 0]).all()                             # the empty window: the image of no event
        if batch == 5 and J > 1:
            assert (f[:, 1] == f[1, 0]).all()                          # every event off the canvas: no event either
        if J == 7:
            fr = np.stack([R.reference(kind, x, y, d, p, off, torch.tensor(cand[:, j]), sigma, name, 0.3, (H, W), CENTRE)[0]
                           .detach().numpy() for j in range(J)], axis=1)
            np.testing.assert_allclose(f, fr, rtol=1e-5, atol=1e-30)


def test_exactly_summable_streams_bit_for_bit():
    """quarter-pixel warped coordinates (tests/edge_cases.py): every image sum is exact, so f equals the batched forward's
    bit for bit where its statistics are exact too (variance, no blur) -- also through several chunks of windows"""
    from event_utils_b200.contrast_max import motion_objective as MO
    c = exact_streams(3, "cmax", 300001)
    h, w = c["Hs"], c["Ws"]
    x, y, t, p = (np.asarray(c[k], np.float32) for k in ("x", "y", "t", "p"))
    off = np.array([0, 100000, 100000, 300001], np.int64)
    models = {"linvel": [(c["vx"], c["vy"])], "xyztheta": [(c["vx"], c["vy"], 0.0, 0.0)],
              "rotation": [(20.0, 12.0, 0.0), (21.0, 13.5, 0.0), (22.25, 10.0, 0.0), (-3.0, 40.0, 0.0)]}
    for kind, prm in models.items():
        cand = np.array([[prm[(b + j) % len(prm)] for j in range(5)] for b in range(3)], np.float64)
        f = candidates(kind, x, y, t, p, off, cand, 0.0, "variance", img_size=(h, w), centre=(20.0, 12.0))
        ref = per_candidate(kind, x, y, t, p, off, cand, 0.0, "variance", img_size=(h, w), centre=(20.0, 12.0))
        assert np.array_equal(f, ref), (kind, f, ref)
        saved = MO.CANDIDATES_WORKSPACE_BYTES
        try:
            MO.CANDIDATES_WORKSPACE_BYTES = 1            # one window per chunk
            fc = candidates(kind, x, y, t, p, off, cand, 0.0, "variance", img_size=(h, w), centre=(20.0, 12.0))
        finally:
            MO.CANDIDATES_WORKSPACE_BYTES = saved
        assert np.array_equal(fc, f), kind


def _sparse_footprints(kind, cands, centre, h, w, seed, n=40000, gap=3):
    """events whose warped footprints lie at least `gap` pixels apart under EVERY candidate: every image pixel then
    receives at most one tap, so each candidate's image is the same whatever the order of the reductions"""
    rng = np.random.default_rng(seed)
    x = (rng.random(n) * (w - 1)).astype(np.float32)
    y = (rng.random(n) * (h - 1)).astype(np.float32)
    d = (-rng.integers(0, 410, n) / 4096.0).astype(np.float32)
    p = (rng.integers(0, 2, n) * 2 - 1).astype(np.float32)
    warped = [R.warp_f32(kind, x, y, d, prm, centre) for prm in cands]
    ok = np.logical_and.reduce([R.contributes(xw, yw, h, w) for xw, yw in warped])
    taken = np.zeros((len(cands), h + 1 + 2 * gap, w + 1 + 2 * gap), bool)
    pick = []
    for i in np.flatnonzero(ok):
        cells = [(int(np.floor(xw[i])) + gap, int(np.floor(yw[i])) + gap) for xw, yw in warped]
        if any(taken[j, cy - gap:cy + gap + 1, cx - gap:cx + gap + 1].any() for j, (cx, cy) in enumerate(cells)):
            continue
        for j, (cx, cy) in enumerate(cells):
            taken[j, cy, cx] = True
        pick.append(i)
    pick = np.array(pick)
    return tuple(a[pick] for a in (x, y, d, p))


def test_non_overlapping_footprints_under_every_model():
    """rotation, 4-DoF and linvel candidates with at most one tap per pixel: the images equal the forward's bit for bit,
    so f agrees to the f64 rounding of the statistics' reduction order"""
    h, w = 180, 240
    centre = (120.0, 90.0)
    models = {"linvel": [(30.0, -20.0), (25.0, -18.0), (33.0, -24.0)],
              "rotation": [(130.0, 85.0, 4.0), (125.0, 90.0, 3.0), (120.0, 80.0, 5.0)],
              "xyztheta": [(20.0, -10.0, 3.0, 2.0), (18.0, -12.0, 2.5, 2.5), (22.0, -8.0, 3.5, 1.5)]}
    for kind, cands in models.items():
        x, y, d, p = _sparse_footprints(kind, cands, centre, h, w, seed=37)
        assert x.shape[0] > 500, x.shape
        xd, yd, dd, pd, _ = batch_stream(38, [30000], h, w)
        off = np.array([0, x.shape[0], x.shape[0] + 30000], np.int64)
        cat = [np.concatenate(a) for a in ((x, xd), (y, yd), (d, dd), (p, pd))]
        cand = np.array([cands, cands], np.float64)
        for name, sigma in (("variance", 0.0), ("soe", 1.0)):
            f = candidates(kind, *cat, off, cand, sigma, name, img_size=(h, w), centre=centre)
            ref = per_candidate(kind, *cat, off, cand, sigma, name, img_size=(h, w), centre=centre)
            np.testing.assert_allclose(f[0], ref[0], rtol=1e-12, atol=0, err_msg=kind)
            np.testing.assert_allclose(f[1], ref[1], rtol=1e-6, atol=0, err_msg=kind)


def test_chunking_changes_no_value():
    from event_utils_b200.contrast_max import motion_objective as MO
    from event_utils_b200 import _lib
    sizes = [9000, 0, 7000, 12000, 1, 5000]
    x, y, d, p, off = batch_stream(51, sizes)
    cand = np.concatenate([candidate_sets("rotation", 5, 70, seed=9), candidate_sets("rotation", 1, 70, seed=10)])
    one = candidates("rotation", x, y, d, p, off, cand, 1.0, "variance")
    per = _lib.load().evk_cmax_motion_candidates_workspace_bytes(1, 32, H, W)
    saved = MO.CANDIDATES_WORKSPACE_BYTES
    try:
        MO.CANDIDATES_WORKSPACE_BYTES = 2 * per + 1       # two windows per chunk: three chunks of windows x three of J
        many = candidates("rotation", x, y, d, p, off, cand, 1.0, "variance")
    finally:
        MO.CANDIDATES_WORKSPACE_BYTES = saved
    np.testing.assert_allclose(many, one, rtol=1e-6, atol=0)


# ---- the fit ------------------------------------------------------------------------------------------------------------
def _scene(rng, n_pts, per_pt, centre, radius):
    ang, rad = rng.uniform(0, 2 * np.pi, n_pts), radius * np.sqrt(rng.uniform(0.05, 1, n_pts))
    x0, y0 = np.repeat(centre[0] + rad * np.cos(ang), per_pt), np.repeat(centre[1] + rad * np.sin(ang), per_pt)
    ps = np.repeat(rng.integers(0, 2, n_pts) * 2.0 - 1.0, per_pt)
    order = rng.permutation(x0.size)
    return x0[order], y0[order], ps[order]


def windows(kind, truths, duration, rng, n_pts=300, per_pt=200):
    """one window per true motion: a scene of points seen during `duration`, moving with that motion"""
    xs, ys, ts, ps, ends = [], [], [], [], []
    for tr in truths:
        centre = (tr[0], tr[1]) if kind == "rotation" else (120.0, 90.0)
        x0, y0, p = _scene(rng, n_pts, per_pt, centre, 60.0)
        t = np.sort(rng.uniform(0, duration, x0.size))
        dt = t - t[-1]
        if kind == "linvel":
            x, y = x0 + dt * tr[0], y0 + dt * tr[1]
        elif kind == "rotation":
            a = tr[2] * dt
            u, v = x0 - tr[0], y0 - tr[1]
            x, y = tr[0] + np.cos(a) * u - np.sin(a) * v, tr[1] + np.sin(a) * u + np.cos(a) * v
        else:
            hx, hy, hz, th = tr
            bx, by = (x0 - 120.0) + dt * hx, (y0 - 90.0) + dt * hy
            m00, m01, m10, m11 = 1 - dt * hz, dt * th, -dt * th, 1 - dt * hz
            det = m00 * m11 - m01 * m10
            x, y = 120.0 + (m11 * bx - m01 * by) / det, 90.0 + (m00 * by - m10 * bx) / det
        xs.append(x), ys.append(y), ts.append(t), ps.append(p)
        ends.append(sum(len(a) for a in xs))
    return [np.concatenate(a) for a in (xs, ys, ts, ps)], ends


def truths_of(kind, rng, B):
    s = lambda: rng.choice([-1, 1], B)
    if kind == "linvel":
        return np.column_stack((rng.uniform(20, 60, B) * s(), rng.uniform(20, 60, B) * s())), 0.2
    if kind == "rotation":
        return np.column_stack((rng.uniform(110, 130, B), rng.uniform(80, 100, B), rng.uniform(3, 8, B) * s())), 0.05
    return np.column_stack((rng.uniform(15, 30, B) * s(), rng.uniform(15, 30, B) * s(), rng.uniform(2, 4, B),
                            rng.uniform(2, 4, B) * s())), 0.2


def recovered(kind, got, truths):
    """the tolerances of the Adam test of test_gpu_cmax_motion_objective.py"""
    if kind == "rotation":
        return (np.abs(got[:, 2] - truths[:, 2]) <= 0.03 * np.abs(truths[:, 2])) & \
            (np.hypot(got[:, 0] - truths[:, 0], got[:, 1] - truths[:, 1]) <= 2.0)
    return np.all(np.abs(got - truths) <= 0.05 * np.abs(truths), axis=1)


def _device_windows(kind, B, seed, **kw):
    rng = np.random.default_rng(seed)
    truths, duration = truths_of(kind, rng, B)
    (x, y, t, p), ends = windows(kind, truths, duration, rng, **kw)
    ev = [torch.from_numpy(a).float().cuda() for a in (x, y, p)]
    return rng, truths, (ev[0], ev[1], torch.from_numpy(t).cuda(), ev[2]), torch.tensor(ends, device="cuda")


def _f_at(kind, ev, ends, params, sigma):
    from event_utils_b200.contrast_max import motion_contrast_objective_torch
    return motion_contrast_objective_torch(*ev, torch.tensor(params, device="cuda"), _warp(kind, (120.0, 90.0)), blur_sigma=sigma,
                                           batch_end_indices=ends).cpu().numpy()


def _assert_recovered(kind, fit, truths, ev, ends):
    """every window within the Adam test's tolerance of its true motion -- or, for at most 2 of 64, at an f below the
    objective's value at the true motion: the objective's own minimum of such a window lies outside the tolerance (a
    few pixels of scene per window), so no minimiser of f meets it"""
    got = fit.params.cpu().numpy()
    ok = recovered(kind, got, truths)
    f_true = _f_at(kind, ev, ends, truths, 1.0)
    beyond = ~ok & (fit.f.cpu().numpy() < f_true)
    assert (ok | beyond).all() and beyond.sum() <= 2, (np.flatnonzero(~ok), got[~ok], truths[~ok], fit.status.cpu().numpy()[~ok],
                                                      fit.f.cpu().numpy()[~ok], f_true[~ok])


RANGES = {"linvel": [[-80.0, 80.0], [-80.0, 80.0]], "rotation": [[105.0, 135.0], [75.0, 105.0], [-10.0, 10.0]]}


@pytest.mark.parametrize("kind", ["linvel", "rotation"])
def test_grid_start_recovers_every_window(kind):
    from event_utils_b200.contrast_max import motion_contrast_fit_torch
    rng, truths, ev, ends = _device_windows(kind, 64, {"linvel": 61, "rotation": 62}[kind])
    fit = motion_contrast_fit_torch(*ev, _warp(kind, (120.0, 90.0)), batch_end_indices=ends, blur_sigma=(2.0, 1.0),
                                    param_ranges=torch.tensor(RANGES[kind], device="cuda"), grid_levels=3, max_iter=40)
    _assert_recovered(kind, fit, truths, ev, ends)
    assert fit.params.dtype == torch.float64 and fit.status.dtype == torch.int8 and fit.iterations.dtype == torch.int32


def _start_near(kind, truths, rng):
    if kind == "rotation":
        return np.column_stack((truths[:, :2] + rng.uniform(-2, 2, (len(truths), 2)),
                                truths[:, 2] * rng.uniform(0.85, 1.15, len(truths))))
    return truths * (1 + rng.uniform(-0.15, 0.15, truths.shape))


def test_4dof_from_a_near_start_recovers_every_window():
    from event_utils_b200.contrast_max import motion_contrast_fit_torch
    rng, truths, ev, ends = _device_windows("xyztheta", 64, 63)
    x0 = torch.tensor(_start_near("xyztheta", truths, rng), device="cuda")
    fit = motion_contrast_fit_torch(*ev, _warp("xyztheta", (120.0, 90.0)), batch_end_indices=ends, blur_sigma=1.0, x0=x0,
                                    param_scale=[1.0, 1.0, 0.1, 0.1], max_iter=60)
    _assert_recovered("xyztheta", fit, truths, ev, ends)


@pytest.mark.parametrize("kind", ["linvel", "rotation", "xyztheta"])
def test_no_worse_than_scipy_and_f_is_the_objective_at_params(kind):
    """per window scipy BFGS (jac=True) on motion_contrast_objective_torch from the same start: the fit's f is no worse
    (see below), equals the objective at its params, and no window ends above its start"""
    import scipy.optimize as opt
    from event_utils_b200.contrast_max import motion_contrast_fit_torch, motion_contrast_objective_torch
    rng, truths, ev, ends = _device_windows(kind, 8, {"linvel": 71, "rotation": 72, "xyztheta": 73}[kind], n_pts=200, per_pt=100)
    x0 = _start_near(kind, truths, rng)
    warp = _warp(kind, (120.0, 90.0))
    scale = {"linvel": [1.0, 1.0], "rotation": [0.5, 0.5, 0.05], "xyztheta": [1.0, 1.0, 0.1, 0.1]}[kind]
    fit = motion_contrast_fit_torch(*ev, warp, batch_end_indices=ends, x0=torch.tensor(x0, device="cuda"), param_scale=scale,
                                    max_iter=60)
    f_fit = fit.f.cpu().numpy()
    f_at = motion_contrast_objective_torch(*ev, fit.params, warp, batch_end_indices=ends).cpu().numpy()
    np.testing.assert_allclose(f_fit, f_at, rtol=1e-6, atol=0)
    f_start = motion_contrast_objective_torch(*ev, torch.tensor(x0, device="cuda"), warp, batch_end_indices=ends).cpu().numpy()
    assert (f_fit <= f_start + 1e-6 * np.abs(f_start)).all(), (f_fit, f_start)
    e = ends.cpu().numpy()
    f_sp = np.empty(len(x0))
    for b in range(len(x0)):
        sl = slice(0 if b == 0 else e[b - 1], e[b])
        wev = [a[sl] for a in ev]

        def fun(q):
            prm = torch.tensor(q, device="cuda", requires_grad=True)
            f = motion_contrast_objective_torch(*wev, prm, warp)
            f.sum().backward()
            return f.item(), prm.grad.cpu().numpy()
        f_sp[b] = opt.minimize(fun, x0[b], jac=True, method="BFGS").fun
    # f32 images make f piecewise smooth with shallow local minima a fraction of a pixel apart, so two local methods
    # from the same start may end in neighbouring ones: no worse to 1e-6 for most windows, and to 1e-4 for every one
    worse = f_fit - f_sp
    assert (worse <= 1e-4 * np.abs(f_sp)).all(), (worse / np.abs(f_sp), fit.status.cpu().numpy())
    assert (worse <= 1e-6 * np.abs(f_sp)).sum() >= 6, (worse / np.abs(f_sp), fit.status.cpu().numpy())


def test_empty_and_nan_windows_change_no_other_window():
    from event_utils_b200.contrast_max import motion_contrast_fit_torch
    rng, truths, (x, y, t, p), ends = _device_windows("rotation", 4, 81, n_pts=200, per_pt=100)
    x0 = _start_near("rotation", truths, rng)
    e = ends.cpu().numpy()
    # window 1's events are cut out (an empty window); then window 2 gets a NaN event and window 3 a NaN start
    keep = torch.ones(x.shape[0], dtype=torch.bool, device="cuda")
    keep[e[0]:e[1]] = False
    x2, y2, t2, p2 = (a[keep].clone() for a in (x, y, t, p))
    n1 = e[1] - e[0]
    ends2 = torch.tensor([e[0], e[0], e[2] - n1, e[3] - n1], device="cuda")
    warp = _warp("rotation")
    kw = dict(batch_end_indices=ends2, param_scale=[0.5, 0.5, 0.05], max_iter=30)
    base = motion_contrast_fit_torch(x2, y2, t2, p2, warp, x0=torch.tensor(x0, device="cuda"), **kw)
    x3 = x2.clone()
    x3[e[0] + 7] = float("nan")                                         # the 8th event of window 2
    start = x0.copy()
    start[3, 2] = np.nan
    bad = motion_contrast_fit_torch(x3, y2, t2, p2, warp, x0=torch.tensor(start, device="cuda"), **kw)
    assert base.status[1].item() == 0 and base.f[1].item() == 0.0 and base.iterations[1].item() == 0
    assert np.array_equal(base.params[1].cpu().numpy(), x0[1])
    assert bad.status[3].item() == 3 and np.isnan(bad.params[3, 2].item())
    assert np.isfinite(bad.f[:3].cpu().numpy()).all()
    # the fits of windows 0 and 2 see the same f up to f32 rounding and one event of 20000
    assert abs(bad.f[0].item() - base.f[0].item()) <= 1e-5 * abs(base.f[0].item())
    assert abs(bad.f[2].item() - base.f[2].item()) <= 1e-3 * abs(base.f[2].item())


def test_no_host_sync_and_constant_launch_count():
    from event_utils_b200 import _lib
    from event_utils_b200.contrast_max import motion_contrast_fit_torch
    L = _lib.lib()
    counts = []
    for B in (1, 64):
        _, _, ev, ends = _device_windows("rotation", B, 90 + B, n_pts=100, per_pt=50)
        ranges = torch.tensor(RANGES["rotation"], device="cuda")
        kw = dict(batch_end_indices=ends, blur_sigma=(2.0, 1.0), param_ranges=ranges, grid_levels=2, max_iter=5)
        motion_contrast_fit_torch(*ev, _warp("rotation"), **kw)           # warm-up: scratch buffers, modules
        torch.cuda.synchronize()
        L.evk_prof_enable(1)
        torch.cuda.set_sync_debug_mode("error")
        try:
            fit = motion_contrast_fit_torch(*ev, _warp("rotation"), **kw)
        finally:
            torch.cuda.set_sync_debug_mode(0)
        ms, timed, launches = ctypes.c_double(), ctypes.c_longlong(), ctypes.c_longlong()
        _lib.check(L.evk_prof_collect(ctypes.byref(ms), ctypes.byref(timed), ctypes.byref(launches)))
        L.evk_prof_enable(0)
        assert torch.isfinite(fit.f).all()
        counts.append(launches.value)
    assert counts[0] == counts[1] and counts[0] > 0, counts
