"""The rotation and 4-DoF motion models on the GPU (evk_cmax_warp_objective_*): f and the gradient against the
K-channel oracle, against linvel where the models coincide, against the generic host-warp path, in batches, and
in the optimisation drivers."""
import numpy as np
import pytest

from cmax_warp_oracle import cmax_objective_warp, iwe_warp, objective_of_images

pytestmark = pytest.mark.gpu

NAMES = ["variance", "sos", "soe", "moa", "isoa", "sosa"]


@pytest.fixture(autouse=True)
def _reset():
    from event_utils_b200.contrast_max import objectives
    objectives.precision, objectives.event_pass = "f64", None
    objectives.clear_cache()
    yield
    objectives.precision, objectives.event_pass = "f64", None
    objectives.clear_cache()


def _objective(name):
    from event_utils_b200.contrast_max import objectives as O
    return getattr(O, name + "_objective")()


def _random_events(seed, n):
    rng = np.random.default_rng(seed)
    xs, ys = rng.random(n) * 239.0, rng.random(n) * 179.0
    ts = np.sort(rng.random(n)) * 0.05
    ps = rng.integers(0, 2, n) * 2.0 - 1.0
    return xs, ys, ts, ps


def _coefficient(name, iwe, sigma, param):
    """the objective's per-pixel coefficient image C and the factor s of g_k = s sum C G(D_k)"""
    from oracle import evk_oracle as O
    P = iwe.size
    img = iwe.astype(np.float64)
    g = O.gaussian_filter_f32(iwe, sigma).astype(np.float64) if sigma > 0 else img
    if name == "variance":
        return 2 * (img - img.mean()), 1.0 / P
    if name == "sos":
        return 2 * img, 1.0 / P
    if name == "soe":
        return np.exp(g), 1.0 / P
    if name == "isoa":
        return (g > param).astype(np.float64), 1.0
    return param * np.exp(-param * g), 1.0


def _gscale(name, iwe, d, sigma, param):
    """per channel: |s| P sqrt(mean(C^2) mean(D_k^2)) -- for the variance sqrt(mean((2(I-mu))^2) mean(D_k^2))"""
    C, s = _coefficient(name, iwe, sigma, param)
    return np.array([s * C.size * np.sqrt(np.mean(C * C) * np.mean(d[k].astype(np.float64) ** 2)) for k in range(d.shape[0])])


def _check(name, f, g, fo, go, scale, rel):
    if name == "isoa":
        assert abs(f - fo) <= 3, (f, fo)                     # pixels within an ulp of the threshold may flip
    else:
        assert abs(f - fo) <= rel * abs(fo), (name, f, fo)
    if name == "moa":
        assert g is None
        return
    tol = (20 * rel if name == "isoa" else rel) * np.maximum(scale, 1e-300)
    assert g.shape == go.shape and np.all(np.abs(g - go) <= tol), (name, g, go, tol)


MODEL_POINTS = [("rotation", (130.0, 85.0, 5.0)), ("rotation", (60.0, 40.0, -40.0)),          # the second leaves the canvas
                ("xyztheta", (20.0, -10.0, 4.0, 3.0)), ("xyztheta", (400.0, -300.0, 30.0, -25.0))]


def _warp(kind):
    from event_utils_b200.contrast_max.warps import pure_rotation_warp, xyztheta_warp
    return pure_rotation_warp() if kind == "rotation" else xyztheta_warp()


def test_against_the_oracle_every_objective_blur_precision_and_event_pass(oracle):
    from event_utils_b200.contrast_max import objectives as OB
    ev = _random_events(11, 400000)
    for kind, params in MODEL_POINTS:
        warp = _warp(kind)
        images = {pol: iwe_warp(warp, params, *ev, compute_gradient=True, use_polarity=pol)[:2] for pol in (True, False)}
        for name in NAMES:
            use_pol = oracle.OBJECTIVE_DEFAULTS[name][0]
            iwe, d = images[use_pol]
            param = oracle.OBJECTIVE_DEFAULTS[name][2]
            for sigma in (0.0, 1.0, 3.0):
                fo, go = objective_of_images(name, iwe, d, sigma, param)
                scale = _gscale(name, iwe, d, sigma, param) if go is not None else None
                for precision, rel in (("f64", 1e-5), ("f32", 1e-4)):
                    OB.precision = precision
                    for event_pass in ("onchip", "l2"):
                        OB.event_pass = event_pass
                        obj = _objective(name)
                        f = obj.evaluate_function(params, *ev, warp, (180, 240), sigma)
                        g = obj.evaluate_gradient(params, *ev, warp, (180, 240), sigma)
                        _check(name, f, g, fo, go, scale, rel)
                OB.precision, OB.event_pass = "f64", None
    # a slice that starts one element in: misaligned device pointers (no 16-byte vector loads)
    kind, params = MODEL_POINTS[2]
    warp = _warp(kind)
    sl = [a[1:] for a in ev]
    for precision, rel in (("f64", 1e-5), ("f32", 1e-4)):
        OB.precision = precision
        for event_pass in ("onchip", "l2"):
            OB.event_pass = event_pass
            res, iwe_g = OB._fused_model(warp, params, *ev, (180, 240), 1.0, True, True, first=1, want_image=True)
            fo, go, iwe, d = cmax_objective_warp("variance", warp, params, *sl, blur_sigma=1.0)
            _check("variance", res[0], res[1:5], fo, go, _gscale("variance", iwe, d, 1.0, None), rel)
            assert np.abs(iwe_g - iwe).max() <= rel * np.abs(iwe).max()


def _summable_events(seed, n):
    """coordinates on a 1/8 grid, times on a 1/32 grid: every tap and every pixel sum is exact in f32, in any order"""
    rng = np.random.default_rng(seed)
    xs, ys = rng.integers(8, 1900, n) / 8.0, rng.integers(8, 1420, n) / 8.0
    ts = np.sort(rng.integers(0, 32, n)) / 32.0
    ps = rng.integers(0, 2, n) * 2.0 - 1.0
    return xs, ys, ts, ps


def test_xyztheta_without_expansion_and_rotation_is_linvel():
    from event_utils_b200.contrast_max import objectives as OB
    from event_utils_b200.contrast_max.warps import linvel_warp, xyztheta_warp
    ev = _summable_events(12, 400000)
    for precision in ("f64", "f32"):
        OB.precision = precision
        for event_pass in ("onchip", "l2"):
            OB.event_pass = event_pass
            for hx, hy in ((48.0, -32.0), (-7.0, 3.0)):
                a, _ = OB.get_iwe((hx, hy, 0.0, 0.0), *ev, xyztheta_warp(), (180, 240))
                b, _ = OB.get_iwe((hx, hy), *ev, linvel_warp(), (180, 240))
                assert np.array_equal(a, b), (precision, event_pass, hx, hy)
                res, _ = OB._fused_model(xyztheta_warp(), (hx, hy, 0.0, 0.0), *ev, (180, 240), 1.0, True, True)
                lin, iwe, d = OB._fused_linvel((hx, hy), *ev, (180, 240), 1.0, True, True, want_images=True, channel_mix=False)
                assert abs(res[0] - lin[0]) <= 1e-6 * abs(lin[0])
                scale = _gscale("variance", iwe, d, 1.0, None)
                assert np.all(np.abs(res[1:3] - lin[1:3]) <= 1e-5 * scale), (res[1:3], lin[1:3], scale)


@pytest.mark.parametrize("kind", ["rotation", "xyztheta"])
def test_fused_equals_the_generic_path_and_the_precomputed_forms(kind):
    from event_utils_b200.contrast_max import objectives as OB
    warp = _warp(kind)

    class generic(type(warp)):
        fused_kind = None
    gw = generic()
    ev = _random_events(13, 200000)
    params = MODEL_POINTS[0 if kind == "rotation" else 2][1]
    for name in ("variance", "sos", "soe", "sosa"):
        f, g = _objective(name).evaluate_function(params, *ev, warp, (180, 240), 1.0), \
            _objective(name).evaluate_gradient(params, *ev, warp, (180, 240), 1.0)
        fg, gg = _objective(name).evaluate_function(params, *ev, gw, (180, 240), 1.0), \
            _objective(name).evaluate_gradient(params, *ev, gw, (180, 240), 1.0)
        iwe, d = OB.get_iwe(params, *ev, warp, (180, 240), compute_gradient=True,
                            use_polarity=_objective(name).use_polarity)
        assert d.shape == (warp.dims, 181, 241)
        scale = _gscale(name, iwe, d, 1.0, 3.0)
        _check(name, f, g, fg, gg, scale, 1e-5)
        fp = _objective(name).evaluate_function(iwe=iwe, blur_sigma=1.0)
        gp = _objective(name).evaluate_gradient(iwe=iwe, d_iwe=d, blur_sigma=1.0)
        _check(name, f, g, fp, gp, scale, 1e-5)
    iwe_f, none = OB.get_iwe(params, *ev, warp, (180, 240))
    iwe_g, _ = OB.get_iwe(params, *ev, gw, (180, 240))
    assert none is None and np.abs(iwe_f - iwe_g).max() <= 1e-5 * np.abs(iwe_g).max()


def test_batch_and_grid_search():
    from event_utils_b200.contrast_max import objectives as OB
    from event_utils_b200.contrast_max.events_cmax import grid_search_initial
    ev = _random_events(14, 100000)
    rng = np.random.default_rng(15)
    for kind, lo, hi in (("rotation", (100, 60, -20), (160, 120, 20)), ("xyztheta", (-50, -50, -5, -5), (50, 50, 5, 5))):
        warp = _warp(kind)
        pts = [tuple(v) for v in rng.uniform(lo, hi, size=(40, warp.dims))]           # > 32: two batches
        for obj in (OB.variance_objective(), OB.sos_objective(), OB.sosa_objective(), OB.moa_objective()):
            f, g = OB.evaluate_candidates(obj, pts, *ev, warp, (180, 240), blur_sigma=1.0)
            assert g is None
            for k in (0, 7, 33, 39):
                fk = obj.evaluate_function(pts[k], *ev, warp, (180, 240), 1.0)
                assert abs(f[k] - fk) <= 1e-6 * abs(fk), (kind, obj.name, k, f[k], fk)
        f, g = OB.evaluate_candidates(OB.variance_objective(), pts[:3], *ev, warp, (180, 240), 1.0, want_grad=True)
        assert g.shape == (3, warp.dims)
        out = grid_search_initial(*ev, warp, OB.variance_objective(), (180, 240), num_samples_per_param=5)
        assert len(out["params"]) == 5 ** warp.dims and len(out["search_axes"]) == warp.dims
        assert out["min_func_eval"] == min(min(out["eval"]), 0)


def _points_scene(seed, n_pts, per_pt, centre, radius):
    rng = np.random.default_rng(seed)
    ang, rad = rng.uniform(0, 2 * np.pi, n_pts), radius * np.sqrt(rng.uniform(0.05, 1, n_pts))
    x0, y0 = np.repeat(centre[0] + rad * np.cos(ang), per_pt), np.repeat(centre[1] + rad * np.sin(ang), per_pt)
    ps = np.repeat(rng.integers(0, 2, n_pts) * 2.0 - 1.0, per_pt)
    return x0, y0, ps, rng


def test_recovers_known_rotation_and_4dof_motion():
    from event_utils_b200.contrast_max import objectives as OB
    from event_utils_b200.contrast_max.events_cmax import optimize_contrast
    from event_utils_b200.contrast_max.warps import pure_rotation_warp, xyztheta_warp
    # rotation about (130, 85) at 5 rad/s over 50 ms
    x0, y0, ps, rng = _points_scene(21, 400, 150, (130.0, 85.0), 75.0)
    ts = np.sort(rng.uniform(0, 0.05, x0.size))
    order = rng.permutation(x0.size)
    x0, y0, ps = x0[order], y0[order], ps[order]
    a = 5.0 * (ts - ts[-1])
    u, v = x0 - 130.0, y0 - 85.0
    xs, ys = 130.0 + np.cos(a) * u - np.sin(a) * v, 85.0 + np.sin(a) * u + np.cos(a) * v
    est = optimize_contrast(xs, ys, ts, ps, pure_rotation_warp(), OB.variance_objective(), x0=np.array([125.0, 90.0, 0.0]),
                            blur_sigma=1.0)
    assert abs(est[2] - 5.0) <= 0.02 * 5.0 and np.hypot(est[0] - 130.0, est[1] - 85.0) <= 1.5, est
    # xyztheta (20, -10) px/s, hz = 4 /s, theta = 3 rad/s about the default centre, positions from the first-order
    # model.  Over 200 ms: the translation moves a point by 4 and 2 px, so 5 % of it is well above the sub-pixel
    # wobble of a bilinear image's contrast (over 50 ms the estimates of hx, hy scatter by 5-25 %)
    truth = np.array([20.0, -10.0, 4.0, 3.0])
    w = xyztheta_warp()
    x0, y0, ps, rng = _points_scene(22, 400, 400, w.center, 50.0)
    ts = np.sort(rng.uniform(0, 0.2, x0.size))
    order = rng.permutation(x0.size)
    x0, y0, ps = x0[order], y0[order], ps[order]
    dt = ts - ts[-1]
    hx, hy, hz, th = truth
    bx, by = (x0 - w.center[0]) + dt * hx, (y0 - w.center[1]) + dt * hy
    m00, m01, m10, m11 = 1 - dt * hz, dt * th, -dt * th, 1 - dt * hz
    det = m00 * m11 - m01 * m10
    xs, ys = w.center[0] + (m11 * bx - m01 * by) / det, w.center[1] + (m00 * by - m10 * bx) / det
    est = optimize_contrast(xs, ys, ts, ps, w, OB.variance_objective(), blur_sigma=1.0)
    assert np.all(np.abs(est - truth) <= 0.05 * np.abs(truth)), est


def test_errors_and_edges():
    from event_utils_b200 import _lib
    from event_utils_b200.contrast_max import objectives as OB
    for kind, params in MODEL_POINTS[::2]:
        warp = _warp(kind)
        e = np.zeros(0)
        with pytest.raises(IndexError):
            OB.variance_objective().evaluate_function(params, e, e, e, e, warp, (180, 240), 1.0)
        xs, ys, ts, ps = _random_events(31, 1000)
        xs[500] = np.nan                     # kept by the bounds mask (NaN compares false), then outside the canvas
        with pytest.raises(IndexError):
            OB.variance_objective().evaluate_function(params, xs, ys, ts, ps, warp, (180, 240), 1.0)
        with pytest.raises(IndexError):
            OB.evaluate_candidates(OB.variance_objective(), [params], xs, ys, ts, ps, warp, (180, 240))
    L = _lib.lib()
    one = np.zeros(6)
    assert L.evk_cmax_warp_objective_f64(None, None, None, None, 0, 1.0, 7, one.ctypes.data, 0.0, 180, 240, 180, 240, 1.0, 0,
                                         0, 0.0, None, None, None, 0, None) == -1
    assert b"unknown warp" in L.evk_last_error()
