"""No-GPU checks of the rotation and 4-DoF motion models (contrast_max/warps.py) and of their K-channel oracle."""
import numpy as np
import pytest

from cmax_warp_oracle import iwe_warp


def _events(seed, n=2000):
    rng = np.random.default_rng(seed)
    xs, ys = rng.uniform(5, 235, n), rng.uniform(5, 175, n)
    ts = np.sort(rng.uniform(0, 0.05, n))
    ps = rng.integers(0, 2, n) * 2.0 - 1.0
    return xs, ys, ts, ps


def _models():
    from event_utils_b200.contrast_max.warps import pure_rotation_warp, xyztheta_warp
    return [(pure_rotation_warp(), (130.0, 85.0, 5.0)), (pure_rotation_warp(), (-40.0, 300.0, -37.0)),
            (xyztheta_warp(), (20.0, -10.0, 4.0, 3.0)), (xyztheta_warp((100.0, 70.0)), (-55.0, 31.0, -6.5, 12.0))]


def test_models_declare_their_parameters():
    from event_utils_b200.contrast_max.warps import pure_rotation_warp, warp_function, xyztheta_warp
    r, x = pure_rotation_warp(), xyztheta_warp()
    assert isinstance(r, warp_function) and isinstance(x, warp_function)
    assert (r.name, r.dims, r.fused_kind) == ("pure_rotation_warp", 3, "rotation")
    assert (x.name, x.dims, x.fused_kind) == ("xyztheta_warp", 4, "xyztheta")
    assert x.center == (120.0, 90.0) and xyztheta_warp(center=(1, 2)).center == (1.0, 2.0)
    assert r.model((1, 2, 3)) == [1.0, 2.0, 3.0]
    assert x.model((1, 2, 3, 4)) == [1.0, 2.0, 3.0, 4.0, 120.0, 90.0]
    xs, ys, ts, ps = _events(0, 10)
    for w, prm in _models():
        xw, yw, jx, jy = w.warp(xs, ys, ts, ps, ts[-1], prm)
        assert jx is None and jy is None and xw.shape == xs.shape and xw.dtype == np.float64
        _, _, jx, jy = w.warp(xs, ys, ts, ps, ts[-1], prm, compute_grad=True)
        assert jx.shape == (w.dims, 10) and jy.shape == (w.dims, 10)


def test_jacobians_match_central_differences():
    xs, ys, ts, ps = _events(1, 500)
    t0 = ts[-1]
    for w, prm in _models():
        _, _, jx, jy = w.warp(xs, ys, ts, ps, t0, prm, compute_grad=True)
        for k in range(w.dims):
            h = 1e-4 * max(1.0, abs(prm[k]))
            up, dn = list(prm), list(prm)
            up[k] += h
            dn[k] -= h
            xu, yu, _, _ = w.warp(xs, ys, ts, ps, t0, up)
            xd, yd, _, _ = w.warp(xs, ys, ts, ps, t0, dn)
            for num, ana in (((xu - xd) / (2 * h), jx[k]), ((yu - yd) / (2 * h), jy[k])):
                scale = max(np.abs(ana).max(), 1e-3)
                assert np.abs(num - ana).max() <= 1e-7 * scale, (w.name, k, np.abs(num - ana).max(), scale)


def test_rotation_preserves_the_radius_and_is_the_identity_at_rest():
    from event_utils_b200.contrast_max.warps import pure_rotation_warp
    w = pure_rotation_warp()
    xs, ys, ts, ps = _events(2)
    cx, cy = 130.0, 85.0
    xw, yw, _, _ = w.warp(xs, ys, ts, ps, ts[-1], (cx, cy, 7.0))
    r0, r1 = np.hypot(xs - cx, ys - cy), np.hypot(xw - cx, yw - cy)
    assert np.abs(r1 - r0).max() <= 1e-9 * r0.max()
    xw, yw, _, _ = w.warp(xs, ys, ts, ps, ts[-1], (cx, cy, 0.0))
    # cx + (x - cx): the identity up to the rounding of the two additions
    assert np.abs(xw - xs).max() <= 2 * np.spacing(256.0) and np.abs(yw - ys).max() <= 2 * np.spacing(256.0)


def test_forward_model_events_warp_back_to_their_rest_positions():
    from event_utils_b200.contrast_max.warps import pure_rotation_warp, xyztheta_warp
    rng = np.random.default_rng(3)
    n = 3000
    x0, y0 = rng.uniform(20, 220, n), rng.uniform(20, 160, n)
    ts = np.sort(rng.uniform(0, 0.05, n))
    dt = ts - ts[-1]
    ps = np.ones(n)
    # rotation about (cx, cy): the event seen at time t is its rest position rotated by omega dt
    cx, cy, om = 130.0, 85.0, 5.0
    a = om * dt
    u, v = x0 - cx, y0 - cy
    xs, ys = cx + np.cos(a) * u - np.sin(a) * v, cy + np.sin(a) * u + np.cos(a) * v
    xw, yw, _, _ = pure_rotation_warp().warp(xs, ys, ts, ps, ts[-1], (cx, cy, om))
    assert np.abs(xw - x0).max() <= 1e-9 and np.abs(yw - y0).max() <= 1e-9
    # xyztheta: solve the first-order model for the position at time t (a 2x2 system per event)
    hx, hy, hz, th = 20.0, -10.0, 4.0, 3.0
    w = xyztheta_warp()
    cx, cy = w.center
    bx, by = (x0 - cx) + dt * hx, (y0 - cy) + dt * hy          # (I - dt A) w = w0 + dt h,  A = [[hz, -th], [th, hz]]
    m00, m01, m10, m11 = 1 - dt * hz, dt * th, -dt * th, 1 - dt * hz
    det = m00 * m11 - m01 * m10
    wu, wv = (m11 * bx - m01 * by) / det, (m00 * by - m10 * bx) / det
    xw, yw, _, _ = w.warp(cx + wu, cy + wv, ts, ps, ts[-1], (hx, hy, hz, th))
    assert np.abs(xw - x0).max() <= 1e-9 and np.abs(yw - y0).max() <= 1e-9


def test_xyztheta_without_expansion_and_rotation_is_linvel_bit_for_bit():
    from event_utils_b200.contrast_max.warps import linvel_warp, xyztheta_warp
    xs, ys, ts, ps = _events(4)
    for hx, hy in ((45.0, -20.0), (0.0, 0.0), (-0.1, 1e-3), (123.456, -987.6)):
        a = xyztheta_warp().warp(xs, ys, ts, ps, ts[-1], (hx, hy, 0.0, 0.0), compute_grad=True)
        b = linvel_warp().warp(xs, ys, ts, ps, ts[-1], (hx, hy), compute_grad=True)
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
        assert np.array_equal(a[2][:2], b[2]) and np.array_equal(a[3][:2], b[3])


def test_small_angle_xyztheta_rotation_agrees_with_pure_rotation_to_second_order():
    from event_utils_b200.contrast_max.warps import pure_rotation_warp, xyztheta_warp
    xs, ys, ts, ps = _events(5)
    w = xyztheta_warp((110.0, 95.0))
    for theta in (0.2, 1.0, 3.0):
        a = np.abs(theta * (ts - ts[-1])).max()
        r = np.hypot(xs - 110.0, ys - 95.0).max()
        xa, ya, _, _ = w.warp(xs, ys, ts, ps, ts[-1], (0.0, 0.0, 0.0, theta))
        xb, yb, _, _ = pure_rotation_warp().warp(xs, ys, ts, ps, ts[-1], (110.0, 95.0, theta))
        err = max(np.abs(xa - xb).max(), np.abs(ya - yb).max())
        assert err <= 0.5 * a * a * r * (1 + 1e-6) + 1e-12, (theta, err, a, r)


@pytest.mark.parametrize("use_polarity", [True, False])
def test_k_channel_oracle_equals_the_linvel_oracle_bit_for_bit(oracle, use_polarity):
    from event_utils_b200.contrast_max.warps import linvel_warp
    rng = np.random.default_rng(6)
    n = 20000
    xs, ys = rng.uniform(-20, 260, n), rng.uniform(-20, 200, n)     # some events leave the bounds mask
    ts, ps = np.sort(rng.uniform(0, 0.1, n)), rng.standard_normal(n)
    for params in ((45.0, -20.0), (-300.0, 150.0), (0.0, 0.0)):
        iwe_o, d_o = oracle.iwe_linvel(params, xs, ys, ts, ps, (180, 240), compute_gradient=True, use_polarity=use_polarity)
        iwe, d, oob = iwe_warp(linvel_warp(), params, xs, ys, ts, ps, (180, 240), compute_gradient=True,
                               use_polarity=use_polarity)
        assert oob == 0 and d.shape == (2, 181, 241)
        assert np.array_equal(iwe, iwe_o) and np.array_equal(d, d_o)
        iwe2, d2, _ = iwe_warp(linvel_warp(), params, xs, ys, ts, ps, (120, 200), use_polarity=use_polarity)
        assert d2 is None and np.array_equal(iwe2, oracle.iwe_linvel(params, xs, ys, ts, ps, (120, 200),
                                                                     use_polarity=use_polarity)[0])
