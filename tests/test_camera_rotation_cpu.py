"""No-GPU checks of the camera-rotation model (camera_rotation_warp): the reference's Jacobian and warp() against central
differences from phi = 0 to 2 rad, warp() against the scipy reference, the identity with pure_rotation_warp, the
second-order agreement with the homography embedding, the f32 coefficients of the kernel, argument validation, the
model code and row plumbing of the batched losses, and the C entries' parameter-count checks, which come before any
CUDA call."""
import numpy as np
import pytest
import torch

import camera_rotation_reference as R

E_ARG = -1
INTR = (199.1, 198.7, 132.1, 110.8)         # fx, fy, cx, cy
AXIS = np.array([0.6, -0.48, 0.64])          # a unit vector on mixed axes
PHIS = [0.0, 1e-6, 1e-4, 1e-2, 0.1, 0.5, 1.0, 2.0]
D = -0.05                                    # every event's d = t - t0 in the Jacobian checks


def _warp_cls():
    from event_utils_b200.contrast_max.warps import camera_rotation_warp
    return camera_rotation_warp


def _events(seed, n, H=180, W=240):
    rng = np.random.default_rng(seed)
    return rng.uniform(2, W - 2, n), rng.uniform(2, H - 2, n)


@pytest.mark.parametrize("phi", PHIS)
def test_reference_jacobian_matches_central_differences(phi):
    x, y = _events(1, 400)
    d = np.full(x.size, D)
    omega = AXIS * phi / abs(D)
    prm = np.concatenate((omega, INTR[:2]))
    J = R.jacobian(x, y, d, omega, INTR)
    for k in range(5):
        h = 1e-5 if k < 3 else 1e-4
        hi, lo = prm.copy(), prm.copy()
        hi[k] += h
        lo[k] -= h
        wp = R.warp(x, y, d, hi[:3], (hi[3], hi[4]) + INTR[2:])
        wm = R.warp(x, y, d, lo[:3], (lo[3], lo[4]) + INTR[2:])
        front = np.isfinite(wp[0]) & np.isfinite(wm[0])      # at 2 rad some events rotate behind the camera
        assert front.mean() > 0.5
        for i in range(2):
            num = (wp[i] - wm[i]) / (2 * h)
            np.testing.assert_allclose(J[i, k][front], num[front], rtol=1e-6, atol=1e-6 * np.abs(J[i, :3]).max() + 1e-9,
                                       err_msg="phi %g row %d column %d" % (phi, i, k))


@pytest.mark.parametrize("phi", PHIS)
def test_warp_matches_the_reference(phi):
    x, y = _events(2, 500)
    t = np.linspace(0.0, 0.05, x.size)
    omega = AXIS * phi / 0.05
    w = _warp_cls()(INTR)
    xw, yw, jx, jy = w.warp(x, y, t, np.ones_like(x), 0.05, omega, compute_grad=True)
    rx, ry = R.warp(x, y, t - 0.05, omega, INTR)
    # behind the camera the reference gives NaN and warp() its formula, which the reference API's bounds mask judges
    front = np.isfinite(rx)
    assert front.mean() > 0.5 and np.isfinite(xw).all()
    np.testing.assert_allclose(xw[front], rx[front], rtol=0, atol=1e-9)
    np.testing.assert_allclose(yw[front], ry[front], rtol=0, atol=1e-9)
    J = R.jacobian(x, y, t - 0.05, omega, INTR)
    assert jx.shape == jy.shape == (3, x.size)
    scale = np.abs(J[:, :3][..., front]).max()
    np.testing.assert_allclose(jx[:, front], J[0, :3][:, front], rtol=1e-9, atol=1e-12 * scale)
    np.testing.assert_allclose(jy[:, front], J[1, :3][:, front], rtol=1e-9, atol=1e-12 * scale)
    xn, yn, _, _ = w.warp(x, y, t, None, 0.05, omega)
    assert np.array_equal(xn, xw) and np.array_equal(yn, yw)


def test_identity_with_pure_rotation_warp():
    from event_utils_b200.contrast_max.warps import pure_rotation_warp
    x, y = _events(3, 1000)
    t = np.sort(np.random.default_rng(3).uniform(0, 0.1, x.size))
    f, cx, cy, wz = 210.0, 130.0, 95.0, 7.0
    cam = _warp_cls()((f, f, cx, cy)).warp(x, y, t, None, t[-1], (0.0, 0.0, wz), compute_grad=True)
    rot = pure_rotation_warp().warp(x, y, t, None, t[-1], (cx, cy, -wz), compute_grad=True)
    np.testing.assert_allclose(cam[0], rot[0], rtol=0, atol=1e-9)
    np.testing.assert_allclose(cam[1], rot[1], rtol=0, atol=1e-9)
    # d/d wz = -d/d omega
    np.testing.assert_allclose(cam[2][2], -rot[2][2], rtol=1e-9, atol=1e-9)
    np.testing.assert_allclose(cam[3][2], -rot[3][2], rtol=1e-9, atol=1e-9)


def test_homography_embedding_agrees_to_second_order():
    from event_utils_b200.contrast_max.warps import homography_warp
    x, y = _events(4, 2000)
    omega = np.array([3.0, -4.0, 2.5])
    hom = homography_warp(center=INTR[2:])
    h = R.embedding(omega, INTR)
    errs = []
    for d in (-0.02, -0.01, -0.005):
        t = np.full(x.size, d)
        xc, yc = R.warp(x, y, t, omega, INTR)
        xh, yh, _, _ = hom.warp(x, y, t, None, 0.0, h)
        errs.append(np.hypot(xc - xh, yc - yh).max())
    ratios = [errs[0] / errs[1], errs[1] / errs[2]]
    assert all(3.5 < r < 4.5 for r in ratios), (errs, ratios)
    # the projection of a homography onto the rotation subspace inverts the embedding
    E = R.embedding_matrix(INTR)
    np.testing.assert_allclose(np.linalg.lstsq(E, h, rcond=None)[0], omega, rtol=1e-12)
    # and the embedding is the first-order term: its Jacobian in w at w = 0 is the camera's
    t = np.full(x.size, -0.01)
    J = R.jacobian(x, y, t, np.zeros(3), INTR)
    _, _, hx, hy = hom.warp(x, y, t, None, 0.0, np.zeros(8), compute_grad=True)
    np.testing.assert_allclose(J[0, :3], (hx.T @ E).T, rtol=1e-9, atol=1e-12)
    np.testing.assert_allclose(J[1, :3], (hy.T @ E).T, rtol=1e-9, atol=1e-12)


def _coefficients_f32(phi):
    """the kernel's f32 A, B and C of camera rotation (model_taps): sine and cosine of phi / 2, the series of C below
    kCamSeriesPhi = 0.5"""
    f32 = np.float32
    phi = np.asarray(phi, f32)
    p2 = (phi * phi).astype(f32)
    half = (f32(0.5) * phi).astype(f32)
    sh, ch = np.sin(half).astype(f32), np.cos(half).astype(f32)
    with np.errstate(all="ignore"):
        r = np.where(phi > 0, sh / half, f32(1)).astype(f32)
        series = (f32(1 / 6) - p2 * (f32(1 / 120) - p2 * (f32(1 / 5040) - p2 * f32(1 / 362880)))).astype(f32)
        direct = ((phi - f32(2) * (sh * ch)) / (p2 * phi)).astype(f32)
    return (r * ch).astype(f32), (f32(0.5) * (r * r)).astype(f32), np.where(phi < f32(0.5), series, direct), direct


def test_f32_coefficients_hold_across_the_series_threshold():
    """A = sin phi / phi, B = (1 - cos phi) / phi^2 and C = (phi - sin phi) / phi^3 in the kernel's f32 forms stay
    within 2e-6 relative of f64 from phi = 0 to 3 rad; the direct C would not below the threshold"""
    phi = np.concatenate(([0.0], np.logspace(-8, np.log10(3.0), 400), [0.4999, 0.5, 0.5001]))
    phi = phi.astype(np.float32).astype(np.float64)        # the f32 angle is the truth's argument
    A, B, C, direct = _coefficients_f32(phi)
    p = np.where(phi > 0, phi, 1.0)
    a64 = np.where(phi > 0, np.sin(p) / p, 1.0)
    b64 = np.where(phi > 1e-4, 2 * np.sin(p / 2) ** 2 / p ** 2, 0.5 - phi ** 2 / 24)
    c64 = np.where(phi > 1e-2, (p - np.sin(p)) / p ** 3, 1 / 6 - phi ** 2 / 120 + phi ** 4 / 5040)
    for got, want, what in ((A, a64, "A"), (B, b64, "B"), (C, c64, "C")):
        rel = np.abs(got.astype(np.float64) - want) / np.abs(want)
        assert rel.max() <= 2e-6, (what, phi[rel.argmax()], rel.max())
    small = (phi > 0) & (phi < 1e-2)
    assert (np.abs(direct[small] - c64[small]) / c64[small]).max() > 1e-2    # the cancellation the series avoids


def test_arguments_are_validated():
    cls = _warp_cls()
    K = np.array([[199.1, 0.0, 132.1], [0.0, 198.7, 110.8], [0.0, 0.0, 1.0]])
    for w in (cls(K), cls(INTR), cls(list(INTR)), cls(torch.tensor(K))):
        assert w.dims == 3 and w.fused_kind is None and w.name == "camera_rotation_warp"
        assert w.center == (132.1, 110.8) and w.focal == (199.1, 198.7)
        assert w.model((1, 2, 3)) == [1.0, 2.0, 3.0, 199.1, 198.7, 132.1, 110.8]
    bad = K.copy()
    bad[0, 1] = 0.5
    with pytest.raises(ValueError, match="no skew"):
        cls(bad)
    bad = K.copy()
    bad[2, 2] = 2.0
    with pytest.raises(ValueError, match="no skew"):
        cls(bad)
    for intr in ((0.0, 200.0, 1.0, 1.0), (200.0, -1.0, 1.0, 1.0), (np.nan, 200.0, 1.0, 1.0), (200.0, np.inf, 1.0, 1.0),
                 (200.0, 200.0, np.nan, 1.0)):
        with pytest.raises(ValueError, match="finite and positive"):
            cls(intr)
    for shape in ((3,), (2, 2), (3, 4)):
        with pytest.raises(ValueError, match="3x3 matrix or"):
            cls(np.ones(shape))


def test_model_code_and_the_rows_of_the_entries():
    from event_utils_b200 import _lib
    from event_utils_b200.contrast_max import _batched as B
    w = _warp_cls()(INTR)
    code = _lib.WARP_CAMERA_ROTATION
    assert code == 6 and B._warp_code(w, "f") == code
    assert B._model(code, w, "variance", 1.0, None, 180, 240)[1] == (132.1, 110.8, 199.1, 198.7)
    assert B._ts_model(code, w, 1.0, 180, 240)[1] == (132.1, 110.8, 199.1, 198.7)
    assert B._model_layout((code, B._centre(code, w), 180, 240), 3)[:2] == ((code,), (5, 132.1, 110.8))
    prm = torch.tensor([[1.0, 2.0, 3.0], [4.0, 5.0, 6.0]], dtype=torch.float32, requires_grad=True)
    rows = B._rows(prm, B._centre(code, w))
    assert rows.dtype == torch.float64 and rows.tolist() == [[1.0, 2.0, 3.0, 199.1, 198.7], [4.0, 5.0, 6.0, 199.1, 198.7]]
    rows.backward(torch.arange(10.0, dtype=torch.float64).reshape(2, 5))
    assert prm.grad.tolist() == [[0.0, 1.0, 2.0], [5.0, 6.0, 7.0]]      # the focal-length columns drop out
    cand = torch.zeros((2, 4, 2, 3), dtype=torch.float64)
    assert B._rows(cand, B._centre(code, w)).shape == (2, 4, 2, 5)
    # every other model's parameters pass through untouched
    from event_utils_b200.contrast_max.warps import xyztheta_warp
    p4 = torch.zeros((2, 4))
    assert B._rows(p4, B._centre(_lib.WARP_XYZTHETA, xyztheta_warp())) is p4

    class sub(type(w)):
        pass
    with pytest.raises(ValueError, match="supports the models") as e:
        B._warp_code(sub(INTR), "f")
    assert "linvel_warp, pure_rotation_warp and xyztheta_warp" in str(e.value) and "camera_rotation_warp" in str(e.value)


@pytest.mark.parametrize("entry", ["contrast", "contrast_grad", "contrast_cand", "ts", "ts_grad", "ts_cand", "seg", "seg_grad",
                                   "seg_cand", "assign"])
def test_entries_check_the_parameter_count_before_any_cuda_call(entry):
    from test_planar_motion_cpu import _entries
    call = _entries()[entry]
    for K in (3, 4, 7):
        rc, msg = call(6, K)
        assert rc == E_ARG and b"has 5 parameters" in msg, msg
    rc, msg = call(7, 5)
    assert rc == E_ARG and b"unknown warp" in msg, msg


def test_single_window_entries_reject_the_camera_rotation():
    import ctypes
    from event_utils_b200 import _lib
    L = _lib.load()
    F = ctypes.c_void_p(1 << 20)
    model = (ctypes.c_double * 7)(1, 2, 3, 200, 200, 120, 90)
    rc = L.evk_cmax_warp_objective_f32(F, F, F, F, 100, 1.0, 6, model, 180, 240, 180, 240, 1.0, 0, 0, 0.0, F, None, F,
                                       1 << 30, None)
    assert rc == E_ARG and b"unknown warp 6" in L.evk_last_error()
    rc = L.evk_cmax_warp_objective_f64(F, F, F, F, 100, 1.0, 6, model, 0.0, 180, 240, 180, 240, 1.0, 0, 0, 0.0, F, None, F,
                                       1 << 30, None)
    assert rc == E_ARG and b"unknown warp 6" in L.evk_last_error()


def test_torch_functions_check_the_parameter_shape():
    from event_utils_b200.contrast_max import motion_contrast_objective_torch, motion_timestamp_objective_torch
    x = torch.zeros(10)
    for fn in (motion_contrast_objective_torch, motion_timestamp_objective_torch):
        for bad in (torch.zeros(5), torch.zeros(2, 5)):
            with pytest.raises(ValueError, match=r"\(B,3\)"):
                fn(x, x, x, x, bad, _warp_cls()(INTR))


def test_reference_gradient_matches_central_differences():
    """autograd through the reference loss (positions from scipy, derivatives from the analytic Jacobian) against
    central differences of the loss, all five columns"""
    rng = np.random.default_rng(5)
    n = 3000
    x = rng.uniform(20, 220, n).astype(np.float32)
    y = rng.uniform(20, 160, n).astype(np.float32)
    d = (-np.sort(rng.integers(0, 410, n))[::-1] / 4096.0).astype(np.float32)
    p = (rng.integers(0, 2, n) * 2 - 1).astype(np.float32)
    prm = torch.tensor([[2.0, -3.0, 4.0, INTR[0], INTR[1]]], dtype=torch.float64, requires_grad=True)
    f, _ = R.contrast(x, y, d, p, [0, n], prm, 1.0, "variance", INTR[2:])
    f.sum().backward()
    g = prm.grad[0].numpy()
    scale = np.abs(g).max()
    for k in range(5):
        h = 1e-7 if k < 3 else 1e-6     # small enough that no event crosses a pixel edge
        fs = []
        for sgn in (1, -1):
            q = prm.detach().clone()
            q[0, k] += sgn * h
            fs.append(float(R.contrast(x, y, d, p, [0, n], q, 1.0, "variance", INTR[2:])[0][0]))
        num = (fs[0] - fs[1]) / (2 * h)
        assert abs(num - g[k]) <= 2e-3 * scale, (k, num, g[k], scale)


def test_scene_maps_back_onto_its_points():
    rng = np.random.default_rng(6)
    omega = np.array([2.0, -5.0, 3.0])
    x, y, t, p = R.rotation_scene(omega, INTR, rng, n_pts=50, per_pt=40, t_end=0.05)
    assert x.size > 1500 and ((x > 0) & (x < 239) & (y > 0) & (y < 179)).all()
    xw, yw = R.warp(x, y, t - 0.05, omega, INTR)
    pts = np.unique(np.round(np.stack((xw, yw), 1), 6), axis=0)
    assert pts.shape[0] <= 50
