"""No-GPU checks of the camera-motion model (camera_motion_warp): the reference's Jacobian against central differences
from phi = 0 to 2 rad and over a range of rho d |v|, warp() against the scipy reference, the identities with
camera_rotation_warp at v = 0 and rho = 0, the exact projective translation at w = 0, the scene generator, argument
validation (inv_depth missing, misaligned or given to another model, segmentation rejecting the model), the model code
and rows of the batched losses, and the C entries' warp and parameter-count checks, which come before any CUDA call."""
import ctypes

import numpy as np
import pytest
import torch

import camera_motion_reference as R
import camera_rotation_reference as CR

E_ARG = -1
INTR = (199.1, 198.7, 132.1, 110.8)         # fx, fy, cx, cy
AXIS = np.array([0.6, -0.48, 0.64])          # a unit vector on mixed axes
VDIR = np.array([0.36, 0.48, -0.8])          # a unit vector on mixed axes
PHIS = [0.0, 1e-4, 1e-2, 0.1, 0.5, 1.0, 2.0]
SHIFTS = [0.0, 1e-3, 0.05, 0.3]              # rho d |v|: the translation against the bearing's unit depth
D = -0.05                                    # every event's d = t - t0 in the Jacobian checks
FAKE = ctypes.c_void_p(1 << 20)              # aligned, never dereferenced


def _warp_cls():
    from event_utils_b200.contrast_max.warps import camera_motion_warp
    return camera_motion_warp


def _events(seed, n, H=180, W=240):
    rng = np.random.default_rng(seed)
    return rng.uniform(2, W - 2, n), rng.uniform(2, H - 2, n), rng.uniform(0.125, 1.0, n)


@pytest.mark.parametrize("shift", SHIFTS)
@pytest.mark.parametrize("phi", PHIS)
def test_reference_jacobian_matches_central_differences(phi, shift):
    x, y, rho = _events(1, 400)
    d = np.full(x.size, D)
    omega = AXIS * phi / abs(D)
    v = VDIR * shift / abs(D)                # rho d |v| = shift at rho = 1
    prm = np.concatenate((omega, v, INTR[:2]))
    J = R.jacobian(x, y, d, rho, omega, v, INTR)

    def at(q):
        return R.warp(x, y, d, rho, q[:3], q[3:6], (q[6], q[7]) + INTR[2:])
    for k in range(8):
        h = 1e-5 if k < 6 else 1e-4
        hi, lo = prm.copy(), prm.copy()
        hi[k] += h
        lo[k] -= h
        wp, wm = at(hi), at(lo)
        front = np.isfinite(wp[0]) & np.isfinite(wm[0])      # at 2 rad some events rotate behind the camera
        assert front.mean() > 0.5
        for i in range(2):
            num = (wp[i] - wm[i]) / (2 * h)
            np.testing.assert_allclose(J[i, k][front], num[front], rtol=1e-5, atol=1e-6 * np.abs(J[i, :6]).max() + 1e-9,
                                       err_msg="phi %g shift %g row %d column %d" % (phi, shift, i, k))


@pytest.mark.parametrize("shift", [0.0, 0.05, 0.3])
@pytest.mark.parametrize("phi", [0.0, 1e-4, 0.1, 1.0, 2.0])
def test_warp_matches_the_reference(phi, shift):
    x, y, rho = _events(2, 500)
    t = np.linspace(0.0, 0.05, x.size)
    omega, v = AXIS * phi / 0.05, VDIR * shift / 0.05
    w = _warp_cls()(INTR)
    xw, yw, jx, jy = w.warp(x, y, t, np.ones_like(x), 0.05, np.concatenate((omega, v)), compute_grad=True, inv_depth=rho)
    rx, ry = R.warp(x, y, t - 0.05, rho, omega, v, INTR)
    front = np.isfinite(rx)
    assert front.mean() > 0.5
    np.testing.assert_allclose(xw[front], rx[front], rtol=0, atol=1e-9)
    np.testing.assert_allclose(yw[front], ry[front], rtol=0, atol=1e-9)
    J = R.jacobian(x, y, t - 0.05, rho, omega, v, INTR)
    assert jx.shape == jy.shape == (6, x.size)
    scale = np.abs(J[:, :6][..., front]).max()
    np.testing.assert_allclose(jx[:, front], J[0, :6][:, front], rtol=1e-9, atol=1e-12 * scale)
    np.testing.assert_allclose(jy[:, front], J[1, :6][:, front], rtol=1e-9, atol=1e-12 * scale)
    xn, yn, _, _ = w.warp(x, y, t, None, 0.05, np.concatenate((omega, v)), inv_depth=rho)
    assert np.array_equal(xn, xw) and np.array_equal(yn, yw)


def test_identities_with_camera_rotation_warp():
    """at v = 0 or rho = 0 the translation adds an exact zero: warp() equals camera_rotation_warp's bit for bit, and its
    w rows are the rotation's to rounding (Qz = Uz / Pz need not be exactly 1)"""
    from event_utils_b200.contrast_max.warps import camera_rotation_warp
    x, y, rho = _events(3, 1000)
    t = np.sort(np.random.default_rng(3).uniform(0, 0.1, x.size))
    om = np.array([3.0, -4.0, 6.0])
    rot = camera_rotation_warp(INTR).warp(x, y, t, None, t[-1], om, compute_grad=True)
    cam = _warp_cls()(INTR)
    for v, r in ((np.zeros(3), rho), (np.array([1.5, -0.5, 2.0]), np.zeros_like(rho))):
        got = cam.warp(x, y, t, None, t[-1], np.concatenate((om, v)), compute_grad=True, inv_depth=r)
        assert np.array_equal(got[0], rot[0]) and np.array_equal(got[1], rot[1])
        np.testing.assert_allclose(got[2][:3], rot[2], rtol=1e-12, atol=1e-12 * np.abs(rot[2]).max())
        np.testing.assert_allclose(got[3][:3], rot[3], rtol=1e-12, atol=1e-12 * np.abs(rot[3]).max())
        # dx'/dv = (rho d) fx iz (1, 0, -X): zero with rho = 0, not with v = 0
        assert (np.abs(got[2][3:]).max() == 0.0) == (not r.any())
    # the reference likewise
    d = t - t[-1]
    for v, r in ((np.zeros(3), rho), (np.array([1.5, -0.5, 2.0]), np.zeros_like(rho))):
        got = R.warp(x, y, d, r, om, v, INTR)
        want = CR.warp(x, y, d, om, INTR)
        np.testing.assert_allclose(got[0], want[0], rtol=0, atol=1e-9)
        np.testing.assert_allclose(got[1], want[1], rtol=0, atol=1e-9)
        J, Jr = R.jacobian(x, y, d, r, om, v, INTR), CR.jacobian(x, y, d, om, INTR)
        np.testing.assert_allclose(J[:, :3], Jr[:, :3], rtol=1e-9, atol=1e-9 * np.abs(Jr).max())
        np.testing.assert_allclose(J[:, 6:], Jr[:, 3:], rtol=1e-9, atol=1e-9 * np.abs(Jr).max())


def test_zero_rotation_is_the_projective_translation():
    """at w = 0 the event's 3-D point (b / rho) moved by d v projects to the warped position"""
    x, y, rho = _events(4, 1000)
    d = -np.random.default_rng(4).uniform(0, 0.05, x.size)
    v = np.array([2.0, -1.0, 3.0])
    fx, fy, cx, cy = INTR
    X = np.stack(((x - cx) / fx / rho, (y - cy) / fy / rho, 1.0 / rho), -1) + d[:, None] * v
    xw, yw = R.warp(x, y, d, rho, np.zeros(3), v, INTR)
    np.testing.assert_allclose(xw, cx + fx * X[:, 0] / X[:, 2], rtol=1e-12)
    np.testing.assert_allclose(yw, cy + fy * X[:, 1] / X[:, 2], rtol=1e-12)
    xm, ym, _, _ = _warp_cls()(INTR).warp(x, y, d, None, 0.0, np.concatenate((np.zeros(3), v)), inv_depth=rho)
    np.testing.assert_allclose(xm, xw, rtol=1e-12)
    np.testing.assert_allclose(ym, yw, rtol=1e-12)


def test_keep_rules_of_the_reference():
    x, y, rho = _events(5, 6)
    rho[1], rho[2], rho[3] = -0.5, np.nan, np.inf
    xw, _ = R.warp(x, y, np.full(6, -0.01), rho, np.zeros(3), np.zeros(3), INTR)
    assert np.isnan(xw[1:4]).all() and np.isfinite(xw[[0, 4, 5]]).all()
    # behind the camera: a point 0.1 m away and a camera that moved 0.2 m backwards since
    xb, _ = R.warp(x[:1], y[:1], np.array([-0.1]), np.array([10.0]), np.zeros(3), np.array([0.0, 0.0, 2.0]), INTR)
    assert np.isnan(xb).all()


def test_scene_maps_back_onto_its_points_at_several_depths():
    rng = np.random.default_rng(6)
    om, v = np.array([1.0, -2.0, 1.5]), np.array([1.5, -0.5, 2.0])
    x, y, t, p, rho = R.motion_scene(om, v, INTR, rng, n_pts=50, per_pt=40, t_end=0.05)
    assert x.size > 1500 and ((x > 0) & (x < 239) & (y > 0) & (y < 179)).all()
    assert 1 / 8.5 < rho.min() and rho.max() < 1 / 0.8 and rho.max() / rho.min() > 3
    xw, yw = R.warp(x, y, t - 0.05, rho, om, v, INTR)
    pts = np.unique(np.round(np.stack((xw, yw), 1), 6), axis=0)
    assert pts.shape[0] <= 50
    # the rotation alone cannot: the translation's parallax spreads every point
    xr, yr = CR.warp(x, y, t - 0.05, om, INTR)
    assert np.unique(np.round(np.stack((xr, yr), 1), 6), axis=0).shape[0] > 1000


def test_warp_class_and_its_arguments():
    cls = _warp_cls()
    K = np.array([[199.1, 0.0, 132.1], [0.0, 198.7, 110.8], [0.0, 0.0, 1.0]])
    for w in (cls(K), cls(INTR), cls(torch.tensor(K))):
        assert w.dims == 6 and w.fused_kind is None and w.name == "camera_motion_warp"
        assert w.center == (132.1, 110.8) and w.focal == (199.1, 198.7)
        assert w.model(range(6)) == [0.0, 1.0, 2.0, 3.0, 4.0, 5.0, 199.1, 198.7, 132.1, 110.8]
    with pytest.raises(ValueError, match="no skew"):
        cls(K + np.eye(3) * [0, 0, 1])
    with pytest.raises(ValueError, match="inverse depth"):
        cls(INTR).warp(np.ones(3), np.ones(3), np.ones(3), None, 1.0, np.zeros(6))
    # so the reference-API objectives, which call warp() without depth, reject the model
    from event_utils_b200.contrast_max import variance_objective
    with pytest.raises(ValueError, match="inverse depth"):
        variance_objective().evaluate_function(np.zeros(6), np.ones(3), np.ones(3), np.arange(3.0), np.ones(3), cls(INTR),
                                               (180, 240), 1.0)


def test_model_code_and_the_rows_of_the_entries():
    from event_utils_b200 import _lib
    from event_utils_b200.contrast_max import _batched as B
    w = _warp_cls()(INTR)
    code = _lib.WARP_CAMERA_MOTION
    assert code == 7 and B._warp_code(w, "f") == code
    assert B._model(code, w, "variance", 1.0, None, 180, 240)[1] == (132.1, 110.8, 199.1, 198.7)
    assert B._ts_model(code, w, 1.0, 180, 240)[1] == (132.1, 110.8, 199.1, 198.7)
    assert B._model_layout((code, B._centre(code, w), 180, 240), 6)[:2] == ((code,), (8, 132.1, 110.8))
    prm = torch.arange(12.0).reshape(2, 6).requires_grad_(True)
    rows = B._rows(prm, B._centre(code, w))
    assert rows.dtype == torch.float64 and rows.shape == (2, 8) and rows[:, 6:].tolist() == [[199.1, 198.7]] * 2
    rows.backward(torch.arange(16.0, dtype=torch.float64).reshape(2, 8))
    assert prm.grad.tolist() == [[0.0, 1.0, 2.0, 3.0, 4.0, 5.0], [8.0, 9.0, 10.0, 11.0, 12.0, 13.0]]
    ev = tuple(torch.zeros(3) for _ in range(4))
    rho = torch.ones(3)
    assert B._depth_entry("evk_cmax_motion_objective", ev, None) == ("evk_cmax_motion_objective", ev)
    stem, got = B._depth_entry("evk_cmax_motion_objective", ev, rho)
    assert stem == "evk_cmax_motion_depth_objective" and got[:4] == ev and got[4] is rho
    assert B._depth_entry("evk_motion_timestamp_candidates", ev, rho)[0] == "evk_motion_timestamp_depth_candidates"

    class sub(type(w)):
        pass
    with pytest.raises(ValueError, match="supports the models") as e:
        B._warp_code(sub(INTR), "f")
    assert "camera_motion_warp" in str(e.value)


def _torch_calls():
    """every torch function that takes inv_depth, as f(warp, inv_depth) on 10 events and one window"""
    from event_utils_b200 import contrast_max as C
    x = torch.zeros(10)
    ts = torch.linspace(0, 0.05, 10)
    p6, c6 = torch.zeros(1, 6), torch.zeros(1, 2, 6)
    return {
        "objective": lambda w, r: C.motion_contrast_objective_torch(x, x, ts, x, p6[:, :w.dims], w, inv_depth=r),
        "candidates": lambda w, r: C.motion_contrast_candidates_torch(x, x, ts, x, c6[..., :w.dims], w, inv_depth=r),
        "fit": lambda w, r: C.motion_contrast_fit_torch(x, x, ts, x, w, x0=np.zeros(w.dims), inv_depth=r),
        "ts_objective": lambda w, r: C.motion_timestamp_objective_torch(x, x, ts, x, p6[:, :w.dims], w, inv_depth=r),
        "ts_candidates": lambda w, r: C.motion_timestamp_candidates_torch(x, x, ts, x, c6[..., :w.dims], w, inv_depth=r),
        "ts_fit": lambda w, r: C.motion_timestamp_fit_torch(x, x, ts, x, w, x0=np.zeros(w.dims), inv_depth=r),
    }


@pytest.mark.parametrize("fn", ["objective", "candidates", "fit", "ts_objective", "ts_candidates", "ts_fit"])
def test_inv_depth_is_checked_before_any_cuda_call(fn):
    from event_utils_b200.contrast_max.warps import camera_rotation_warp, xyztheta_warp
    call = _torch_calls()[fn]
    w = _warp_cls()(INTR)
    with pytest.raises(ValueError, match="needs inv_depth"):
        call(w, None)
    for bad in (torch.ones(9), torch.ones(11), torch.ones(10, 1), np.ones(2)):
        with pytest.raises(ValueError, match=r"inv_depth must have shape \(10,\)"):
            call(w, bad)
    with pytest.raises(ValueError, match="floating-point"):
        call(w, torch.ones(10, dtype=torch.int64))
    with pytest.raises(ValueError, match="must not require grad"):
        call(w, torch.ones(10, requires_grad=True))
    for other in (camera_rotation_warp(INTR), xyztheta_warp()):
        with pytest.raises(ValueError, match="the other models take none"):
            call(other, torch.ones(10))


def test_segmentation_rejects_the_model():
    from event_utils_b200 import contrast_max as C
    x = torch.zeros(10)
    w = _warp_cls()(INTR)
    calls = (lambda: C.motion_segmentation_objective_torch(x, x, x, x, torch.ones(10, 2), torch.zeros(1, 2, 6), w),
             lambda: C.motion_segmentation_candidates_torch(x, x, x, x, torch.zeros(1, 2, 1, 6), torch.ones(10, 2), w),
             lambda: C.motion_segmentation_assign_torch(x, x, x, x, torch.zeros(1, 2, 6), w, torch.ones(10, 2)),
             lambda: C.motion_segmentation_fit_torch(x, x, x, x, w, x0=np.zeros((2, 6))))
    for call in calls:
        with pytest.raises(ValueError, match="does not take camera_motion_warp"):
            call()


def _depth_entries():
    """every depth entry as f(warp, K) -> (rc, message), all other arguments valid"""
    from event_utils_b200 import _lib
    L = _lib.load()
    F, B, N, H, W, S, J, WS = FAKE, 2, 100, 60, 80, 1.0, 4, 1 << 40
    calls = {
        "contrast": lambda w, K: L.evk_cmax_motion_depth_objective_f32(F, F, F, F, F, F, B, N, w, F, K, 40.0, 30.0, H, W, S, 0,
                                                                       0.0, F, F, F, WS, None),
        "contrast_grad": lambda w, K: L.evk_cmax_motion_depth_objective_grad_f32(F, F, F, F, F, F, B, N, w, F, K, 40.0, 30.0, H,
                                                                                 W, S, 0, 0.0, F, F, F, F, WS, None),
        "contrast_cand": lambda w, K: L.evk_cmax_motion_depth_candidates_f32(F, F, F, F, F, F, B, N, w, F, J, K, 40.0, 30.0, H, W,
                                                                             S, 0, 0.0, F, F, WS, None),
        "ts": lambda w, K: L.evk_motion_timestamp_depth_objective_f32(F, F, F, F, F, F, F, B, N, w, F, K, 40.0, 30.0, H, W, S, F,
                                                                      F, F, F, WS, None),
        "ts_grad": lambda w, K: L.evk_motion_timestamp_depth_objective_grad_f32(F, F, F, F, F, F, F, B, N, w, F, K, 40.0, 30.0,
                                                                                H, W, S, F, F, F, F, F, WS, None),
        "ts_cand": lambda w, K: L.evk_motion_timestamp_depth_candidates_f32(F, F, F, F, F, F, F, B, N, w, F, J, K, 40.0, 30.0, H,
                                                                            W, S, F, F, WS, None),
    }
    return {k: (lambda c: lambda w, K: (c(w, K), L.evk_last_error()))(c) for k, c in calls.items()}


DEPTH_ENTRIES = ["contrast", "contrast_grad", "contrast_cand", "ts", "ts_grad", "ts_cand"]


@pytest.mark.parametrize("entry", DEPTH_ENTRIES)
def test_depth_entries_check_the_warp_and_the_parameter_count_before_any_cuda_call(entry):
    call = _depth_entries()[entry]
    for K in (5, 6, 7, 9):
        rc, msg = call(7, K)
        assert rc == E_ARG and b"has 8 parameters" in msg, msg
    for warp, K in ((1, 3), (2, 4), (3, 2), (4, 6), (5, 8), (6, 5), (8, 8), (0, 8)):
        rc, msg = call(warp, K)
        assert rc == E_ARG and b"takes no inverse depth" in msg, msg


@pytest.mark.parametrize("entry", DEPTH_ENTRIES)
def test_depth_entries_need_the_depth_array(entry):
    """a null inv_depth with events is a bad argument, the twins' first check after the blur sigma"""
    from event_utils_b200 import _lib
    L = _lib.load()
    F, B, N, H, W, S, J, WS = FAKE, 2, 100, 60, 80, 1.0, 4, 1 << 40
    calls = {
        "contrast": lambda: L.evk_cmax_motion_depth_objective_f32(F, F, F, F, None, F, B, N, 7, F, 8, 40.0, 30.0, H, W, S, 0,
                                                                  0.0, F, F, F, WS, None),
        "contrast_grad": lambda: L.evk_cmax_motion_depth_objective_grad_f32(F, F, F, F, None, F, B, N, 7, F, 8, 40.0, 30.0, H, W,
                                                                            S, 0, 0.0, F, F, F, F, WS, None),
        "contrast_cand": lambda: L.evk_cmax_motion_depth_candidates_f32(F, F, F, F, None, F, B, N, 7, F, J, 8, 40.0, 30.0, H, W,
                                                                        S, 0, 0.0, F, F, WS, None),
        "ts": lambda: L.evk_motion_timestamp_depth_objective_f32(F, F, F, F, F, None, F, B, N, 7, F, 8, 40.0, 30.0, H, W, S, F,
                                                                 F, F, F, WS, None),
        "ts_grad": lambda: L.evk_motion_timestamp_depth_objective_grad_f32(F, F, F, F, F, None, F, B, N, 7, F, 8, 40.0, 30.0, H,
                                                                           W, S, F, F, F, F, F, WS, None),
        "ts_cand": lambda: L.evk_motion_timestamp_depth_candidates_f32(F, F, F, F, F, None, F, B, N, 7, F, J, 8, 40.0, 30.0, H,
                                                                       W, S, F, F, WS, None),
    }
    assert calls[entry]() == E_ARG and b"bad arguments" in L.evk_last_error()


@pytest.mark.parametrize("entry", ["contrast", "contrast_grad", "contrast_cand", "ts", "ts_grad", "ts_cand", "seg", "seg_grad",
                                   "seg_cand", "assign"])
def test_the_other_entries_reject_the_camera_motion(entry):
    from test_planar_motion_cpu import _entries
    call = _entries()[entry]
    for K in (6, 8):
        rc, msg = call(7, K)
        assert rc == E_ARG and b"unknown warp 7" in msg, msg


def test_workspace_queries_are_the_twins():
    from event_utils_b200 import _lib
    L = _lib.load()
    for B, H, W in ((1, 60, 80), (7, 180, 240), (0, 2, 2), (-1, 60, 80), (3, 1, 80)):
        assert L.evk_cmax_motion_depth_objective_workspace_bytes(B, H, W) == L.evk_cmax_motion_objective_workspace_bytes(B, H, W)
        assert (L.evk_motion_timestamp_depth_objective_workspace_bytes(B, H, W) ==
                L.evk_motion_timestamp_objective_workspace_bytes(B, H, W))
        for J in (1, 8, 32, 33):
            assert (L.evk_cmax_motion_depth_candidates_workspace_bytes(B, J, H, W) ==
                    L.evk_cmax_motion_candidates_workspace_bytes(B, J, H, W))
            assert (L.evk_motion_timestamp_depth_candidates_workspace_bytes(B, J, H, W) ==
                    L.evk_motion_timestamp_candidates_workspace_bytes(B, J, H, W))
    assert L.evk_cmax_motion_depth_objective_workspace_bytes(2, 60, 80) > 0


def test_reference_gradient_matches_central_differences():
    """autograd through the reference loss (positions from scipy, derivatives from the analytic Jacobian) against
    central differences of the loss, all eight columns"""
    rng = np.random.default_rng(7)
    n = 3000
    x = rng.uniform(20, 220, n).astype(np.float32)
    y = rng.uniform(20, 160, n).astype(np.float32)
    d = (-np.sort(rng.integers(0, 410, n))[::-1] / 4096.0).astype(np.float32)
    p = (rng.integers(0, 2, n) * 2 - 1).astype(np.float32)
    rho = rng.uniform(0.125, 1.0, n).astype(np.float32)
    prm = torch.tensor([[2.0, -3.0, 4.0, 1.5, -1.0, 2.0, INTR[0], INTR[1]]], dtype=torch.float64, requires_grad=True)
    f, _ = R.contrast(x, y, d, p, rho, [0, n], prm, 1.0, "variance", INTR[2:])
    f.sum().backward()
    g = prm.grad[0].numpy()
    for k in range(8):
        h = 1e-7 if k < 6 else 1e-6     # small enough that no event crosses a pixel edge
        fs = []
        for sgn in (1, -1):
            q = prm.detach().clone()
            q[0, k] += sgn * h
            fs.append(float(R.contrast(x, y, d, p, rho, [0, n], q, 1.0, "variance", INTR[2:])[0][0]))
        num = (fs[0] - fs[1]) / (2 * h)
        assert abs(num - g[k]) <= 2e-3 * np.abs(g).max(), (k, num, g[k])
