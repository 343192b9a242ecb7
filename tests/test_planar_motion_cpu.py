"""No-GPU checks of the planar motion models (affine_warp, homography_warp): their warp() against the closed forms and
central differences, the embeddings xyztheta -> affine -> homography bit for bit, the model codes of the batched losses,
and the argument errors of the C entries, which are raised before any CUDA call."""
import ctypes

import numpy as np
import pytest
import torch

import planar_motion_reference as P

E_ARG = -1
CENTRE = (120.0, 90.0)
AFFINE = (20.0, -10.0, 3.0, -2.0, 1.5, -4.0)
HOMOGRAPHY = AFFINE + (0.02, -0.03)


def _warps():
    from event_utils_b200.contrast_max.warps import affine_warp, homography_warp, xyztheta_warp
    return affine_warp, homography_warp, xyztheta_warp


def _events(seed, n):
    rng = np.random.default_rng(seed)
    x, y = rng.uniform(5, 235, n), rng.uniform(5, 175, n)
    t = np.sort(rng.uniform(0, 0.1, n))
    return x, y, t, rng.integers(0, 2, n) * 2.0 - 1


def test_warp_matches_the_closed_forms_and_central_differences():
    affine_warp, homography_warp, _ = _warps()
    x, y, t, p = _events(1, 2000)
    t0 = t[-1]
    d, u, v = t - t0, x - CENTRE[0], y - CENTRE[1]
    for warp, prm in ((affine_warp(), AFFINE), (homography_warp(), HOMOGRAPHY)):
        xw, yw, jx, jy = warp.warp(x, y, t, p, t0, prm, compute_grad=True)
        hx, hy, a11, a12, a21, a22 = prm[:6]
        g1, g2 = (prm[6], prm[7]) if len(prm) == 8 else (0.0, 0.0)
        A = np.array([[a11, a12], [a21, a22]])
        n = np.stack((u, v)) - d * (A @ np.stack((u, v)) + np.array([[hx], [hy]]))
        w = 1 - d * (g1 * u + g2 * v)
        np.testing.assert_allclose(xw, CENTRE[0] + n[0] / w, rtol=0, atol=1e-9)
        np.testing.assert_allclose(yw, CENTRE[1] + n[1] / w, rtol=0, atol=1e-9)
        assert jx.shape == jy.shape == (warp.dims, x.size)
        np.testing.assert_allclose(jx, P.jacobian(warp.name.split("_")[0], x, y, d, prm)[0], rtol=1e-12, atol=1e-15)
        for k in range(warp.dims):
            h = 1e-6 * max(1.0, abs(prm[k]))
            hi, lo = list(prm), list(prm)
            hi[k] += h
            lo[k] -= h
            xp, yp, _, _ = warp.warp(x, y, t, p, t0, hi)
            xm, ym, _, _ = warp.warp(x, y, t, p, t0, lo)
            np.testing.assert_allclose((xp - xm) / (2 * h), jx[k], rtol=1e-5, atol=1e-7)
            np.testing.assert_allclose((yp - ym) / (2 * h), jy[k], rtol=1e-5, atol=1e-7)


def test_embeddings_bit_for_bit():
    affine_warp, homography_warp, xyztheta_warp = _warps()
    x, y, t, p = _events(2, 3000)
    hx, hy, hz, th = 20.0, -10.0, 3.0, 2.0
    xyz = xyztheta_warp().warp(x, y, t, p, t[-1], (hx, hy, hz, th), True)
    aff = affine_warp().warp(x, y, t, p, t[-1], (hx, hy, hz, -th, th, hz), True)
    for a, b in zip(xyz[:2], aff[:2]):
        assert np.array_equal(a, b)
    assert np.array_equal(aff[2][0], xyz[2][0]) and np.array_equal(aff[3][1], xyz[3][1])
    assert np.array_equal(aff[2][2], xyz[2][2]) and np.array_equal(aff[3][5], xyz[3][2])
    hom = homography_warp().warp(x, y, t, p, t[-1], (hx, hy, hz, -th, th, hz, 0.0, 0.0), True)
    for a, b in zip(hom[:4], aff[:4]):
        assert np.array_equal(a[:6] if a.ndim == 2 else a, b)
    # the f32 restatement of the kernel's warp, likewise
    x32, y32, d32 = (np.asarray(a, np.float32) for a in (x, y, t - t[-1]))
    from motion_objective_reference import warp_f32 as warp4
    w4 = warp4("xyztheta", x32, y32, d32, (hx, hy, hz, th))
    wa = P.warp_f32("affine", x32, y32, d32, (hx, hy, hz, -th, th, hz))
    wh = P.warp_f32("homography", x32, y32, d32, (hx, hy, hz, -th, th, hz, 0.0, 0.0))
    for a, b, c in zip(w4, wa, wh):
        assert np.array_equal(a, b) and np.array_equal(b, c)


def test_horizon_in_the_f32_warp():
    x = np.array([200.0, 10.0, 120.0], np.float32)
    y = np.array([90.0, 90.0, 90.0], np.float32)
    d = np.full(3, -0.1, np.float32)
    # w = 1 - d g1 u = 1 + 0.1 * 0.1 * u: u = 80 -> 1.8, u = -110 -> -0.1 (past the horizon), u = 0 -> 1
    xw, yw = P.warp_f32("homography", x, y, d, (0, 0, 0, 0, 0, 0, 0.1, 0.0))
    assert np.isnan(xw[1]) and np.isnan(yw[1])
    assert np.isfinite(xw[[0, 2]]).all()
    assert P.contributes(xw, yw, 180, 240).tolist() == [True, False, True]


def test_model_codes_and_dims():
    from event_utils_b200 import _lib
    from event_utils_b200.contrast_max import _batched as B
    affine_warp, homography_warp, _ = _warps()
    for cls, code, K in ((affine_warp, _lib.WARP_AFFINE, 6), (homography_warp, _lib.WARP_HOMOGRAPHY, 8)):
        w = cls(center=(40.0, 30.0))
        assert B._warp_code(w, "f") == code and w.dims == K and w.fused_kind is None
        assert w.model(list(range(K))) == [float(k) for k in range(K)] + [40.0, 30.0]
        assert B._model(code, w, "variance", 1.0, None, 60, 80)[1] == (40.0, 30.0)
        assert B._ts_model(code, w, 1.0, 60, 80)[1] == (40.0, 30.0)

        class sub(cls):
            pass
        with pytest.raises(ValueError, match="supports the models") as e:
            B._warp_code(sub(), "f")
        assert "linvel_warp, pure_rotation_warp and xyztheta_warp" in str(e.value)
    assert (_lib.WARP_AFFINE, _lib.WARP_HOMOGRAPHY) == (4, 5)


FAKE = ctypes.c_void_p(1 << 20)     # aligned, never dereferenced


def _entries():
    """every batched motion entry as f(warp, K) -> (rc, message), all other arguments valid"""
    from event_utils_b200 import _lib
    L = _lib.load()
    F, B, N, H, W, S, J, WS = FAKE, 2, 100, 60, 80, 1.0, 4, 1 << 40
    calls = {
        "contrast": lambda w, K: L.evk_cmax_motion_objective_f32(F, F, F, F, F, B, N, w, F, K, 40.0, 30.0, H, W, S, 0, 0.0, F, F,
                                                                 F, WS, None),
        "contrast_grad": lambda w, K: L.evk_cmax_motion_objective_grad_f32(F, F, F, F, F, B, N, w, F, K, 40.0, 30.0, H, W, S, 0,
                                                                           0.0, F, F, F, F, WS, None),
        "contrast_cand": lambda w, K: L.evk_cmax_motion_candidates_f32(F, F, F, F, F, B, N, w, F, J, K, 40.0, 30.0, H, W, S, 0, 0.0,
                                                                       F, F, WS, None),
        "ts": lambda w, K: L.evk_motion_timestamp_objective_f32(F, F, F, F, F, F, B, N, w, F, K, 40.0, 30.0, H, W, S, F, F, F, F, WS,
                                                                None),
        "ts_grad": lambda w, K: L.evk_motion_timestamp_objective_grad_f32(F, F, F, F, F, F, B, N, w, F, K, 40.0, 30.0, H, W, S, F, F,
                                                                          F, F, F, WS, None),
        "ts_cand": lambda w, K: L.evk_motion_timestamp_candidates_f32(F, F, F, F, F, F, B, N, w, F, J, K, 40.0, 30.0, H, W, S, F, F,
                                                                      WS, None),
        "seg": lambda w, K: L.evk_cmax_motion_segment_f32(F, F, F, F, F, 2, F, B, N, w, F, K, 40.0, 30.0, H, W, S, 0, 0.0, F, F, F,
                                                          WS, None),
        "seg_grad": lambda w, K: L.evk_cmax_motion_segment_grad_f32(F, F, F, F, F, 2, F, B, N, w, F, K, 40.0, 30.0, H, W, S, 0, 0.0,
                                                                    F, F, F, F, F, WS, None),
        "seg_cand": lambda w, K: L.evk_cmax_motion_segment_candidates_f32(F, F, F, F, F, 2, F, B, N, w, F, J, K, 40.0, 30.0, H, W,
                                                                          S, 0, 0.0, F, F, WS, None),
        "assign": lambda w, K: L.evk_cmax_motion_segment_assign_f32(F, F, F, 2, F, B, N, w, F, K, 40.0, 30.0, H, W, F, S, 1e-6, F,
                                                                    F, WS, None),
    }
    return {k: (lambda c: lambda w, K: (c(w, K), L.evk_last_error()))(c) for k, c in calls.items()}


@pytest.mark.parametrize("entry", ["contrast", "contrast_grad", "contrast_cand", "ts", "ts_grad", "ts_cand", "seg", "seg_grad",
                                   "seg_cand", "assign"])
def test_entries_check_the_parameter_count_before_any_cuda_call(entry):
    call = _entries()[entry]
    rc, msg = call(4, 4)
    assert rc == E_ARG and b"has 6 parameters" in msg, msg
    rc, msg = call(5, 6)
    assert rc == E_ARG and b"has 8 parameters" in msg, msg
    rc, msg = call(7, 8)
    assert rc == E_ARG and b"unknown warp" in msg, msg


def test_torch_functions_check_the_parameter_shape():
    from event_utils_b200.contrast_max import motion_contrast_objective_torch, motion_timestamp_objective_torch
    affine_warp, homography_warp, _ = _warps()
    x = torch.zeros(10)
    for fn in (motion_contrast_objective_torch, motion_timestamp_objective_torch):
        with pytest.raises(ValueError, match=r"\(B,6\)"):
            fn(x, x, x, x, torch.zeros(4), affine_warp())
        with pytest.raises(ValueError, match=r"\(B,8\)"):
            fn(x, x, x, x, torch.zeros(2, 6), homography_warp())


@pytest.mark.parametrize("kind", ["affine", "homography"])
def test_reference_gradient_matches_central_differences(kind):
    rng = np.random.default_rng(3)
    n = 3000
    x = rng.uniform(20, 220, n).astype(np.float32)
    y = rng.uniform(20, 160, n).astype(np.float32)
    d = (-np.sort(rng.integers(0, 410, n))[::-1] / 4096.0).astype(np.float32)
    p = (rng.integers(0, 2, n) * 2 - 1).astype(np.float32)
    prm0 = AFFINE if kind == "affine" else HOMOGRAPHY
    prm = torch.tensor([prm0], dtype=torch.float64, requires_grad=True)
    f, _ = P.contrast(kind, x, y, d, p, [0, n], prm, 1.0, "variance")
    f.sum().backward()
    g = prm.grad[0].numpy()
    scale = np.abs(g).max()
    for k in range(prm.shape[1]):
        h = 1e-8 if k >= 6 else 1e-6     # small enough that no event crosses a pixel edge
        fs = []
        for sgn in (1, -1):
            q = prm.detach().clone()
            q[0, k] += sgn * h
            fs.append(float(P.contrast(kind, x, y, d, p, [0, n], q, 1.0, "variance")[0][0]))
        num = (fs[0] - fs[1]) / (2 * h)
        assert abs(num - g[k]) <= 2e-3 * scale, (kind, k, num, g[k], scale)
