"""No-GPU checks of motion segmentation: the workspace queries and argument errors of the evk_cmax_motion_segment_*
entries, the shape checks of the torch functions, and the f64 reference of tests/motion_segmentation_reference.py
against central differences in the parameters and the memberships."""
import ctypes

import numpy as np
import pytest
import torch

import motion_segmentation_reference as S

E_ARG, E_WORKSPACE, E_UNSUPPORTED = -1, -3, -5


def _lib():
    from event_utils_b200 import _lib
    return _lib.load()


def test_workspace_queries():
    L = _lib()
    for B, M, H, W in ((1, 1, 2, 2), (5, 2, 180, 240), (64, 4, 60, 80), (0, 3, 10, 10), (3, 8, 20, 30)):
        assert L.evk_cmax_motion_segment_workspace_bytes(B, M, H, W) == L.evk_cmax_motion_objective_workspace_bytes(B * M, H, W)
        for J in (1, 32 // M):
            assert L.evk_cmax_motion_segment_candidates_workspace_bytes(B, M, J, H, W) == \
                L.evk_cmax_motion_candidates_workspace_bytes(B * M, J, H, W)
    for bad in ((-1, 2, 10, 10), (2, 0, 10, 10), (2, 9, 10, 10), (2, 2, 1, 10), (2, 2, 10, 1)):
        assert L.evk_cmax_motion_segment_workspace_bytes(*bad) == 0, bad
    for bad in ((2, 4, 9, 10, 10), (2, 8, 5, 10, 10), (2, 2, 0, 10, 10), (2, 0, 4, 10, 10), (2, 9, 1, 10, 10)):
        assert L.evk_cmax_motion_segment_candidates_workspace_bytes(*bad) == 0, bad


FAKE = ctypes.c_void_p(1 << 20)     # aligned, never dereferenced


def _args(**kw):
    a = dict(batch=4, n=1000, warp=1, M=2, J=4, K=3, H=60, W=80, sigma=1.0, objective=0, ws_bytes=1 << 40, weights=FAKE,
             eps=1e-6)
    a.update(kw)
    return a


def _forward(**kw):
    a = _args(**kw)
    L = _lib()
    rc = L.evk_cmax_motion_segment_f32(FAKE, FAKE, FAKE, FAKE, a["weights"], a["M"], FAKE, a["batch"], a["n"], a["warp"], FAKE,
                                       a["K"], 40.0, 30.0, a["H"], a["W"], a["sigma"], a["objective"], 3.0, FAKE, FAKE, FAKE,
                                       a["ws_bytes"], None)
    return rc, L.evk_last_error()


def _grad(**kw):
    a = _args(**kw)
    L = _lib()
    rc = L.evk_cmax_motion_segment_grad_f32(FAKE, FAKE, FAKE, FAKE, a["weights"], a["M"], FAKE, a["batch"], a["n"], a["warp"],
                                            FAKE, a["K"], 40.0, 30.0, a["H"], a["W"], a["sigma"], a["objective"], 3.0, FAKE, FAKE,
                                            FAKE, FAKE, FAKE, a["ws_bytes"], None)
    return rc, L.evk_last_error()


def _candidates(**kw):
    a = _args(**kw)
    L = _lib()
    rc = L.evk_cmax_motion_segment_candidates_f32(FAKE, FAKE, FAKE, FAKE, a["weights"], a["M"], FAKE, a["batch"], a["n"],
                                                  a["warp"], FAKE, a["J"], a["K"], 40.0, 30.0, a["H"], a["W"], a["sigma"],
                                                  a["objective"], 3.0, FAKE, FAKE, a["ws_bytes"], None)
    return rc, L.evk_last_error()


def _assign(**kw):
    a = _args(**kw)
    L = _lib()
    rc = L.evk_cmax_motion_segment_assign_f32(FAKE, FAKE, FAKE, a["M"], FAKE, a["batch"], a["n"], a["warp"], FAKE, a["K"], 40.0,
                                              30.0, a["H"], a["W"], FAKE, a["sigma"], a["eps"], FAKE, FAKE, a["ws_bytes"], None)
    return rc, L.evk_last_error()


@pytest.mark.parametrize("entry", [_forward, _grad, _candidates, _assign])
def test_argument_errors_without_a_gpu(entry):
    for M in (0, 9, -1):
        rc, msg = entry(M=M)
        assert rc == E_ARG and b"n_models" in msg, (M, msg)
    rc, msg = entry(batch=32768, M=2, J=1)                  # 65536 canvases
    assert rc == E_ARG and b"65535" in msg, msg
    assert entry(K=2)[0] == E_ARG                           # rotation has K = 3
    assert entry(warp=3, K=3)[0] == E_ARG                   # linvel has K = 2
    assert entry(warp=7)[0] == E_ARG
    assert entry(batch=-1)[0] == E_ARG
    assert entry(H=1)[0] == E_ARG
    assert entry(sigma=float("nan"))[0] == E_ARG
    if entry is not _assign:
        rc, msg = entry(weights=None)
        assert rc == E_ARG and b"null weights" in msg, msg
        for obj in (3, 4):                                  # moa, isoa
            rc, msg = entry(objective=obj)
            assert rc == E_UNSUPPORTED and b"piecewise constant" in msg
        assert entry(objective=9)[0] == E_ARG
    else:
        for eps in (-1e-9, float("nan"), float("inf")):
            rc, msg = entry(eps=eps)
            assert rc == E_ARG and b"eps" in msg, (eps, msg)
    L = _lib()
    if entry is _candidates:
        for M, J in ((4, 9), (8, 5), (2, 0)):
            rc, msg = entry(M=M, J=J)
            assert rc == E_ARG and b"n_cand" in msg, (M, J, msg)
        rc, msg = entry(batch=8192, M=2, J=4)               # 65536 canvases
        assert rc == E_ARG and b"65535" in msg
        need = L.evk_cmax_motion_segment_candidates_workspace_bytes(4, 2, 4, 60, 80)
    else:
        need = L.evk_cmax_motion_segment_workspace_bytes(4, 2, 60, 80)
    rc, msg = entry(ws_bytes=need - 1)
    assert rc == E_WORKSPACE and b"workspace" in msg


def test_python_shape_checks():
    from event_utils_b200.contrast_max import (linvel_warp, motion_segmentation_assign_torch, motion_segmentation_candidates_torch,
                                               motion_segmentation_fit_torch, motion_segmentation_objective_torch,
                                               pure_rotation_warp)
    e = torch.zeros(10)
    w = torch.full((10, 2), 0.5)
    rot = pure_rotation_warp()
    with pytest.raises(ValueError, match="weights must have shape"):
        motion_segmentation_objective_torch(e, e, e, e, torch.ones(9, 2), torch.zeros(2, 3), rot)
    with pytest.raises(ValueError, match="weights must have shape"):
        motion_segmentation_objective_torch(e, e, e, e, torch.ones(10, 9), torch.zeros(9, 3), rot)
    with pytest.raises(ValueError, match="weights must have shape"):
        motion_segmentation_objective_torch(e, e, e, e, torch.ones(10), torch.zeros(1, 3), rot)
    with pytest.raises(ValueError, match="floating-point"):
        motion_segmentation_objective_torch(e, e, e, e, torch.ones(10, 2, dtype=torch.int32), torch.zeros(2, 3), rot)
    with pytest.raises(ValueError, match="params must have shape"):
        motion_segmentation_objective_torch(e, e, e, e, w, torch.zeros(3, 3), rot)          # 3 models, weights have 2
    with pytest.raises(ValueError, match="params must have shape"):
        motion_segmentation_objective_torch(e, e, e, e, w, torch.zeros(1, 2, 2), rot)       # K = 2 for rotation
    with pytest.raises(ValueError, match="piecewise constant"):
        motion_segmentation_objective_torch(e, e, e, e, w, torch.zeros(2, 3), rot, objective="isoa")
    with pytest.raises(ValueError, match="must not require grad"):
        motion_segmentation_objective_torch(e.clone().requires_grad_(True), e, e, e, w, torch.zeros(2, 3), rot)
    with pytest.raises(ValueError, match="candidates must have shape"):
        motion_segmentation_candidates_torch(e, e, e, e, torch.zeros(1, 2, 3), w, rot)
    with pytest.raises(ValueError, match="candidates must have shape"):
        motion_segmentation_candidates_torch(e, e, e, e, torch.zeros(1, 3, 4, 3), w, rot)    # 3 models
    with pytest.raises(ValueError, match="candidates must have shape"):
        motion_segmentation_candidates_torch(e, e, e, e, torch.zeros(1, 2, 0, 3), w, rot)    # J = 0
    with pytest.raises(ValueError, match="eps"):
        motion_segmentation_assign_torch(e, e, e, e, torch.zeros(2, 3), rot, w, eps=-1.0)
    with pytest.raises(ValueError, match="x0 must have shape"):
        motion_segmentation_fit_torch(e, e, e, e, linvel_warp(), torch.zeros(2, 3))
    with pytest.raises(ValueError, match="x0 must have shape"):
        motion_segmentation_fit_torch(e, e, e, e, linvel_warp(), torch.zeros(9, 2))          # M <= 8
    with pytest.raises(ValueError, match="x0 must have shape"):
        motion_segmentation_fit_torch(e, e, e, e, linvel_warp(), torch.zeros(3, 2, 2), batch_end_indices=[4, 10])
    with pytest.raises(ValueError, match="weights0 has 2 models"):
        motion_segmentation_fit_torch(e, e, e, e, linvel_warp(), torch.zeros(3, 2), weights0=w)
    with pytest.raises(ValueError, match="line_search_steps"):
        motion_segmentation_fit_torch(e, e, e, e, linvel_warp(), torch.zeros(2, 2), line_search_steps=0)


def _events(seed, n, margin=20.0):
    rng = np.random.default_rng(seed)
    x = (margin + rng.random(n) * (239 - 2 * margin)).astype(np.float32)
    y = (margin + rng.random(n) * (179 - 2 * margin)).astype(np.float32)
    t = np.sort(rng.integers(0, 410, n)) / 4096.0
    p = (rng.integers(0, 2, n) * 2 - 1).astype(np.float32)
    return x, y, (t - t[-1]).astype(np.float32), p


MODELS = {"linvel": [(30.0, -20.0), (-45.0, 10.0)], "rotation": [(130.0, 85.0, 4.0), (110.0, 95.0, -3.0)],
          "xyztheta": [(20.0, -10.0, 3.0, 2.0), (-15.0, 12.0, -2.0, 1.0)]}


@pytest.mark.parametrize("kind", ["linvel", "rotation", "xyztheta"])
@pytest.mark.parametrize("name", ["variance", "soe", "sosa"])
def test_reference_gradients_match_central_differences(kind, name):
    x, y, d, p = _events(2, 1500)
    rng = np.random.default_rng(3)
    w = torch.tensor(rng.random((1500, 2)), dtype=torch.float64, requires_grad=True)
    prm = torch.tensor([MODELS[kind]], dtype=torch.float64, requires_grad=True)
    off = [0, 1500]
    gf = torch.tensor([[1.0, -0.7]], dtype=torch.float64)
    f, _ = S.reference(kind, x, y, d, p, w, off, prm, 1.0, name, 0.5)
    (f * gf).sum().backward()
    g, gw = prm.grad[0].numpy(), w.grad.numpy()

    def F(q, ww):
        return float((S.reference(kind, x, y, d, p, ww, off, q, 1.0, name, 0.5)[0] * gf).sum())
    for m in range(2):
        scale = np.abs(g[m]).max()
        for k in range(prm.shape[2]):
            h = 1e-7 if (kind == "rotation" and k == 2) else 1e-6      # no event crosses a pixel edge
            q = [prm.detach().clone() for _ in range(2)]
            q[0][0, m, k] += h
            q[1][0, m, k] -= h
            num = (F(q[0], w.detach()) - F(q[1], w.detach())) / (2 * h)
            assert abs(num - g[m, k]) <= 2e-3 * scale, (kind, name, m, k, num, g[m, k])
    wscale = np.abs(gw).max()
    assert wscale > 0
    for e in (0, 7, 500, 1499):
        for m in range(2):
            h = 1e-4
            wp, wm = w.detach().clone(), w.detach().clone()
            wp[e, m] += h
            wm[e, m] -= h
            num = (F(prm.detach(), wp) - F(prm.detach(), wm)) / (2 * h)
            assert abs(num - gw[e, m]) <= 1e-4 * wscale, (kind, name, e, m, num, gw[e, m])


def test_reference_at_one_model_is_the_motion_objective():
    import motion_objective_reference as R
    x, y, d, p = _events(4, 3000)
    prm = torch.tensor([[(130.0, 85.0, 4.0)], [(110.0, 95.0, -3.0)]], dtype=torch.float64)
    off = [0, 1000, 3000]
    w = torch.ones((3000, 1), dtype=torch.float64)
    f, img = S.reference("rotation", x, y, d, p, w, off, prm, 1.0, "variance")
    fr, imgr, _ = R.reference("rotation", x, y, d, p, off, prm[:, 0], 1.0, "variance")
    assert torch.equal(img[:, 0], imgr) and torch.equal(f[:, 0], fr)


def test_reference_assignment_rules():
    x, y, d, p = _events(5, 2000)
    prm = np.array([MODELS["linvel"]], np.float64)
    off = [0, 1500]
    w = torch.full((2000, 2), 0.5, dtype=torch.float64)
    _, img = S.reference("linvel", x, y, d, p, w, off, torch.tensor(prm), 1.0, "variance")
    a = S.assign("linvel", x, y, d, off, prm, np.abs(img.numpy()), 1.0, 1e-6)
    np.testing.assert_allclose(a.sum(1), 1.0, rtol=1e-12)
    assert (a[1500:] == 0.5).all()                                  # outside every window
    z = S.assign("linvel", x, y, d, off, prm, np.zeros_like(img.numpy()), 1.0, 0.0)
    assert (z == 0.5).all()                                         # every c = 0 with eps = 0
