"""No-GPU checks of tests/motion_timestamp_reference.py, the f64 reference of the batched parametric average-timestamp
loss, and of the host side of motion_timestamp_objective_torch: the reference's gradient agrees with central differences
for every model; for linvel it agrees with the dense-flow timestamp reference under the uniform flow -v; a rotating scene
has its smallest loss at the true angular velocity; and the argument errors."""
import numpy as np
import pytest
import torch

import flow_timestamp_reference as FR
import motion_timestamp_reference as R

H, W = 30, 40
CENTRE = (20.0, 15.0)
PARAMS = {"linvel": [(30.0, -20.0), (-55.0, 12.5)],
          "rotation": [(20.0, 15.0, 4.0), (18.0, 17.0, -6.0)],
          "xyztheta": [(20.0, -10.0, 3.0, 2.0), (-30.0, 15.0, -2.0, 4.0)]}


def stream(seed, n, margin):
    """events inside [margin, W-1-margin] x [margin, H-1-margin], sorted stamps t in [0, 0.1] and d = t - t[-1]"""
    rng = np.random.default_rng(seed)
    x = (margin + rng.random(n) * (W - 1 - 2 * margin)).astype(np.float32)
    y = (margin + rng.random(n) * (H - 1 - 2 * margin)).astype(np.float32)
    t = (np.sort(rng.random(n)) * 0.1).astype(np.float32)
    d = (t - t[-1]).astype(np.float32)
    p = (rng.integers(0, 2, n) * 2 - 1).astype(np.float32)
    return x, y, t, d, p


@pytest.mark.parametrize("kind", ["linvel", "rotation", "xyztheta"])
@pytest.mark.parametrize("reverse", [False, True])
def test_reference_gradient_matches_central_differences(kind, reverse):
    x, y, t, d, p = stream(2, 3000, 3.0)
    offsets = [0, 1800, 3000]
    tau = FR.tau_f32(t, offsets, reverse)
    prm = torch.tensor(PARAMS[kind], dtype=torch.float64, requires_grad=True)
    g = np.array([1.0, -0.7])
    f, _, _ = R.reference(kind, x, y, d, tau, p, offsets, prm, 1.0, (H, W), CENTRE)
    (f * torch.from_numpy(g)).sum().backward()
    grad = prm.grad.numpy()
    # a step far below a pixel of motion (|d| <= 0.1), so that no floor or keep decision changes
    h = 1e-6
    for b in range(2):
        for k in range(prm.shape[1]):
            fp, fm = prm.detach().clone(), prm.detach().clone()
            fp[b, k] += h
            fm[b, k] -= h
            num = (float(R.reference(kind, x, y, d, tau, p, offsets, fp, 1.0, (H, W), CENTRE)[0][b]) -
                   float(R.reference(kind, x, y, d, tau, p, offsets, fm, 1.0, (H, W), CENTRE)[0][b])) * g[b] / (2 * h)
            assert abs(num - grad[b, k]) <= 1e-6 * np.abs(grad[b]).max() + 1e-5 * abs(num), (kind, b, k, num, grad[b, k])
    assert (np.abs(grad) > 0).all()


@pytest.mark.parametrize("reverse", [False, True])
@pytest.mark.parametrize("sigma", [0.0, 2.0])
def test_linvel_matches_the_flow_timestamp_reference(reverse, sigma):
    """linvel v is the uniform flow -v: the same f, T, C and, summed over the field, the same gradient (no event lands
    at x' = 0 or y' = 0, where the two keep rules differ)"""
    x, y, t, d, p = stream(4, 5000, 0.0)
    offsets = [0, 2000, 5000]
    tau = FR.tau_f32(t, offsets, reverse)
    v = torch.tensor([[60.0, -45.0], [-80.0, 30.0]], dtype=torch.float64, requires_grad=True)
    for b in range(2):
        sl = slice(offsets[b], offsets[b + 1])
        xw, yw = R.warp_f32("linvel", x[sl], y[sl], d[sl], v[b].detach().numpy())
        assert not ((xw == 0) | (yw == 0)).any()
        assert 0.5 < R.contributes(xw, yw, H, W).mean() < 1.0      # some events leave the canvas
    f, T, C = R.reference("linvel", x, y, d, tau, p, offsets, v, sigma, (H, W))
    g = torch.tensor([1.0, -0.4], dtype=torch.float64)
    (f * g).sum().backward()
    flow = (-v.detach()).view(2, 2, 1, 1).expand(2, 2, H, W).clone().requires_grad_(True)
    ff, Tf, Cf = FR.reference(x, y, d, tau, p, offsets, flow, sigma)
    (ff * g).sum().backward()
    np.testing.assert_allclose(f.detach().numpy(), ff.detach().numpy(), rtol=1e-12)
    np.testing.assert_allclose(T.detach().numpy(), Tf.detach().numpy(), rtol=0, atol=1e-12)
    np.testing.assert_allclose(C.detach().numpy(), Cf.detach().numpy(), rtol=0, atol=1e-9)
    np.testing.assert_allclose(v.grad.numpy(), -flow.grad.sum((2, 3)).numpy(), rtol=1e-9,
                               atol=1e-12 * np.abs(v.grad.numpy()).max())


def test_contribute_rule_empty_and_nan_samples():
    x, y, t, d, p = stream(6, 4000, 0.0)
    offsets = [0, 3000, 3000, 4000]
    tau = FR.tau_f32(t, offsets)
    prm = torch.tensor([(300.0, -200.0), (1.0, 1.0), (float("nan"), 0.0)], dtype=torch.float64)
    xw, yw = R.warp_f32("linvel", x[:3000], y[:3000], d[:3000], (300.0, -200.0))
    keep = R.contributes(xw, yw, H, W)
    assert 0.1 < keep.mean() < 0.9
    f, T, C = R.reference("linvel", x, y, d, tau, p, offsets, prm, 2.0, (H, W))
    for s, sel in enumerate((p[:3000] > 0, p[:3000] <= 0)):
        # every contributing event lands whole on the canvas, every other one adds nothing
        assert abs(float(C[0, s].sum()) - (H + 1) * (W + 1) - (keep & sel).sum()) < 1e-9 * len(x)
    # the empty sample and the sample whose every x' is NaN: T = 0, C = 1, f = 0 (no NaN)
    for b in (1, 2):
        assert float(f[b]) == 0.0 and (T[b] == 0).all() and (C[b] == 1).all()


def test_rotating_scene_has_its_minimum_at_the_true_omega():
    """the premise of the GPU recovery test: on a rotating scene (t0 = the last stamp, blur 1) the reference's f over
    omega_true (1 + a), a in -20 % .. 20 %, is smallest at a = 0"""
    omega = 6.0
    x, y, t, p = R.rotating_scene(n_pts=150, per_pt=60, omega=omega)
    d = (t - t[-1]).astype(np.float32)
    tau = FR.tau_f32(t.astype(np.float32), [0, len(t)])
    x, y, p = (a.astype(np.float32) for a in (x, y, p))
    fs = []
    grid = np.linspace(-0.2, 0.2, 9)
    for a in grid:
        prm = torch.tensor([[120.0, 90.0, omega * (1 + a)]], dtype=torch.float64)
        fs.append(float(R.reference("rotation", x, y, d, tau, p, [0, len(t)], prm, 1.0)[0][0]))
    assert int(np.argmin(fs)) == 4, list(zip(grid, fs))


@pytest.mark.parametrize("name", ["evk_motion_timestamp_objective_f32", "evk_motion_timestamp_objective_grad_f32"])
def test_bad_blur_sigma_is_rejected_before_any_cuda_call(name):
    """the blur-sigma rule of every entry that takes a sigma: called with fake, never dereferenced pointers and a huge
    workspace, a NaN blur_sigma is EVK_E_ARG and one needing a radius over 64 is EVK_E_UNSUPPORTED, each with a message
    that names the sigma (without a GPU here, a call that reached CUDA could not return those codes)"""
    import ctypes
    from event_utils_b200 import _lib
    L = _lib.load()
    fn = getattr(L, name)
    fake = ctypes.c_void_p(1 << 20)
    defaults = {ctypes.c_void_p: fake, ctypes.c_int64: 10, ctypes.c_double: 1.0, ctypes.c_int: 4, ctypes.c_size_t: 1 << 40}
    args = [defaults[t] for t in fn.argtypes]
    where = 15                                   # x y t_rel tau p offsets batch n warp params K cx cy H W blur_sigma
    assert fn.argtypes[where] is ctypes.c_double and fn.argtypes[where - 1] is ctypes.c_int
    args[8], args[10] = _lib.WARP_ROTATION, 3
    for sigma, rc in ((float("nan"), -1), (16.125, -5), (1e9, -5), (float("inf"), -5)):
        args[where] = sigma
        assert fn(*args) == rc, (name, sigma)
        msg = L.evk_last_error()
        assert b"blur sigma" in msg and msg.startswith(b"evk_"), (name, sigma, msg)


def test_argument_errors():
    from event_utils_b200.contrast_max import (linvel_warp, motion_timestamp_objective_torch, pure_rotation_warp,
                                               xyztheta_warp)
    x = torch.zeros(10)

    class other_warp(pure_rotation_warp):
        pass

    for bad in (other_warp(), object()):
        with pytest.raises(ValueError, match="supports the models"):
            motion_timestamp_objective_torch(x, x, x, x, torch.zeros(3), bad)
    for warp, bad in ((linvel_warp(), torch.zeros(3)), (pure_rotation_warp(), torch.zeros(2, 2)),
                      (xyztheta_warp(), torch.zeros(1, 3)), (linvel_warp(), torch.zeros(1, 1, 2))):
        with pytest.raises(ValueError, match="must have shape"):
            motion_timestamp_objective_torch(x, x, x, x, bad, warp)
    with pytest.raises(ValueError, match="floating-point"):
        motion_timestamp_objective_torch(x, x, x, x, torch.zeros(2, dtype=torch.int64), linvel_warp())
    with pytest.raises(ValueError, match="2 samples of events for a batch of 3 parameter vectors"):
        motion_timestamp_objective_torch(x, x, x, x, torch.zeros(3, 2), linvel_warp(), batch_end_indices=[4, 10])
    with pytest.raises(ValueError, match="1 samples of events for a batch of 2 parameter vectors"):
        motion_timestamp_objective_torch(x, x, x, x, torch.zeros(2, 2), linvel_warp(), batch_end_indices=torch.tensor([10]))
    with pytest.raises(ValueError, match="must not require grad"):
        motion_timestamp_objective_torch(x.clone().requires_grad_(True), x, x, x, torch.zeros(2), linvel_warp())
    with pytest.raises(ValueError, match="same length"):
        motion_timestamp_objective_torch(x, x[:9], x, x, torch.zeros(2), linvel_warp())
