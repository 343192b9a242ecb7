"""No-GPU checks of tests/motion_objective_reference.py, the f64 reference of the batched parametric contrast objective:
per sample it agrees with the K-channel oracle of tests/cmax_warp_oracle.py (f and IWE), its autograd gradient agrees
with central differences, and xyztheta without expansion and rotation has linvel's gradient.  Also the argument errors
of motion_contrast_objective_torch, which are raised before any GPU work."""
import numpy as np
import pytest
import torch

import motion_objective_reference as R
from cmax_warp_oracle import iwe_warp, objective_f

POINTS = {"linvel": (30.0, -20.0), "rotation": (130.0, 85.0, 4.0), "xyztheta": (20.0, -10.0, 3.0, 2.0)}


def _warp(kind):
    from event_utils_b200.contrast_max.warps import linvel_warp, pure_rotation_warp, xyztheta_warp
    return {"linvel": linvel_warp, "rotation": pure_rotation_warp, "xyztheta": xyztheta_warp}[kind]()


def _events(seed, n, margin=2.0):
    """f32-exact events inside the sensor (margin px from the border), stamps on a 2^-12 grid in [0, 0.1]"""
    rng = np.random.default_rng(seed)
    x = (margin + rng.random(n) * (239 - 2 * margin)).astype(np.float32)
    y = (margin + rng.random(n) * (179 - 2 * margin)).astype(np.float32)
    t = np.sort(rng.integers(0, 410, n)) / 4096.0
    p = (rng.integers(0, 2, n) * 2 - 1).astype(np.float32)
    return x, y, t, p


@pytest.mark.parametrize("kind", ["linvel", "rotation", "xyztheta"])
@pytest.mark.parametrize("name", ["variance", "sos", "soe", "sosa"])
@pytest.mark.parametrize("sigma", [0.0, 1.0])
def test_reference_matches_the_warp_oracle(oracle, kind, name, sigma):
    x, y, t, p = _events(1, 6000)
    d = (t - t[-1]).astype(np.float32)                      # exact: the f64 warp of the oracle sees the same dt
    prm = POINTS[kind]
    param = 0.5
    f, iwe, _ = R.reference(kind, x, y, d, p, [0, len(x)], torch.tensor([prm], dtype=torch.float64), sigma, name, param)
    iwe_o, _, oob = iwe_warp(_warp(kind), prm, x.astype(np.float64), y.astype(np.float64), t, p.astype(np.float64))
    assert oob == 0
    np.testing.assert_allclose(iwe[0].detach().numpy(), iwe_o, rtol=0, atol=1e-5 * np.abs(iwe_o).max())
    fo = objective_f(name, iwe_o, sigma, param)
    assert abs(float(f[0]) - fo) <= 1e-6 * abs(fo), (kind, name, sigma, float(f[0]), fo)


@pytest.mark.parametrize("kind", ["linvel", "rotation", "xyztheta"])
@pytest.mark.parametrize("name", ["variance", "soe", "sosa"])
def test_reference_gradient_matches_central_differences(kind, name):
    x, y, t, p = _events(2, 3000, margin=20.0)
    d = (t - t[-1]).astype(np.float32)
    prm = torch.tensor([POINTS[kind]], dtype=torch.float64, requires_grad=True)
    f, _, _ = R.reference(kind, x, y, d, p, [0, len(x)], prm, 1.0, name, 0.5)
    f.sum().backward()
    g = prm.grad[0].numpy()
    scale = np.abs(g).max()
    for k in range(prm.shape[1]):
        h = 1e-7 if (kind == "rotation" and k == 2) else 1e-6     # small enough that no event crosses a pixel edge
        fp, fm = [], []
        for sgn, out in ((1, fp), (-1, fm)):
            q = prm.detach().clone()
            q[0, k] += sgn * h
            out.append(float(R.reference(kind, x, y, d, p, [0, len(x)], q, 1.0, name, 0.5)[0][0]))
        num = (fp[0] - fm[0]) / (2 * h)
        assert abs(num - g[k]) <= 2e-3 * scale, (kind, name, k, num, g[k], scale)


def test_xyztheta_without_expansion_and_rotation_has_the_linvel_gradient():
    x, y, t, p = _events(3, 5000, margin=10.0)
    d = (t - t[-1]).astype(np.float32)
    for name, sigma in (("variance", 1.0), ("soe", 0.0), ("sosa", 3.0)):
        lin = torch.tensor([[48.0, -32.0]], dtype=torch.float64, requires_grad=True)
        xyz = torch.tensor([[48.0, -32.0, 0.0, 0.0]], dtype=torch.float64, requires_grad=True)
        fl, il, _ = R.reference("linvel", x, y, d, p, [0, len(x)], lin, sigma, name, 0.5)
        fx, ix, _ = R.reference("xyztheta", x, y, d, p, [0, len(x)], xyz, sigma, name, 0.5)
        assert torch.equal(il, ix) and float(fl[0].detach()) == float(fx[0].detach())
        fl.sum().backward()
        fx.sum().backward()
        np.testing.assert_allclose(xyz.grad[0, :2].numpy(), lin.grad[0].numpy(), rtol=1e-12, atol=0)


def test_reference_keep_rule_and_empty_samples():
    x, y, t, p = _events(4, 4000, margin=0.0)
    d = (t - t[-1]).astype(np.float32)
    prm = torch.tensor([[400.0, -300.0], [0.0, 0.0], [0.0, 0.0]], dtype=torch.float64)
    f, iwe, _ = R.reference("linvel", x, y, d, p, [0, 3000, 3000, 4000], prm, 0.0, "variance")
    xw, yw = R.warp_f32("linvel", x[:3000], y[:3000], d[:3000], (400.0, -300.0))
    k = R.contributes(xw, yw, 180, 240)
    assert 0.1 < k.mean() < 0.9
    assert abs(float(iwe[0].sum()) - float(p[:3000][k].astype(np.float64).sum())) < 1e-9 * k.sum()
    assert float(f[1]) == 0.0 and (iwe[1] == 0).all()


def test_argument_errors():
    from event_utils_b200.contrast_max import linvel_warp, motion_contrast_objective_torch, pure_rotation_warp, xyztheta_warp
    from event_utils_b200.contrast_max.warps import warp_function
    x = torch.zeros(10)
    with pytest.raises(ValueError, match="has shape|must have shape"):
        motion_contrast_objective_torch(x, x, x, x, torch.zeros(3), linvel_warp())
    with pytest.raises(ValueError, match="must have shape"):
        motion_contrast_objective_torch(x, x, x, x, torch.zeros(2, 4), pure_rotation_warp())

    class other(warp_function):
        def __init__(self):
            super().__init__("other", 2)

        def warp(self, xs, ys, ts, ps, t0, params, compute_grad=False):
            return xs, ys, None, None

    class sub(linvel_warp):
        fused_kind = None
    for w in (other(), sub()):
        with pytest.raises(ValueError, match="linvel_warp, pure_rotation_warp and xyztheta_warp"):
            motion_contrast_objective_torch(x, x, x, x, torch.zeros(2), w)
    for name in ("moa", "isoa"):
        with pytest.raises(ValueError, match="piecewise constant"):
            motion_contrast_objective_torch(x, x, x, x, torch.zeros(4), xyztheta_warp(), objective=name)
    with pytest.raises(ValueError, match="unknown objective"):
        motion_contrast_objective_torch(x, x, x, x, torch.zeros(2), linvel_warp(), objective="r2")
    with pytest.raises(ValueError, match="must not require grad"):
        motion_contrast_objective_torch(x.clone().requires_grad_(True), x, x, x, torch.zeros(2), linvel_warp())
    with pytest.raises(ValueError, match="must not require grad"):
        motion_contrast_objective_torch(x, x, x, x, torch.zeros(2), linvel_warp(), t0=torch.zeros((), requires_grad=True))
