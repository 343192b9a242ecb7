"""No-GPU checks of the grid-flow contrast loss and fit (contrast_max/grid_flow.py): the f64 reference of
tests/grid_flow_reference.py against the dense-flow reference, the smoothness term, the argument checks that run before
any CUDA call, and the C entries' limits and workspace queries."""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import flow_objective_reference as FR
import grid_flow_reference as GR


def stream(seed, sizes, H, W, integer):
    rng = np.random.default_rng(seed)
    n = sum(sizes)
    if integer:
        x, y = rng.integers(0, W, n).astype(np.float32), rng.integers(0, H, n).astype(np.float32)
    else:
        x, y = (rng.random(n) * (W - 1)).astype(np.float32), (rng.random(n) * (H - 1)).astype(np.float32)
    p = (rng.integers(0, 2, n) * 2 - 1).astype(np.float32)
    d = (-rng.random(n) * 0.1).astype(np.float32)
    off = np.concatenate(([0], np.cumsum(sizes))).astype(np.int64)
    return x, y, d, p, off


@pytest.mark.parametrize("name", ["variance", "soe"])
@pytest.mark.parametrize("grid", [(2, 2), (3, 4), (5, 7)])
def test_reference_equals_dense_reference_on_the_interpolated_flow(name, grid):
    """integer event coordinates: f, IWE and gradient of the grid reference equal the dense-flow reference's on
    F.interpolate(grid, (H, W), bilinear, align_corners=True), the gradient through that composition"""
    H, W = 12, 16
    x, y, d, p, off = stream(1, [400, 300], H, W, True)
    rng = np.random.default_rng(2)
    g0 = torch.from_numpy(rng.standard_normal((2, 2) + grid) * 20.0)
    g1 = g0.clone().requires_grad_(True)
    f, iwe = GR.reference(x, y, d, p, off, g1, H, W, 1.0, name, 0.3)
    f.sum().backward()
    g2 = g0.clone().requires_grad_(True)
    dense = F.interpolate(g2, (H, W), mode="bilinear", align_corners=True)
    fd, iwed, _ = FR.reference(x, y, d, p, off, dense, 1.0, name, 0.3)
    fd.sum().backward()
    np.testing.assert_allclose(f.detach().numpy(), fd.detach().numpy(), rtol=1e-5)
    np.testing.assert_allclose(iwe.detach().numpy(), iwed.detach().numpy(), atol=1e-4)
    np.testing.assert_allclose(g1.grad.numpy(), g2.grad.numpy(), rtol=1e-4, atol=1e-6 * np.abs(g2.grad.numpy()).max())


def test_full_resolution_grid_is_the_dense_flow():
    """gh = H, gw = W: the grid reference is the dense-flow reference on the same field, at any coordinates"""
    H, W = 9, 11
    x, y, d, p, off = stream(3, [500], H, W, False)
    g = torch.from_numpy(np.random.default_rng(4).standard_normal((1, 2, H, W)) * 15.0)
    f, iwe = GR.reference(x, y, d, p, off, g, H, W, 0.0, "variance")
    fd, iwed, _ = FR.reference(x, y, d, p, off, g, 0.0, "variance")
    np.testing.assert_allclose(f.numpy(), fd.numpy(), rtol=1e-6)
    np.testing.assert_allclose(iwe.numpy(), iwed.numpy(), atol=1e-5)


def test_charbonnier_smoothness_and_gradient_match_autograd():
    from event_utils_b200.contrast_max import charbonnier_smoothness
    g = torch.from_numpy(np.random.default_rng(5).standard_normal((3, 2, 4, 5)) * 3.0).requires_grad_(True)
    R, dR = charbonnier_smoothness(g.detach(), 0.7)
    e = 0.7
    dh = g[..., :, 1:] - g[..., :, :-1]
    dv = g[..., 1:, :] - g[..., :-1, :]
    Ra = (torch.sqrt(dh ** 2 + e * e) - e).sum((1, 2, 3)) + (torch.sqrt(dv ** 2 + e * e) - e).sum((1, 2, 3))
    Ra.sum().backward()
    np.testing.assert_allclose(R.numpy(), Ra.detach().numpy(), rtol=1e-12)
    np.testing.assert_allclose(dR.numpy(), g.grad.numpy(), rtol=1e-12, atol=1e-15)
    # a constant flow costs nothing
    R0, dR0 = charbonnier_smoothness(torch.full((2, 3, 3), 4.0, dtype=torch.float64), 1.0)
    assert R0.item() == 0.0 and (dR0 == 0).all()


def test_argument_checks_run_before_any_cuda_call():
    from event_utils_b200.contrast_max import (grid_flow_contrast_candidates_torch, grid_flow_contrast_objective_torch,
                                              grid_flow_fit_torch)
    x = torch.zeros(8)
    t = torch.arange(8.0)
    with pytest.raises(ValueError, match="node grid"):
        grid_flow_contrast_objective_torch(x, x, t, x, torch.zeros(2, 13, 4), (12, 16))
    with pytest.raises(ValueError, match="node grid"):
        grid_flow_contrast_objective_torch(x, x, t, x, torch.zeros(2, 65, 65), (100, 100))
    with pytest.raises(ValueError, match="shape"):
        grid_flow_contrast_objective_torch(x, x, t, x, torch.zeros(3, 3, 4), (12, 16))
    with pytest.raises(ValueError, match="piecewise constant"):
        grid_flow_contrast_objective_torch(x, x, t, x, torch.zeros(2, 3, 4), (12, 16), objective="moa")
    with pytest.raises(ValueError, match="shape"):
        grid_flow_contrast_candidates_torch(x, x, t, x, torch.zeros(1, 2, 3, 4), (12, 16))
    with pytest.raises(ValueError, match="K = 2 gh gw <= 512"):
        grid_flow_fit_torch(x, x, t, x, (120, 160), grid_shapes=((3, 4), (16, 17)), x0=torch.zeros(2, 3, 4))
    with pytest.raises(ValueError, match="x0 or param_ranges"):
        grid_flow_fit_torch(x, x, t, x, (120, 160))
    with pytest.raises(ValueError, match="x0 must have shape"):
        grid_flow_fit_torch(x, x, t, x, (120, 160), x0=torch.zeros(2, 4, 3))
    with pytest.raises(ValueError, match="line_search_steps"):
        grid_flow_fit_torch(x, x, t, x, (120, 160), x0=torch.zeros(2, 3, 4), line_search_steps=33)
    with pytest.raises(ValueError, match="smoothness"):
        grid_flow_fit_torch(x, x, t, x, (120, 160), x0=torch.zeros(2, 3, 4), smoothness=-1.0)
    with pytest.raises(ValueError, match="node grid"):
        grid_flow_fit_torch(x, x, t, x, (12, 16), grid_shapes=((13, 4),), x0=torch.zeros(2, 13, 4))


def test_entry_limits_and_workspace_queries():
    """the queries return 0 for what the entries reject, and the entries reject it with EVK_E_ARG before any CUDA call"""
    from event_utils_b200 import _lib
    L = _lib.load()
    q, qc = L.evk_cmax_grid_flow_objective_workspace_bytes, L.evk_cmax_grid_flow_candidates_workspace_bytes
    assert q(4, 12, 16, 480, 640) == L.evk_cmax_motion_objective_workspace_bytes(4, 480, 640)
    assert q(1, 64, 64, 480, 640) > 0 and q(1, 64, 65, 480, 640) == 0          # gh gw <= 4096
    assert q(1, 1, 4, 12, 16) == 0 and q(1, 13, 4, 12, 16) == 0 and q(1, 3, 17, 12, 16) == 0
    assert q(65535, 2, 2, 4, 4) > 0 and q(65536, 2, 2, 4, 4) == 0 and q(-1, 2, 2, 4, 4) == 0
    assert qc(2, 8, 12, 16, 480, 640) == L.evk_cmax_motion_candidates_workspace_bytes(2, 8, 480, 640)
    assert qc(1, 3, 64, 64, 480, 640) > 0 and qc(1, 4, 64, 64, 480, 640) == 0   # n_cand gh gw <= 12288
    assert qc(1, 32, 16, 24, 480, 640) > 0 and qc(1, 33, 2, 2, 480, 640) == 0 and qc(1, 0, 2, 2, 480, 640) == 0
    assert qc(2047, 32, 2, 2, 4, 4) > 0 and qc(2048, 32, 2, 2, 4, 4) == 0           # batch n_cand <= 65535
    one = ctypes.c_void_p(256)
    ws = ctypes.c_void_p(1 << 20)
    assert L.evk_cmax_grid_flow_objective_f32(one, one, one, one, one, 1, 10, one, 64, 65, 480, 640, 1.0, 0, 0.0, one, one,
                                              ws, 1 << 40, None) == -1
    assert b"gh gw <= 4096" in L.evk_last_error()
    assert L.evk_cmax_grid_flow_objective_grad_f32(one, one, one, one, one, 1, 10, one, 1, 4, 12, 16, 1.0, 0, 0.0, one, one,
                                                   one, ws, 1 << 40, None) == -1
    assert L.evk_cmax_grid_flow_candidates_f32(one, one, one, one, one, 1, 10, one, 4, 64, 64, 480, 640, 1.0, 0, 0.0, one,
                                               ws, 1 << 40, None) == -1
    assert L.evk_cmax_grid_flow_candidates_f32(one, one, one, one, one, 1, 10, one, 2, 3, 4, 12, 16, 1.0, 3, 0.0, one,
                                               ws, 1 << 40, None) == -5   # moa: EVK_E_UNSUPPORTED
    assert L.evk_cmax_grid_flow_objective_f32(one, one, one, one, one, 1, 10, one, 3, 4, 12, 16, 1.0, 0, 0.0, one, one,
                                              ws, 16, None) == -3         # workspace too small


@pytest.mark.parametrize("name", ["evk_cmax_grid_flow_objective_f32", "evk_cmax_grid_flow_objective_grad_f32",
                                  "evk_cmax_grid_flow_candidates_f32"])
def test_bad_blur_sigma_is_rejected_before_any_cuda_call(name):
    """the blur-sigma rule of the other batched entries: NaN is EVK_E_ARG, a radius over 64 EVK_E_UNSUPPORTED"""
    from event_utils_b200 import _lib
    L = _lib.load()
    fn = getattr(L, name)
    fake = ctypes.c_void_p(1 << 20)
    defaults = {ctypes.c_void_p: fake, ctypes.c_int64: 10, ctypes.c_double: 1.0, ctypes.c_int: 4, ctypes.c_size_t: 1 << 40}
    args = [defaults[t] for t in fn.argtypes]
    where = 12 if name != "evk_cmax_grid_flow_candidates_f32" else 13   # after gh, gw, H, W (candidates: and n_cand)
    assert fn.argtypes[where] is ctypes.c_double
    for sigma, rc in ((float("nan"), -1), (16.125, -5), (float("inf"), -5)):
        args[where] = sigma
        assert fn(*args) == rc, (name, sigma)
        assert b"blur sigma" in L.evk_last_error()
