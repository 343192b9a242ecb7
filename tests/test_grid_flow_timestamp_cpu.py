"""No-GPU checks of the grid-flow average-timestamp loss and fit (contrast_max/grid_flow_timestamp.py): the f64 reference
of tests/grid_flow_timestamp_reference.py against the dense-flow timestamp reference, the argument checks that run
before any CUDA call, and the C entries' limits and workspace queries."""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import flow_timestamp_reference as FTR
import grid_flow_timestamp_reference as GTR


def stream(seed, sizes, H, W, integer):
    rng = np.random.default_rng(seed)
    n = sum(sizes)
    if integer:
        x, y = rng.integers(0, W, n).astype(np.float32), rng.integers(0, H, n).astype(np.float32)
    else:
        x, y = (rng.random(n) * (W - 1)).astype(np.float32), (rng.random(n) * (H - 1)).astype(np.float32)
    p = (rng.integers(0, 2, n) * 2 - 1).astype(np.float32)
    p[::37] = np.nan                                       # dropped from both images
    off = np.concatenate(([0], np.cumsum(sizes))).astype(np.int64)
    t = np.concatenate([np.sort(rng.random(s)) for s in sizes]).astype(np.float32)
    d = (t - 1.0).astype(np.float32)
    return x, y, d, FTR.tau_f32(t, off), p, off


@pytest.mark.parametrize("sigma", [0.0, 1.0])
@pytest.mark.parametrize("grid", [(2, 2), (3, 4), (5, 7)])
def test_reference_equals_dense_reference_on_the_interpolated_flow(sigma, grid):
    """integer event coordinates: f, T, C and the gradient of the grid reference equal the dense-flow timestamp
    reference's on F.interpolate(grid, (H, W), bilinear, align_corners=True), the gradient through that composition"""
    H, W = 12, 16
    x, y, d, tau, p, off = stream(1, [400, 300], H, W, True)
    g0 = torch.from_numpy(np.random.default_rng(2).standard_normal((2, 2) + grid) * 6.0)
    g1 = g0.clone().requires_grad_(True)
    f, T, C = GTR.reference(x, y, d, tau, p, off, g1, H, W, sigma)
    f.sum().backward()
    g2 = g0.clone().requires_grad_(True)
    dense = F.interpolate(g2, (H, W), mode="bilinear", align_corners=True)
    fd, Td, Cd = FTR.reference(x, y, d, tau, p, off, dense, sigma)
    fd.sum().backward()
    np.testing.assert_allclose(f.detach().numpy(), fd.detach().numpy(), rtol=1e-5)
    np.testing.assert_allclose(T.detach().numpy(), Td.detach().numpy(), atol=1e-5)
    np.testing.assert_allclose(C.detach().numpy(), Cd.detach().numpy(), atol=1e-4)
    np.testing.assert_allclose(g1.grad.numpy(), g2.grad.numpy(), rtol=1e-4, atol=1e-6 * np.abs(g2.grad.numpy()).max())


def test_full_resolution_grid_is_the_dense_flow():
    """gh = H, gw = W: the grid reference is the dense-flow timestamp reference on the same field, at any coordinates"""
    H, W = 9, 11
    x, y, d, tau, p, off = stream(3, [500], H, W, False)
    g = torch.from_numpy(np.random.default_rng(4).standard_normal((1, 2, H, W)) * 5.0)
    f, T, C = GTR.reference(x, y, d, tau, p, off, g, H, W, 0.0)
    fd, Td, Cd = FTR.reference(x, y, d, tau, p, off, g, 0.0)
    np.testing.assert_allclose(f.numpy(), fd.numpy(), rtol=1e-6)
    np.testing.assert_allclose(T.numpy(), Td.numpy(), atol=1e-6)
    np.testing.assert_allclose(C.numpy(), Cd.numpy(), atol=1e-5)


def test_argument_checks_run_before_any_cuda_call():
    from event_utils_b200.contrast_max import (grid_flow_timestamp_candidates_torch, grid_flow_timestamp_fit_torch,
                                              grid_flow_timestamp_objective_torch)
    x = torch.zeros(8)
    t = torch.arange(8.0)
    nan = float("nan")
    with pytest.raises(ValueError, match="node grid"):
        grid_flow_timestamp_objective_torch(x, x, t, x, torch.zeros(2, 13, 4), (12, 16))
    with pytest.raises(ValueError, match="node grid"):
        grid_flow_timestamp_objective_torch(x, x, t, x, torch.zeros(2, 65, 65), (100, 100))
    with pytest.raises(ValueError, match="shape"):
        grid_flow_timestamp_objective_torch(x, x, t, x, torch.zeros(3, 3, 4), (12, 16))
    with pytest.raises(ValueError, match="blur_sigma"):
        grid_flow_timestamp_objective_torch(x, x, t, x, torch.zeros(2, 3, 4), (12, 16), blur_sigma=nan)
    with pytest.raises(ValueError, match="must not require grad"):
        grid_flow_timestamp_objective_torch(x.requires_grad_(True), x, t, x, torch.zeros(2, 3, 4), (12, 16))
    x = torch.zeros(8)
    with pytest.raises(ValueError, match="shape"):
        grid_flow_timestamp_candidates_torch(x, x, t, x, torch.zeros(1, 2, 3, 4), (12, 16))
    with pytest.raises(ValueError, match="node grid"):
        grid_flow_timestamp_candidates_torch(x, x, t, x, torch.zeros(1, 3, 2, 3, 17), (12, 16))
    with pytest.raises(ValueError, match="blur_sigma"):
        grid_flow_timestamp_candidates_torch(x, x, t, x, torch.zeros(1, 3, 2, 3, 4), (12, 16), blur_sigma=nan)
    fit = grid_flow_timestamp_fit_torch
    with pytest.raises(ValueError, match="K = 2 gh gw <= 512"):
        fit(x, x, t, x, (120, 160), grid_shapes=((3, 4), (16, 17)), x0=torch.zeros(2, 3, 4))
    with pytest.raises(ValueError, match="x0 or param_ranges"):
        fit(x, x, t, x, (120, 160))
    with pytest.raises(ValueError, match="x0 must have shape"):
        fit(x, x, t, x, (120, 160), x0=torch.zeros(2, 4, 3))
    with pytest.raises(ValueError, match="bounds must have shape"):
        fit(x, x, t, x, (120, 160), x0=torch.zeros(2, 3, 4), bounds=[[-1.0, 1.0]])
    with pytest.raises(ValueError, match="bounds must have shape"):
        fit(x, x, t, x, (120, 160), param_ranges=[[-1, 1], [-1, 1]], bounds=np.zeros((3, 2, 2)))
    with pytest.raises(ValueError, match="line_search_steps"):
        fit(x, x, t, x, (120, 160), x0=torch.zeros(2, 3, 4), line_search_steps=33)
    with pytest.raises(ValueError, match="smoothness"):
        fit(x, x, t, x, (120, 160), x0=torch.zeros(2, 3, 4), smoothness=-1.0)
    with pytest.raises(ValueError, match="node grid"):
        fit(x, x, t, x, (12, 16), grid_shapes=((13, 4),), x0=torch.zeros(2, 13, 4))
    with pytest.raises(ValueError, match="blur_sigma"):
        fit(x, x, t, x, (120, 160), x0=torch.zeros(2, 3, 4), blur_sigma=[2.0, nan])


def test_entry_limits_and_workspace_queries():
    """the queries return 0 for what the entries reject, and the entries reject it with EVK_E_ARG before any CUDA call"""
    from event_utils_b200 import _lib
    L = _lib.load()
    q, qc = L.evk_grid_flow_timestamp_objective_workspace_bytes, L.evk_grid_flow_timestamp_candidates_workspace_bytes
    assert q(4, 12, 16, 480, 640) == L.evk_flow_timestamp_objective_workspace_bytes(4, 480, 640)
    assert q(1, 64, 64, 480, 640) > 0 and q(1, 64, 65, 480, 640) == 0          # gh gw <= 4096
    assert q(1, 1, 4, 12, 16) == 0 and q(1, 13, 4, 12, 16) == 0 and q(1, 3, 17, 12, 16) == 0
    assert q(32767, 2, 2, 4, 4) > 0 and q(32768, 2, 2, 4, 4) == 0 and q(-1, 2, 2, 4, 4) == 0   # two images per window
    assert qc(2, 8, 12, 16, 480, 640) == L.evk_motion_timestamp_candidates_workspace_bytes(2, 8, 480, 640)
    assert qc(1, 3, 64, 64, 480, 640) > 0 and qc(1, 4, 64, 64, 480, 640) == 0   # n_cand gh gw <= 12288
    assert qc(1, 32, 16, 24, 480, 640) > 0 and qc(1, 33, 2, 2, 480, 640) == 0 and qc(1, 0, 2, 2, 480, 640) == 0
    assert qc(1023, 32, 2, 2, 4, 4) > 0 and qc(1024, 32, 2, 2, 4, 4) == 0           # batch n_cand <= 32767
    assert qc(32767, 1, 2, 2, 4, 4) > 0 and qc(32768, 1, 2, 2, 4, 4) == 0
    one = ctypes.c_void_p(256)
    ws = ctypes.c_void_p(1 << 20)
    assert L.evk_grid_flow_timestamp_objective_f32(one, one, one, one, one, one, 1, 10, one, 64, 65, 480, 640, 1.0, one,
                                                   one, one, ws, 1 << 40, None) == -1
    assert b"gh gw <= 4096" in L.evk_last_error()
    assert L.evk_grid_flow_timestamp_objective_f32(one, one, one, one, one, one, 32768, 10, one, 2, 2, 4, 4, 1.0, one,
                                                   one, one, ws, 1 << 40, None) == -1
    assert b"batch <= 32767" in L.evk_last_error()
    assert L.evk_grid_flow_timestamp_objective_f32(one, one, one, None, one, one, 1, 10, one, 3, 4, 12, 16, 1.0, one,
                                                   one, one, ws, 1 << 40, None) == -1       # no tau
    assert L.evk_grid_flow_timestamp_objective_grad_f32(one, one, one, one, one, one, 1, 10, one, 1, 4, 12, 16, 1.0, one,
                                                        one, one, one, ws, 1 << 40, None) == -1
    assert L.evk_grid_flow_timestamp_candidates_f32(one, one, one, one, one, one, 1, 10, one, 4, 64, 64, 480, 640, 1.0,
                                                    one, ws, 1 << 40, None) == -1
    assert L.evk_grid_flow_timestamp_candidates_f32(one, one, one, one, one, one, 1024, 10, one, 32, 2, 2, 4, 4, 1.0,
                                                    one, ws, 1 << 40, None) == -1
    assert L.evk_grid_flow_timestamp_objective_f32(one, one, one, one, one, one, 1, 10, one, 3, 4, 12, 16, 1.0, one, one,
                                                   one, ws, 16, None) == -3         # workspace too small
    need = qc(2, 3, 3, 4, 12, 16)
    assert L.evk_grid_flow_timestamp_candidates_f32(one, one, one, one, one, one, 2, 10, one, 3, 3, 4, 12, 16, 1.0, one,
                                                    ws, need - 1, None) == -3


@pytest.mark.parametrize("name", ["evk_grid_flow_timestamp_objective_f32", "evk_grid_flow_timestamp_objective_grad_f32",
                                  "evk_grid_flow_timestamp_candidates_f32"])
def test_bad_blur_sigma_is_rejected_before_any_cuda_call(name):
    """the blur-sigma rule of the other batched entries: NaN is EVK_E_ARG, a radius over 64 EVK_E_UNSUPPORTED"""
    from event_utils_b200 import _lib
    L = _lib.load()
    fn = getattr(L, name)
    fake = ctypes.c_void_p(1 << 20)
    defaults = {ctypes.c_void_p: fake, ctypes.c_int64: 10, ctypes.c_double: 1.0, ctypes.c_int: 4, ctypes.c_size_t: 1 << 40}
    args = [defaults[t] for t in fn.argtypes]
    where = 13 if name != "evk_grid_flow_timestamp_candidates_f32" else 14   # after gh, gw, H, W (candidates: and n_cand)
    assert fn.argtypes[where] is ctypes.c_double
    for sigma, rc in ((float("nan"), -1), (16.125, -5), (float("inf"), -5)):
        args[where] = sigma
        assert fn(*args) == rc, (name, sigma)
        assert b"blur sigma" in L.evk_last_error()
