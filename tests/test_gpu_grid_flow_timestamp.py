"""The grid-flow average-timestamp loss, its candidates pass and the coarse-to-fine fit (evk_grid_flow_timestamp_*,
contrast_max/grid_flow_timestamp.py) against the f64 reference of tests/grid_flow_timestamp_reference.py, the dense-flow
timestamp loss through bilinear upsampling, and synthetic windows with known flows."""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import flow_timestamp_reference as FTR
import grid_flow_timestamp_reference as GTR
from conftest import assert_close_to_max
from test_gpu_grid_flow import affine_windows

pytestmark = pytest.mark.gpu


def batch_stream(seed, sizes, H, W, grid, mag, integer=False):
    """concatenated windows with stamps t in [0, 0.1] (sorted per window), d = t - t_last of the window, some NaN
    polarities, and a random node grid (B,2,gh,gw) of up to `mag` px per unit time"""
    rng = np.random.default_rng(seed)
    n = sum(sizes)
    if integer:
        x, y = rng.integers(0, W, n).astype(np.float32), rng.integers(0, H, n).astype(np.float32)
    else:
        x, y = (rng.random(n) * (W - 1)).astype(np.float32), (rng.random(n) * (H - 1)).astype(np.float32)
    p = (rng.integers(0, 2, n) * 2 - 1).astype(np.float32)
    p[::41] = np.nan
    off = np.concatenate(([0], np.cumsum(sizes))).astype(np.int64)
    t = np.concatenate([np.sort(rng.random(s)) * 0.1 for s in sizes]).astype(np.float32)
    d = np.empty(n, np.float32)
    for b in range(len(sizes)):
        if sizes[b]:
            d[off[b]:off[b + 1]] = t[off[b]:off[b + 1]] - t[off[b + 1] - 1]
    g = (rng.standard_normal((len(sizes), 2) + tuple(grid)) * mag).astype(np.float32)
    return x, y, t, d, p, off, g


def cuda(*arrays):
    return [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in arrays]


def run_forward(x, y, d, tau, p, off, grids, H, W, sigma):
    from event_utils_b200 import _lib
    L = _lib.lib()
    B, _, gh, gw = grids.shape
    X, Y, D, U, P, O, G = cuda(x, y, d, tau, p, off, grids)
    f = torch.empty(B, dtype=torch.float64, device="cuda")
    T = torch.empty((B, 2, H + 1, W + 1), device="cuda")
    C = torch.empty((B, 2, H + 1, W + 1), device="cuda")
    ws = torch.empty(L.evk_grid_flow_timestamp_objective_workspace_bytes(B, gh, gw, H, W), dtype=torch.uint8, device="cuda")
    _lib.check(L.evk_grid_flow_timestamp_objective_f32(X.data_ptr(), Y.data_ptr(), D.data_ptr(), U.data_ptr(), P.data_ptr(),
                                                       O.data_ptr(), B, x.shape[0], G.data_ptr(), gh, gw, H, W, sigma,
                                                       f.data_ptr(), T.data_ptr(), C.data_ptr(), ws.data_ptr(), ws.numel(),
                                                       None))
    torch.cuda.synchronize()
    return f.cpu().numpy(), T.cpu().numpy(), C.cpu().numpy()


def torch_loss(x, y, t, p, off, grids, H, W, sigma, reverse=False):
    """grid_flow_timestamp_objective_torch with t0 = each window's last stamp, so that d = t - t_last"""
    from event_utils_b200.contrast_max import grid_flow_timestamp_objective_torch
    g = torch.from_numpy(grids).cuda().requires_grad_(True)
    f = grid_flow_timestamp_objective_torch(*cuda(x, y, t, p), g, (H, W), blur_sigma=sigma, timestamp_reverse=reverse,
                                            batch_end_indices=torch.from_numpy(off[1:]).cuda())
    return f, g


@pytest.mark.parametrize("sigma", [0.0, 1.0, 2.0])
@pytest.mark.parametrize("reverse", [False, True])
@pytest.mark.parametrize("batch", [1, 5])
@pytest.mark.parametrize("grid", [(2, 2), (3, 4), (12, 16)])
def test_f_and_images_against_reference(sigma, reverse, batch, grid):
    H, W = 45, 60
    sizes = [8000] if batch == 1 else [6000, 0, 4000, 8000, 5000]
    x, y, t, d, p, off, g = batch_stream(7 + batch, sizes, H, W, grid, 60.0)
    tau = FTR.tau_f32(t, off, reverse)
    f, T, C = run_forward(x, y, d, tau, p, off, g, H, W, sigma)
    fr, Tr, Cr = (a.detach().numpy() for a in GTR.reference(x, y, d, tau, p, off, torch.from_numpy(g).double(), H, W, sigma))
    for b in range(batch):
        assert_close_to_max(T[b], Tr[b], 1e-5, "T %d" % b)
        assert_close_to_max(C[b], Cr[b], 1e-5, "C %d" % b)
        assert abs(f[b] - fr[b]) <= 1e-5 * max(abs(fr[b]), 1e-30), (b, f[b], fr[b])
    if batch == 5:
        assert (T[1] == 0).all() and (C[1] == 1).all() and f[1] == 0
    # the public function forms d and tau as the reference does
    ft, _ = torch_loss(x, y, t, p, off, g, H, W, sigma, reverse)
    np.testing.assert_allclose(ft.detach().cpu().numpy(), fr, rtol=1e-5)


@pytest.mark.parametrize("sigma", [0.0, 1.0])
@pytest.mark.parametrize("reverse", [False, True])
@pytest.mark.parametrize("grid", [(2, 2), (3, 4), (12, 16)])
def test_gradient_against_reference_and_the_composition(sigma, reverse, grid):
    """the node gradient against autograd through the f64 reference, and, at integer event coordinates, against autograd
    through F.interpolate(align_corners=True) -> flow_timestamp_objective_torch"""
    from event_utils_b200.contrast_max import flow_timestamp_objective_torch
    H, W = 45, 60
    sizes = [6000, 0, 4000, 8000]
    wts = torch.from_numpy(np.random.default_rng(5).standard_normal(len(sizes)))
    for integer in (False, True):
        x, y, t, d, p, off, g = batch_stream(3, sizes, H, W, grid, 60.0, integer)
        f, gg = torch_loss(x, y, t, p, off, g, H, W, sigma, reverse)
        (f * wts.cuda()).sum().backward()
        got = gg.grad.cpu().numpy().astype(np.float64)
        tau = FTR.tau_f32(t, off, reverse)
        g64 = torch.from_numpy(g).double().requires_grad_(True)
        fr, _, _ = GTR.reference(x, y, d, tau, p, off, g64, H, W, sigma)
        (fr * wts).sum().backward()
        assert_close_to_max(got, g64.grad.numpy(), 1e-4, "grad sigma %g grid %s" % (sigma, grid))
        assert (got[1] == 0).all()
        if integer:
            gc = torch.from_numpy(g).cuda().requires_grad_(True)
            dense = F.interpolate(gc, (H, W), mode="bilinear", align_corners=True)
            fd = flow_timestamp_objective_torch(*cuda(x, y, t, p), dense, blur_sigma=sigma, timestamp_reverse=reverse,
                                                batch_end_indices=torch.from_numpy(off[1:]).cuda())
            (fd * wts.cuda()).sum().backward()
            np.testing.assert_allclose(f.detach().cpu().numpy(), fd.detach().cpu().numpy(), rtol=1e-5)
            assert_close_to_max(got, gc.grad.cpu().numpy(), 1e-4, "composition sigma %g grid %s" % (sigma, grid))


@pytest.mark.parametrize("grid,J", [((2, 2), 32), ((3, 4), 7), ((12, 16), 7), ((48, 64), 7)])
def test_candidates_equal_the_forward(grid, J):
    """J up to the node limit: 32 candidates of a 2 x 2 grid in one pass, and 4 per pass of a 48 x 64 grid"""
    from event_utils_b200.contrast_max import grid_flow_timestamp_candidates_torch
    H, W = 60, 80
    sizes = [9000, 0, 7000]
    x, y, t, d, p, off, _ = batch_stream(11, sizes, H, W, grid, 40.0)
    cand = (np.random.default_rng(12).standard_normal((len(sizes), J, 2) + grid) * 40.0).astype(np.float32)
    fc = grid_flow_timestamp_candidates_torch(*cuda(x, y, t, p), torch.from_numpy(cand).cuda(), (H, W), blur_sigma=1.0,
                                              batch_end_indices=torch.from_numpy(off[1:]).cuda())
    assert fc.shape == (len(sizes), J) and fc.dtype == torch.float64
    tau = FTR.tau_f32(t, off)
    for j in range(J):
        f, _, _ = run_forward(x, y, d, tau, p, off, np.ascontiguousarray(cand[:, j]), H, W, 1.0)
        np.testing.assert_allclose(fc[:, j].cpu().numpy(), f, rtol=1e-6)


def exact_stream(H, W, sizes, grid, seed=0):
    """integer events, node ratios that are powers of 2, a uniform node grid of multiples of 8 and d multiples of 1/16:
    every interpolated flow is exact, every warped position a multiple of 1/2 and every bilinear weight dyadic, so every
    count image sum is exact in f32 whatever the order of the additions"""
    rng = np.random.default_rng(seed)
    n = sum(sizes)
    x, y = rng.integers(4, W - 4, n).astype(np.float32), rng.integers(4, H - 4, n).astype(np.float32)
    p = (rng.integers(0, 2, n) * 2 - 1).astype(np.float32)
    off = np.concatenate(([0], np.cumsum(sizes))).astype(np.int64)
    t = np.concatenate([np.sort(rng.integers(0, 3, s)) / 16.0 for s in sizes]).astype(np.float32)
    d = np.empty(n, np.float32)
    for b in range(len(sizes)):
        if sizes[b]:
            d[off[b]:off[b + 1]] = t[off[b]:off[b + 1]] - t[off[b + 1] - 1]
    g = (rng.integers(-4, 5, (len(sizes), 2, 1, 1)) * 8.0 * np.ones((1, 1) + grid)).astype(np.float32)
    return x, y, t, d, p, off, g


def test_counts_are_exact_on_exactly_summable_streams():
    H, W = 17, 33
    x, y, t, d, p, off, g = exact_stream(H, W, [20000, 0, 15000], (3, 5))
    tau = FTR.tau_f32(t, off)
    f, T, C = run_forward(x, y, d, tau, p, off, g, H, W, 0.0)
    fr, Tr, Cr = GTR.reference(x, y, d, tau, p, off, torch.from_numpy(g).double(), H, W, 0.0)
    assert (C == Cr.numpy().astype(np.float32)).all()
    assert_close_to_max(T, Tr.numpy(), 1e-6)
    np.testing.assert_allclose(f, fr.numpy(), rtol=1e-6)


def test_chunking_empty_and_nan_windows(monkeypatch):
    """window chunks and candidate passes change no value beyond the order of the f32 atomics, an empty window has zero
    gradient, a NaN node makes only its window's f NaN, and a candidate that warps an event to a non-finite position
    makes only its own f NaN"""
    from event_utils_b200.contrast_max import grid_flow_timestamp as GFT
    H, W = 17, 33
    sizes = [9000, 0, 7000, 8000]
    x, y, t, d, p, off, g = exact_stream(H, W, sizes, (3, 5), seed=1)
    cand = np.stack([g + 8.0 * j for j in range(40)], 1)
    args = cuda(x, y, t, p)
    ends = torch.from_numpy(off[1:]).cuda()
    kw = dict(blur_sigma=0.0, batch_end_indices=ends)
    f_all = GFT.grid_flow_timestamp_candidates_torch(*args, torch.from_numpy(cand).cuda(), (H, W), **kw)
    monkeypatch.setattr(GFT, "TIMESTAMP_CANDIDATES_WORKSPACE_BYTES", 1)     # one window per call
    f_one = GFT.grid_flow_timestamp_candidates_torch(*args, torch.from_numpy(cand).cuda(), (H, W), **kw)
    torch.testing.assert_close(f_all, f_one, rtol=1e-6, atol=0)
    f64, _, _ = run_forward(x, y, d, FTR.tau_f32(t, off), p, off, g, H, W, 0.0)
    np.testing.assert_allclose(f_all[:, 0].cpu().numpy(), f64, rtol=1e-6)
    f, gg = torch_loss(x, y, t, p, off, g, H, W, 0.0)
    f.sum().backward()
    assert (gg.grad[1] == 0).all() and torch.isfinite(gg.grad).all()
    bad = g.copy()
    bad[2, 0, 1, 1] = np.nan
    fb, gb = torch_loss(x, y, t, p, off, bad, H, W, 0.0)
    fb.sum().backward()
    fb = fb.detach().cpu()
    assert torch.isnan(fb[2]) and torch.isfinite(fb[[0, 1, 3]]).all()
    torch.testing.assert_close(fb[[0, 1, 3]], f.detach().cpu()[[0, 1, 3]], rtol=1e-6, atol=0)
    assert_close_to_max(gb.grad[[0, 1, 3]].cpu().numpy(), gg.grad[[0, 1, 3]].cpu().numpy(), 1e-6)
    cb = cand[:, :3].copy()
    cb[2, 1, 0, 1, 1] = np.nan
    fc = GFT.grid_flow_timestamp_candidates_torch(*args, torch.from_numpy(cb).cuda(), (H, W), **kw).cpu()
    assert torch.isnan(fc[2, 1]) and torch.isfinite(fc[[0, 1, 3]]).all() and torch.isfinite(fc[2, [0, 2]]).all()


def test_no_host_round_trips_and_constant_launch_count():
    from event_utils_b200 import _lib
    from event_utils_b200.contrast_max import grid_flow_timestamp_candidates_torch, grid_flow_timestamp_objective_torch
    L = _lib.lib()
    H, W = 60, 80
    counts = []
    for sizes in ([40000], [2500] * 16):
        x, y, t, d, p, off, g = batch_stream(2, sizes, H, W, (6, 8), 40.0)
        torch_loss(x, y, t, p, off, g, H, W, 1.0)     # warm-up
        gt = torch.from_numpy(g).cuda().requires_grad_(True)
        cand = torch.from_numpy(g).cuda().unsqueeze(1).repeat(1, 5, 1, 1, 1)
        ev = cuda(x, y, t, p)
        ends = torch.from_numpy(off[1:]).cuda()
        grid_flow_timestamp_candidates_torch(*ev, cand, (H, W), batch_end_indices=ends)
        torch.cuda.synchronize()
        L.evk_prof_enable(1)
        torch.cuda.set_sync_debug_mode("error")
        try:
            f = grid_flow_timestamp_objective_torch(*ev, gt, (H, W), batch_end_indices=ends)
            f.sum().backward()
            grid_flow_timestamp_candidates_torch(*ev, cand, (H, W), batch_end_indices=ends)
        finally:
            torch.cuda.set_sync_debug_mode(0)
        ms, timed, launches = ctypes.c_double(), ctypes.c_longlong(), ctypes.c_longlong()
        _lib.check(L.evk_prof_collect(ctypes.byref(ms), ctypes.byref(timed), ctypes.byref(launches)))
        L.evk_prof_enable(0)
        assert torch.isfinite(gt.grad).all()
        counts.append(launches.value)
    assert counts[0] == counts[1] and counts[0] > 0, counts


def test_limits():
    """batch n_cand = 32767 canvases (two tail images each), and the node limits of the loss (gh gw = 4096) and of a
    candidates pass (n_cand gh gw = 12288)"""
    from event_utils_b200.contrast_max import grid_flow_timestamp_candidates_torch
    rng = np.random.default_rng(8)
    H, W = 6, 8
    B, J = 1057, 31                                     # 1057 x 31 = 32767
    per = 3
    x, y = (rng.random(B * per) * (W - 1)).astype(np.float32), (rng.random(B * per) * (H - 1)).astype(np.float32)
    t = (np.sort(rng.random((B, per)), 1).reshape(-1) * 0.1).astype(np.float32)
    p = np.ones(B * per, np.float32)
    off = np.arange(0, B * per + 1, per, dtype=np.int64)
    d = (t - np.repeat(t[off[1:] - 1], per)).astype(np.float32)
    cand = (rng.standard_normal((B, J, 2, 2, 2)) * 5).astype(np.float32)
    fc = grid_flow_timestamp_candidates_torch(*cuda(x, y, t, p), torch.from_numpy(cand).cuda(), (H, W),
                                              batch_end_indices=torch.from_numpy(off[1:]).cuda()).cpu().numpy()
    tau = FTR.tau_f32(t, off)
    for b in (0, 567, B - 1):
        sl = slice(off[b], off[b + 1])
        for j in (0, J - 1):
            f, _, _ = run_forward(x[sl], y[sl], d[sl], tau[sl], p[sl], np.array([0, per], np.int64),
                                  np.ascontiguousarray(cand[b:b + 1, j]), H, W, 2.0)
            np.testing.assert_allclose(fc[b, j], f[0], rtol=1e-6)
    # the node limits: a 64 x 64 grid on a 64 x 64 sensor (the dense flow), forward and gradient; 4 candidates of a 48 x 64
    # grid in one pass
    H = W = 64
    x, y, t, d, p, off, g = batch_stream(9, [20000, 10000], H, W, (64, 64), 20.0)
    f, gg = torch_loss(x, y, t, p, off, g, H, W, 1.0)
    f.sum().backward()
    tau = FTR.tau_f32(t, off)
    g64 = torch.from_numpy(g).double().requires_grad_(True)
    fr, _, _ = GTR.reference(x, y, d, tau, p, off, g64, H, W, 1.0)
    fr.sum().backward()
    np.testing.assert_allclose(f.detach().cpu().numpy(), fr.detach().numpy(), rtol=1e-5)
    assert_close_to_max(gg.grad.cpu().numpy(), g64.grad.numpy(), 1e-4)
    g48 = g[:, :, :48, :]
    cand = np.stack([g48, g48 * 0.5, g48 * -1.0, g48 * 0.25], 1)
    fc = grid_flow_timestamp_candidates_torch(*cuda(x, y, t, p), torch.from_numpy(cand).cuda(), (H, W), blur_sigma=1.0,
                                              batch_end_indices=torch.from_numpy(off[1:]).cuda())
    for j in range(4):
        fj, _, _ = run_forward(x, y, d, tau, p, off, np.ascontiguousarray(cand[:, j]), H, W, 1.0)
        np.testing.assert_allclose(fc[:, j].cpu().numpy(), fj, rtol=1e-6)


@pytest.mark.parametrize("reverse", [False, True])
def test_fit_recovers_affine_flows(reverse):
    """The affine-flow windows of test_gpu_grid_flow.py, the contrast fit's tolerance: RMS node error x window length
    <= 1.5 px on at least B - 1 of B windows, and every miss at F <= F(truth), with the default smoothness (1e-2, chosen
    on these windows: the bounded fit recovered all 8 within 0.6 px, with either stamp order)."""
    from event_utils_b200.contrast_max import (charbonnier_smoothness, grid_flow_timestamp_fit_torch,
                                              grid_flow_timestamp_objective_torch)
    H, W = 90, 120
    B = 8
    ev, ends, truth = affine_windows(21, B, 30000, H, W)
    fit = grid_flow_timestamp_fit_torch(*ev, (H, W), grid_shapes=((3, 4), (6, 8)), batch_end_indices=ends,
                                        param_ranges=[[-80, 80], [-80, 80]], max_iter=40, blur_sigma=1.0,
                                        timestamp_reverse=reverse)
    assert fit.flow.shape == (B, 2, 6, 8) and fit.flow.dtype == torch.float64
    lam = 1e-2
    tr = torch.from_numpy(truth(6, 8)).cuda()
    f_truth = grid_flow_timestamp_objective_torch(*ev, tr, (H, W), blur_sigma=1.0, timestamp_reverse=reverse,
                                                  batch_end_indices=ends).double()
    F_truth = f_truth + lam * charbonnier_smoothness(tr, 1.0)[0]
    err = (fit.flow - tr).pow(2).mean((1, 2, 3)).sqrt()
    hit = err * 0.1 <= 1.5
    assert int(hit.sum()) >= B - 1, (err, fit.status, fit.f, F_truth)
    assert bool((hit | (fit.f <= F_truth)).all()), (err, fit.f, F_truth)
    np.testing.assert_allclose(fit.loss.cpu().numpy(), (fit.f - lam * charbonnier_smoothness(fit.flow, 1.0)[0]).cpu().numpy())


def test_bounded_fit_never_leaves_its_box():
    """per-window boxes, from x0 and from the global start: every node of every stage's result lies in its box"""
    from event_utils_b200.contrast_max import grid_flow_timestamp_fit_torch
    H, W = 90, 120
    B = 4
    ev, ends, _ = affine_windows(23, B, 20000, H, W)
    box = torch.tensor([[[-20.0, 5.0], [-3.0, 30.0]]], dtype=torch.float64).repeat(B, 1, 1)
    box[1] = torch.tensor([[0.0, 1.0], [-1.0, 0.0]])
    for kw in (dict(x0=torch.zeros(2, 3, 4)), dict(param_ranges=[[-80, 80], [-80, 80]])):
        for shapes in (((3, 4),), ((3, 4), (6, 8))):
            fit = grid_flow_timestamp_fit_torch(*ev, (H, W), grid_shapes=shapes, batch_end_indices=ends, bounds=box,
                                                max_iter=20, blur_sigma=1.0, **kw)
            lo, hi = box[..., 0].cuda().view(B, 2, 1, 1), box[..., 1].cuda().view(B, 2, 1, 1)
            assert bool(((fit.flow >= lo) & (fit.flow <= hi)).all()), (kw, shapes)
            assert torch.isfinite(fit.f).all()


def test_fit_beats_the_global_fit_on_two_objects():
    from event_utils_b200.contrast_max import grid_flow_timestamp_fit_torch, linvel_warp, motion_timestamp_fit_torch
    H, W = 90, 120
    B = 6
    ev, ends, _ = affine_windows(22, B, 30000, H, W, two_objects=True)
    ranges = [[-80, 80], [-80, 80]]
    lin = motion_timestamp_fit_torch(*ev, linvel_warp(), ends, img_size=(H, W), param_ranges=ranges, max_iter=40)
    fit = grid_flow_timestamp_fit_torch(*ev, (H, W), grid_shapes=((3, 4), (6, 8)), smoothness=1e-2, batch_end_indices=ends,
                                        param_ranges=ranges, max_iter=40)
    assert bool((fit.loss < lin.f).all()), (fit.loss, lin.f)
