"""The grid-flow contrast loss, its candidates pass and the coarse-to-fine fit (evk_cmax_grid_flow_*, contrast_max/grid_flow.py)
against the f64 reference of tests/grid_flow_reference.py, the dense-flow loss through bilinear upsampling, and synthetic
windows with known flows."""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import grid_flow_reference as GR
from conftest import assert_close_to_max

pytestmark = pytest.mark.gpu

OBJ = {"variance": 0, "sos": 1, "soe": 2, "sosa": 5}


def batch_stream(seed, sizes, H, W, grid, mag, integer=False):
    """concatenated windows, d = t - t0 in [-0.1, 0], and a random node grid (B,2,gh,gw) of up to `mag` px per unit time"""
    rng = np.random.default_rng(seed)
    n = sum(sizes)
    if integer:
        x, y = rng.integers(0, W, n).astype(np.float32), rng.integers(0, H, n).astype(np.float32)
    else:
        x, y = (rng.random(n) * (W - 1)).astype(np.float32), (rng.random(n) * (H - 1)).astype(np.float32)
    p = (rng.integers(0, 2, n) * 2 - 1).astype(np.float32)
    off = np.concatenate(([0], np.cumsum(sizes))).astype(np.int64)
    d = np.empty(n, np.float32)
    for b in range(len(sizes)):
        d[off[b]:off[b + 1]] = -np.sort(rng.random(sizes[b]))[::-1] * 0.1
    g = (rng.standard_normal((len(sizes), 2) + tuple(grid)) * mag).astype(np.float32)
    return x, y, d, p, off, g


def cuda(*arrays):
    return [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in arrays]


def run_forward(x, y, d, p, off, grids, H, W, sigma, name, param=3.0):
    from event_utils_b200 import _lib
    L = _lib.lib()
    B, _, gh, gw = grids.shape
    X, Y, D, P, O, G = cuda(x, y, d, p, off, grids)
    f = torch.empty(B, dtype=torch.float64, device="cuda")
    iwe = torch.empty((B, H + 1, W + 1), device="cuda")
    ws = torch.empty(L.evk_cmax_grid_flow_objective_workspace_bytes(B, gh, gw, H, W), dtype=torch.uint8, device="cuda")
    _lib.check(L.evk_cmax_grid_flow_objective_f32(X.data_ptr(), Y.data_ptr(), D.data_ptr(), P.data_ptr(), O.data_ptr(), B,
                                                  x.shape[0], G.data_ptr(), gh, gw, H, W, sigma, OBJ[name], param, f.data_ptr(),
                                                  iwe.data_ptr(), ws.data_ptr(), ws.numel(), None))
    torch.cuda.synchronize()
    return f.cpu().numpy(), iwe.cpu().numpy()


def torch_loss(x, y, d, p, off, grids, H, W, sigma, name, param=3.0):
    """grid_flow_contrast_objective_torch with ts = d and t0 = 0, so that d reaches the kernel unchanged"""
    from event_utils_b200.contrast_max import grid_flow_contrast_objective_torch
    g = torch.from_numpy(grids).cuda().requires_grad_(True)
    f = grid_flow_contrast_objective_torch(*cuda(x, y, d, p), g, (H, W), t0=0.0, objective=name, blur_sigma=sigma,
                                           obj_param=param, batch_end_indices=torch.from_numpy(off[1:]).cuda())
    return f, g


GRIDS = [((45, 60), (2, 2)), ((45, 60), (3, 4)), ((45, 60), (12, 16)), ((12, 16), (12, 16))]


@pytest.mark.parametrize("name", ["variance", "sos", "soe", "sosa"])
@pytest.mark.parametrize("sigma", [0.0, 1.0, 3.0])
@pytest.mark.parametrize("batch", [1, 5])
@pytest.mark.parametrize("size,grid", GRIDS)
def test_f_and_iwe_against_reference(name, sigma, batch, size, grid):
    H, W = size
    sizes = [8000] if batch == 1 else [6000, 0, 4000, 8000, 5000]
    x, y, d, p, off, g = batch_stream(7 + batch, sizes, H, W, grid, 30.0)
    param = 0.3
    f, iwe = run_forward(x, y, d, p, off, g, H, W, sigma, name, param)
    fr, iwer = GR.reference(x, y, d, p, off, torch.from_numpy(g).double(), H, W, sigma, name, param)
    fr, iwer = fr.detach().numpy(), iwer.detach().numpy()
    for b in range(batch):
        assert_close_to_max(iwe[b], iwer[b], 1e-5, "iwe %d" % b)
        assert abs(f[b] - fr[b]) <= 1e-5 * max(abs(fr[b]), 1e-30), (b, f[b], fr[b])
    if batch == 5:
        assert (iwe[1] == 0).all()
    if grid == size:
        # the full-resolution grid is the dense flow
        from event_utils_b200.contrast_max import flow_contrast_objective_torch
        fd = flow_contrast_objective_torch(*cuda(x, y, d, p), torch.from_numpy(g).cuda(), t0=0.0, objective=name,
                                           blur_sigma=sigma, obj_param=param, batch_end_indices=torch.from_numpy(off[1:]).cuda())
        np.testing.assert_allclose(f, fd.cpu().numpy(), rtol=1e-5)


@pytest.mark.parametrize("name", ["variance", "sos", "soe", "sosa"])
@pytest.mark.parametrize("sigma", [0.0, 1.0])
@pytest.mark.parametrize("grid", [(2, 2), (3, 4), (12, 16)])
def test_gradient_against_reference_and_the_composition(name, sigma, grid):
    """the node gradient against autograd through the f64 reference, and, at integer event coordinates, against autograd
    through F.interpolate(align_corners=True) -> flow_contrast_objective_torch"""
    from event_utils_b200.contrast_max import flow_contrast_objective_torch
    H, W = 45, 60
    sizes = [6000, 0, 4000, 8000]
    wts = torch.from_numpy(np.random.default_rng(5).standard_normal(len(sizes)))
    for integer in (False, True):
        x, y, d, p, off, g = batch_stream(3, sizes, H, W, grid, 30.0, integer)
        f, gg = torch_loss(x, y, d, p, off, g, H, W, sigma, name, 0.3)
        (f * wts.cuda()).sum().backward()
        got = gg.grad.cpu().numpy().astype(np.float64)
        g64 = torch.from_numpy(g).double().requires_grad_(True)
        fr, _ = GR.reference(x, y, d, p, off, g64, H, W, sigma, name, 0.3)
        (fr * wts).sum().backward()
        assert_close_to_max(got, g64.grad.numpy(), 1e-4, "grad %s sigma %g grid %s" % (name, sigma, grid))
        assert (got[1] == 0).all()
        if integer:
            gc = torch.from_numpy(g).cuda().requires_grad_(True)
            dense = F.interpolate(gc, (H, W), mode="bilinear", align_corners=True)
            fd = flow_contrast_objective_torch(*cuda(x, y, d, p), dense, t0=0.0, objective=name, blur_sigma=sigma,
                                               obj_param=0.3, batch_end_indices=torch.from_numpy(off[1:]).cuda())
            (fd * wts.cuda()).sum().backward()
            np.testing.assert_allclose(f.detach().cpu().numpy(), fd.detach().cpu().numpy(), rtol=1e-5)
            assert_close_to_max(got, gc.grad.cpu().numpy(), 1e-4, "composition %s sigma %g grid %s" % (name, sigma, grid))


@pytest.mark.parametrize("grid", [(3, 4), (12, 16), (48, 64)])
def test_candidates_equal_the_forward(grid):
    from event_utils_b200.contrast_max import grid_flow_contrast_candidates_torch
    H, W = 60, 80
    sizes = [9000, 0, 7000]
    J = 7
    x, y, d, p, off, _ = batch_stream(11, sizes, H, W, grid, 20.0)
    cand = (np.random.default_rng(12).standard_normal((len(sizes), J, 2) + grid) * 20.0).astype(np.float32)
    fc = grid_flow_contrast_candidates_torch(*cuda(x, y, d, p), torch.from_numpy(cand).cuda(), (H, W), t0=0.0,
                                             objective="soe", batch_end_indices=torch.from_numpy(off[1:]).cuda())
    assert fc.shape == (len(sizes), J) and fc.dtype == torch.float64
    for j in range(J):
        f, _ = run_forward(x, y, d, p, off, np.ascontiguousarray(cand[:, j]), H, W, 1.0, "soe")
        np.testing.assert_allclose(fc[:, j].cpu().numpy(), f, rtol=1e-6)


def exact_stream(H, W, sizes, grid, seed=0):
    """integer events, node ratios (gw-1)/(W-1), (gh-1)/(H-1) that are powers of 2, a uniform node grid of multiples of 8
    and d multiples of 1/16: every interpolated flow is exact, every warped position a multiple of 1/2 and every bilinear
    weight dyadic, so every IWE sum is exact in f32 whatever the order of the additions"""
    rng = np.random.default_rng(seed)
    n = sum(sizes)
    x, y = rng.integers(4, W - 4, n).astype(np.float32), rng.integers(4, H - 4, n).astype(np.float32)
    p = (rng.integers(0, 2, n) * 2 - 1).astype(np.float32)
    d = (-rng.integers(0, 3, n) / 16.0).astype(np.float32)
    off = np.concatenate(([0], np.cumsum(sizes))).astype(np.int64)
    g = (rng.integers(-4, 5, (len(sizes), 2, 1, 1)) * 8.0 * np.ones((1, 1) + grid)).astype(np.float32)
    return x, y, d, p, off, g


def test_iwe_is_exact_on_exactly_summable_streams():
    H, W = 17, 33
    x, y, d, p, off, g = exact_stream(H, W, [20000, 0, 15000], (3, 5))
    f, iwe = run_forward(x, y, d, p, off, g, H, W, 0.0, "variance")
    fr, iwer = GR.reference(x, y, d, p, off, torch.from_numpy(g).double(), H, W, 0.0, "variance")
    assert (iwe == iwer.numpy().astype(np.float32)).all()
    np.testing.assert_allclose(f, fr.numpy(), rtol=1e-12)


def test_chunking_empty_and_nan_windows(monkeypatch):
    """window chunks and candidate passes change no value (exact stream, variance without blur: f bit for bit), an empty
    window has zero gradient, and a NaN node makes only its window's f NaN"""
    from event_utils_b200.contrast_max import grid_flow as GF
    H, W = 17, 33
    sizes = [9000, 0, 7000, 8000]
    x, y, d, p, off, g = exact_stream(H, W, sizes, (3, 5), seed=1)
    cand = np.stack([g + 8.0 * j for j in range(40)], 1)
    args = cuda(x, y, d, p)
    ends = torch.from_numpy(off[1:]).cuda()
    kw = dict(t0=0.0, blur_sigma=0.0, batch_end_indices=ends)
    f_all = GF.grid_flow_contrast_candidates_torch(*args, torch.from_numpy(cand).cuda(), (H, W), **kw)
    monkeypatch.setattr(GF, "CANDIDATES_WORKSPACE_BYTES", 1)     # one window per call
    f_one = GF.grid_flow_contrast_candidates_torch(*args, torch.from_numpy(cand).cuda(), (H, W), **kw)
    assert torch.equal(f_all, f_one)
    f64, _ = run_forward(x, y, d, p, off, g, H, W, 0.0, "variance")
    assert np.array_equal(f64, f_all[:, 0].cpu().numpy())
    f, gg = torch_loss(x, y, d, p, off, g, H, W, 0.0, "variance")
    f.sum().backward()
    assert (gg.grad[1] == 0).all() and torch.isfinite(gg.grad).all()
    bad = g.copy()
    bad[2, 0, 1, 1] = np.nan
    fb, gb = torch_loss(x, y, d, p, off, bad, H, W, 0.0, "variance")
    fb.sum().backward()
    fb = fb.detach().cpu()
    assert torch.isnan(fb[2]) and torch.equal(fb[[0, 1, 3]], f.detach().cpu()[[0, 1, 3]])
    # the node sums of the other windows meet in f64 atomics, in any order
    assert_close_to_max(gb.grad[[0, 1, 3]].cpu().numpy(), gg.grad[[0, 1, 3]].cpu().numpy(), 1e-6)


def test_no_host_round_trips_and_constant_launch_count():
    from event_utils_b200 import _lib
    from event_utils_b200.contrast_max import grid_flow_contrast_candidates_torch, grid_flow_contrast_objective_torch
    L = _lib.lib()
    H, W = 60, 80
    counts = []
    for sizes in ([40000], [2500] * 16):
        x, y, d, p, off, g = batch_stream(2, sizes, H, W, (6, 8), 20.0)
        torch_loss(x, y, d, p, off, g, H, W, 1.0, "soe")     # warm-up
        gt = torch.from_numpy(g).cuda().requires_grad_(True)
        cand = torch.from_numpy(g).cuda().unsqueeze(1).repeat(1, 5, 1, 1, 1)
        ev = cuda(x, y, d, p)
        ends = torch.from_numpy(off[1:]).cuda()
        grid_flow_contrast_candidates_torch(*ev, cand, (H, W), objective="soe", batch_end_indices=ends)
        torch.cuda.synchronize()
        L.evk_prof_enable(1)
        torch.cuda.set_sync_debug_mode("error")
        try:
            f = grid_flow_contrast_objective_torch(*ev, gt, (H, W), objective="soe", batch_end_indices=ends)
            f.sum().backward()
            grid_flow_contrast_candidates_torch(*ev, cand, (H, W), objective="soe", batch_end_indices=ends)
        finally:
            torch.cuda.set_sync_debug_mode(0)
        ms, timed, launches = ctypes.c_double(), ctypes.c_longlong(), ctypes.c_longlong()
        _lib.check(L.evk_prof_collect(ctypes.byref(ms), ctypes.byref(timed), ctypes.byref(launches)))
        L.evk_prof_enable(0)
        assert torch.isfinite(gt.grad).all()
        counts.append(launches.value)
    assert counts[0] == counts[1] and counts[0] > 0, counts


def test_limits():
    """batch n_cand = 65535 canvases, and the node limits of the loss (gh gw = 4096) and of a candidates pass
    (n_cand gh gw = 12288)"""
    from event_utils_b200.contrast_max import grid_flow_contrast_candidates_torch
    rng = np.random.default_rng(8)
    H, W = 6, 8
    B, J = 4369, 15
    per = 3
    x, y = (rng.random(B * per) * (W - 1)).astype(np.float32), (rng.random(B * per) * (H - 1)).astype(np.float32)
    d = (-rng.random(B * per) * 0.1).astype(np.float32)
    p = np.ones(B * per, np.float32)
    off = np.arange(0, B * per + 1, per, dtype=np.int64)
    cand = (rng.standard_normal((B, J, 2, 2, 2)) * 5).astype(np.float32)
    fc = grid_flow_contrast_candidates_torch(*cuda(x, y, d, p), torch.from_numpy(cand).cuda(), (H, W), t0=0.0,
                                             batch_end_indices=torch.from_numpy(off[1:]).cuda()).cpu().numpy()
    for b in (0, 1234, B - 1):
        for j in (0, J - 1):
            f, _ = run_forward(x[off[b]:off[b + 1]], y[off[b]:off[b + 1]], d[off[b]:off[b + 1]], p[off[b]:off[b + 1]],
                               np.array([0, per], np.int64), np.ascontiguousarray(cand[b:b + 1, j]), H, W, 1.0, "variance")
            np.testing.assert_allclose(fc[b, j], f[0], rtol=1e-6)
    # the node limits: a 64 x 64 grid on a 64 x 64 sensor (the dense flow), forward and gradient; 3 candidates of it
    H = W = 64
    x, y, d, p, off, g = batch_stream(9, [20000, 10000], H, W, (64, 64), 10.0)
    f, gg = torch_loss(x, y, d, p, off, g, H, W, 1.0, "variance")
    f.sum().backward()
    g64 = torch.from_numpy(g).double().requires_grad_(True)
    fr, _ = GR.reference(x, y, d, p, off, g64, H, W, 1.0, "variance")
    fr.sum().backward()
    np.testing.assert_allclose(f.detach().cpu().numpy(), fr.detach().numpy(), rtol=1e-5)
    assert_close_to_max(gg.grad.cpu().numpy(), g64.grad.numpy(), 1e-4)
    cand = np.stack([g, g * 0.5, g * -1.0], 1)
    fc = grid_flow_contrast_candidates_torch(*cuda(x, y, d, p), torch.from_numpy(cand).cuda(), (H, W), t0=0.0,
                                             batch_end_indices=torch.from_numpy(off[1:]).cuda())
    np.testing.assert_allclose(fc[:, 0].cpu().numpy(), f.detach().cpu().numpy(), rtol=1e-6)


def affine_windows(seed, B, n, H, W, two_objects=False):
    """windows of edge events moving with an affine flow (u, v) = A [1, x, y] (exactly bilinear, so every node grid holds
    it), or two objects, the left and right halves of the sensor, with two uniform flows.  Returns the events, window ends
    and the truth as a function of the grid shape."""
    rng = np.random.default_rng(seed)
    xs, ys, ts, ps, ends, coefs = [], [], [], [], [], []
    for b in range(B):
        seg = rng.random((60, 4)) * [W - 4, H - 4, W - 4, H - 4] + 2     # edges over the whole sensor: every node has events
        s = rng.integers(0, 60, n)
        a = rng.random(n)
        x0 = seg[s, 0] + a * (seg[s, 2] - seg[s, 0])
        y0 = seg[s, 1] + a * (seg[s, 3] - seg[s, 1])
        t = np.sort(rng.random(n)) * 0.1
        dt = t - t[-1]
        if two_objects:
            v1, v2 = rng.uniform(-60, 60, 2), rng.uniform(-60, 60, 2)
            uv = np.where((x0 < W / 2)[:, None], v1, v2)
            coefs.append(None)
            x, y = x0 - uv[:, 0] * dt, y0 - uv[:, 1] * dt
        else:
            A = np.array([[rng.uniform(-50, 50), rng.uniform(-0.3, 0.3), rng.uniform(-0.3, 0.3)],
                          [rng.uniform(-50, 50), rng.uniform(-0.3, 0.3), rng.uniform(-0.3, 0.3)]])
            coefs.append(A)
            x, y = x0.copy(), y0.copy()
            for _ in range(6):   # x + u(x, y) dt = x0 at the event's own position
                u = A[0, 0] + A[0, 1] * x + A[0, 2] * y
                v = A[1, 0] + A[1, 1] * x + A[1, 2] * y
                x, y = x0 - u * dt, y0 - v * dt
        xs.append(x); ys.append(y); ts.append(t); ps.append(np.where(rng.random(n) < 0.8, 1.0, -1.0))
        ends.append((b + 1) * n)
    ev = [torch.from_numpy(np.concatenate(c)).float().cuda() for c in (xs, ys, ts, ps)]

    def truth(gh, gw):
        jj, ii = np.meshgrid(np.arange(gw) * (W - 1) / (gw - 1), np.arange(gh) * (H - 1) / (gh - 1))
        return np.stack([np.stack([A[c, 0] + A[c, 1] * jj + A[c, 2] * ii for c in range(2)]) for A in coefs])
    return ev, torch.tensor(ends, device="cuda"), truth


def test_fit_recovers_affine_flows():
    from event_utils_b200.contrast_max import charbonnier_smoothness, grid_flow_contrast_objective_torch, grid_flow_fit_torch
    H, W = 90, 120
    B = 8
    ev, ends, truth = affine_windows(21, B, 30000, H, W)
    lam = 1e-2
    fit = grid_flow_fit_torch(*ev, (H, W), grid_shapes=((3, 4), (6, 8)), smoothness=lam, batch_end_indices=ends,
                              param_ranges=[[-80, 80], [-80, 80]], max_iter=40, blur_sigma=1.0)
    assert fit.flow.shape == (B, 2, 6, 8) and fit.flow.dtype == torch.float64
    tr = torch.from_numpy(truth(6, 8)).cuda()
    f_truth = grid_flow_contrast_objective_torch(*ev, tr, (H, W), blur_sigma=1.0, batch_end_indices=ends).double()
    F_truth = f_truth + lam * charbonnier_smoothness(tr, 1.0)[0]
    # the RMS node error as a displacement over the 0.1 s window, against the 1 px blur that sets the resolution of the
    # contrast (the border nodes see few events and the smoothness pulls on them)
    err = (fit.flow - tr).pow(2).mean((1, 2, 3)).sqrt()
    hit = err * 0.1 <= 1.5
    assert int(hit.sum()) >= B - 1, (err, fit.status, fit.f, F_truth)
    assert bool((hit | (fit.f <= F_truth)).all()), (err, fit.f, F_truth)
    np.testing.assert_allclose(fit.contrast.cpu().numpy(), (fit.f - lam * charbonnier_smoothness(fit.flow, 1.0)[0]).cpu().numpy())


def test_fit_beats_the_global_fit_on_two_objects():
    from event_utils_b200.contrast_max import grid_flow_contrast_objective_torch, grid_flow_fit_torch, linvel_warp, \
        motion_contrast_fit_torch
    H, W = 90, 120
    B = 6
    ev, ends, _ = affine_windows(22, B, 30000, H, W, two_objects=True)
    ranges = [[-80, 80], [-80, 80]]
    lin = motion_contrast_fit_torch(*ev, linvel_warp(), ends, img_size=(H, W), param_ranges=ranges, max_iter=40)
    uniform = (-lin.params).view(B, 2, 1, 1).expand(B, 2, 3, 4).contiguous()
    f_lin = grid_flow_contrast_objective_torch(*ev, uniform, (H, W), batch_end_indices=ends).double()
    fit = grid_flow_fit_torch(*ev, (H, W), grid_shapes=((3, 4), (6, 8)), smoothness=1e-4, batch_end_indices=ends,
                              param_ranges=ranges, max_iter=40)
    assert bool((fit.contrast < f_lin).all()), (fit.contrast, f_lin)
    assert bool((fit.contrast < lin.f).all()), (fit.contrast, lin.f)
