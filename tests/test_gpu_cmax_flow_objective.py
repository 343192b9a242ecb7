"""The batched dense-flow contrast objective (evk_cmax_flow_objective_f32 / _grad_f32, flow_contrast_objective_torch)
against the f64 reference of tests/flow_objective_reference.py, the existing single-sample entry, and linvel."""
import ctypes

import numpy as np
import pytest
import torch

import flow_objective_reference as R
from conftest import assert_close_to_max
from exact_bounds import gamma

pytestmark = pytest.mark.gpu

OBJ = {"variance": 0, "sos": 1, "soe": 2, "sosa": 5}


def batch_stream(seed, sizes, H, W, mag, integer=False, leave=None):
    """concatenated samples; per sample events in the sensor, d = t - t0 in [-0.1, 0] (t0 = the sample's last stamp),
    a random smooth flow of up to `mag` px per window.  leave: index of a sample whose flow sends every event off the
    canvas."""
    rng = np.random.default_rng(seed)
    n = sum(sizes)
    if integer:
        x = rng.integers(0, W, n).astype(np.float32)
        y = rng.integers(0, H, n).astype(np.float32)
    else:
        x = (rng.random(n) * (W - 1)).astype(np.float32)
        y = (rng.random(n) * (H - 1)).astype(np.float32)
    p = (rng.integers(0, 2, n) * 2 - 1).astype(np.float32)
    d = np.empty(n, np.float32)
    off = np.concatenate(([0], np.cumsum(sizes))).astype(np.int64)
    for b in range(len(sizes)):
        d[off[b]:off[b + 1]] = -np.sort(rng.random(sizes[b]))[::-1] * 0.1
    yy, xx = np.mgrid[0:H, 0:W]
    flows = []
    for b in range(len(sizes)):
        a, c = rng.random(2) * 6.28
        f = np.stack((np.cos(xx / (W / 5.0) + a), np.sin(yy / (H / 4.0) + c))) * rng.random() * mag * 10.0
        if b == leave:
            f = np.full((2, H, W), -50.0 * (W + H), np.float64)     # d <= 0: every event moves far right and down
            d[off[b]:off[b + 1]] = np.minimum(d[off[b]:off[b + 1]], -0.02)
        flows.append(f)
    return x, y, d, p, off, np.stack(flows).astype(np.float32)


def run_forward(x, y, d, p, off, flows, sigma, name, param=3.0):
    from event_utils_b200 import _lib
    L = _lib.lib()
    B, _, H, W = flows.shape
    X, Y, D, P, O, F = (torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (x, y, d, p, off, flows))
    f = torch.empty(B, dtype=torch.float64, device="cuda")
    iwe = torch.empty((B, H + 1, W + 1), device="cuda")
    ws = torch.empty(L.evk_cmax_flow_objective_workspace_bytes(B, H, W), dtype=torch.uint8, device="cuda")
    _lib.check(L.evk_cmax_flow_objective_f32(X.data_ptr(), Y.data_ptr(), D.data_ptr(), P.data_ptr(), O.data_ptr(), B, x.shape[0],
                                             F.data_ptr(), H, W, sigma, OBJ[name], param, f.data_ptr(), iwe.data_ptr(),
                                             ws.data_ptr(), ws.numel(), None))
    torch.cuda.synchronize()
    return f.cpu().numpy(), iwe.cpu().numpy()


def torch_loss(x, y, d, p, off, flows, sigma, name, param=3.0, t0=0.0):
    """flow_contrast_objective_torch on device inputs with ts = d and t0 = 0, so that d reaches the kernel unchanged"""
    from event_utils_b200.contrast_max import flow_contrast_objective_torch
    fl = torch.from_numpy(flows).cuda().requires_grad_(True)
    ev = [torch.from_numpy(a).cuda() for a in (x, y, d, p)]
    f = flow_contrast_objective_torch(*ev, fl, t0=t0, objective=name, blur_sigma=sigma, obj_param=param,
                                      batch_end_indices=torch.from_numpy(off[1:]).cuda())
    return f, fl


@pytest.mark.parametrize("name", ["variance", "sos", "soe", "sosa"])
@pytest.mark.parametrize("sigma", [0.0, 1.0, 3.0])
@pytest.mark.parametrize("batch", [1, 5])
@pytest.mark.parametrize("integer", [False, True])
def test_f_and_iwe_against_reference(name, sigma, batch, integer):
    H, W = 45, 60
    sizes = [20000] if batch == 1 else [15000, 0, 9000, 20000, 12000]
    x, y, d, p, off, flows = batch_stream(7 + batch, sizes, H, W, 50.0, integer, leave=3 if batch == 5 else None)
    param = 0.3
    f, iwe = run_forward(x, y, d, p, off, flows, sigma, name, param)
    fr, iwer, _ = R.reference(x, y, d, p, off, torch.from_numpy(flows).double(), sigma, name, param)
    fr = fr.detach().numpy()
    iwer = iwer.detach().numpy()
    for b in range(batch):
        assert_close_to_max(iwe[b], iwer[b], 1e-5, "iwe %d" % b)
        assert abs(f[b] - fr[b]) <= 1e-5 * max(abs(fr[b]), 1e-30), (b, f[b], fr[b])
    if batch == 5:
        assert (iwe[1] == 0).all() and (iwe[3] == 0).all()


@pytest.mark.parametrize("name", ["variance", "sos", "soe", "sosa"])
@pytest.mark.parametrize("sigma", [0.0, 1.0, 3.0])
def test_gradient_against_reference(name, sigma):
    H, W = 45, 60
    sizes = [15000, 0, 9000, 20000, 12000]
    x, y, d, p, off, flows = batch_stream(3, sizes, H, W, 50.0, leave=3)
    param = 0.3
    f, fl = torch_loss(x, y, d, p, off, flows, sigma, name, param)
    g = torch.from_numpy(np.random.default_rng(5).standard_normal(len(sizes)))
    (f * g.cuda().to(f.dtype)).sum().backward()
    got = fl.grad.cpu().numpy().astype(np.float64)
    flow64 = torch.from_numpy(flows).double().requires_grad_(True)
    fr, iwer, mag = R.reference(x, y, d, p, off, flow64, sigma, name, param)
    (fr * g).sum().backward()
    ref = flow64.grad.numpy()
    assert_close_to_max(got, ref, 1e-4, "grad_flow %s sigma %g" % (name, sigma))
    M, cnt = R.grad_magnitude(x, y, d, p, off, flow64, sigma, name, param, g.numpy(), iwer.detach().numpy(), mag.numpy())
    bound = gamma(cnt + 32) * M
    err = np.abs(got - ref)
    bad = err > bound
    assert not bad.any(), "%d cells outside the bound, e.g. err %r bound %r" % (bad.sum(), err[bad][:3], bound[bad][:3])
    assert (got[1] == 0).all() and (got[3] == 0).all()


def test_parity_with_the_single_sample_entry():
    """in-canvas stream: the new forward's variance f and IWE equal evk_cmax_flow_variance_f32's (unchanged entry)"""
    from event_utils_b200 import _lib
    L = _lib.lib()
    H, W = 180, 240
    rng = np.random.default_rng(11)
    n = 300000
    x = (20 + rng.random(n) * (W - 41)).astype(np.float32)
    y = (20 + rng.random(n) * (H - 41)).astype(np.float32)
    t = np.sort(rng.random(n)).astype(np.float32) * np.float32(0.1)
    p = (rng.integers(0, 2, n) * 2 - 1).astype(np.float32)
    fl = (rng.standard_normal((2, H, W)) * 20).astype(np.float32)
    t0 = t[-1]
    d = (t - t0).astype(np.float32)
    f, iwe = run_forward(x, y, d, p, np.array([0, n], np.int64), fl[None], 1.0, "variance")
    X, Y, T, P, F = (torch.from_numpy(a).cuda() for a in (x, y, t, p, fl))
    ws = torch.empty(L.evk_cmax_workspace_bytes(H, W), dtype=torch.uint8, device="cuda")
    res = torch.empty(8, dtype=torch.float64, device="cuda")
    iwe_old = torch.empty((H + 1, W + 1), device="cuda")
    _lib.check(L.evk_cmax_flow_variance_f32(X.data_ptr(), Y.data_ptr(), T.data_ptr(), P.data_ptr(), n, F.data_ptr(), float(t0),
                                            H, W, 1.0, 0, res.data_ptr(), iwe_old.data_ptr(), ws.data_ptr(), ws.numel(), None))
    torch.cuda.synchronize()
    assert res[4].item() == 0
    assert_close_to_max(iwe[0], iwe_old.cpu().numpy(), 1e-6)
    assert abs(f[0] - res[0].item()) <= 1e-6 * abs(res[0].item())


def test_cross_check_against_linvel():
    """uniform flow v at sigma 0 on the 180x240 canvas: f(v) = variance_objective(linvel at -v), v.grad = -its gradient"""
    from event_utils_b200.contrast_max import flow_contrast_objective_torch, linvel_warp, variance_objective
    H, W = 180, 240
    rng = np.random.default_rng(4)
    n = 200000
    x = 30 + rng.random(n) * (W - 61)
    y = 30 + rng.random(n) * (H - 61)
    t = np.sort(rng.random(n)) * 0.1
    p = rng.integers(0, 2, n) * 2.0 - 1
    obj, warp = variance_objective(), linvel_warp()
    for v0 in ((30.0, -20.0), (-55.0, 12.5)):
        v = torch.tensor(v0, dtype=torch.float64, device="cuda", requires_grad=True)
        ev = [torch.from_numpy(a).cuda() for a in (x, y, t, p)]
        f = flow_contrast_objective_torch(*ev, v.view(2, 1, 1).expand(2, H, W), blur_sigma=0.0)
        f.sum().backward()
        fl = obj.evaluate_function((-v0[0], -v0[1]), x, y, t, p, warp, (H, W), 0.0)
        gl = obj.evaluate_gradient((-v0[0], -v0[1]), x, y, t, p, warp, (H, W), 0.0)
        assert f.shape == (1,) and f.dtype == torch.float64
        assert abs(f.item() - fl) <= 1e-4 * abs(fl), (f.item(), fl)
        np.testing.assert_allclose(v.grad.cpu().numpy(), -np.asarray(gl), rtol=1e-4, atol=1e-4 * np.abs(gl).max())


def test_batch_behaviour():
    H, W = 60, 80
    sizes = [30000, 5000, 0, 22000]
    x, y, d, p, off, flows = batch_stream(21, sizes, H, W, 30.0)
    f, fl = torch_loss(x, y, d, p, off, flows, 1.0, "variance")
    g = torch.tensor([0.5, -2.0, 1.0, 3.0], dtype=torch.float32, device="cuda")
    (f * g).sum().backward()
    for b in range(len(sizes)):
        xb, yb, db, pb = (a[off[b]:off[b + 1]] for a in (x, y, d, p))
        fb, flb = torch_loss(xb, yb, db, pb, np.array([0, sizes[b]], np.int64), flows[b:b + 1], 1.0, "variance")
        (fb * g[b]).sum().backward()
        assert abs(f[b].item() - fb.item()) <= 1e-6 * max(abs(fb.item()), 1e-30)
        assert_close_to_max(fl.grad[b].cpu().numpy(), flb.grad[0].cpu().numpy(), 1e-5, "sample %d" % b)
    # sample b's loss puts no gradient into the other samples' flows
    f, fl = torch_loss(x, y, d, p, off, flows, 1.0, "variance")
    f[0].backward()
    assert (fl.grad[1:] == 0).all() and (fl.grad[0] != 0).any()
    # NaN in flow[b] at an event's pixel: f_b NaN, the others finite
    bad = flows.copy()
    bad[3, 0, int(y[off[3] + 7]), int(x[off[3] + 7])] = np.nan
    f, fl = torch_loss(x, y, d, p, off, bad, 1.0, "variance")
    f.sum().backward()
    fc = f.detach().cpu().numpy()
    assert np.isnan(fc[3]) and np.isfinite(fc[:3]).all()
    assert torch.isfinite(fl.grad[:3]).all()


def test_no_host_round_trips_and_constant_launch_count():
    from event_utils_b200 import _lib
    L = _lib.lib()
    H, W = 60, 80
    counts = []
    for sizes in ([40000], [2500] * 16):
        x, y, d, p, off, flows = batch_stream(2, sizes, H, W, 30.0)
        torch_loss(x, y, d, p, off, flows, 1.0, "soe")     # warm-up: scratch buffers, modules
        fl = torch.from_numpy(flows).cuda().requires_grad_(True)
        ev = [torch.from_numpy(a).cuda() for a in (x, y, d, p)]
        ends = torch.from_numpy(off[1:]).cuda()
        torch.cuda.synchronize()
        L.evk_prof_enable(1)
        from event_utils_b200.contrast_max import flow_contrast_objective_torch
        torch.cuda.set_sync_debug_mode("error")
        try:
            f = flow_contrast_objective_torch(*ev, fl, objective="soe", blur_sigma=1.0, batch_end_indices=ends)
            f.sum().backward()
        finally:
            torch.cuda.set_sync_debug_mode(0)
        ms, timed, launches = ctypes.c_double(), ctypes.c_longlong(), ctypes.c_longlong()
        _lib.check(L.evk_prof_collect(ctypes.byref(ms), ctypes.byref(timed), ctypes.byref(launches)))
        L.evk_prof_enable(0)
        assert torch.isfinite(fl.grad).all()
        counts.append(launches.value)
    assert counts[0] == counts[1] and counts[0] > 0, counts


def test_gradient_descent_recovers_a_uniform_velocity():
    """a textured scene of edges moving with flow u_true; Adam on a uniform 2-vector from zero finds u_true within 5%"""
    from event_utils_b200.contrast_max import flow_contrast_objective_torch
    H, W = 120, 160
    rng = np.random.default_rng(9)
    u_true = np.array([32.0, -21.0])
    n = 200000
    # edges: points on 24 random line segments, each event at a random time; sharp at t0 when warped by u_true
    seg = rng.random((24, 4)) * [W - 40, H - 40, W - 40, H - 40] + 20
    s = rng.integers(0, 24, n)
    a = rng.random(n)
    x0 = seg[s, 0] + a * (seg[s, 2] - seg[s, 0])
    y0 = seg[s, 1] + a * (seg[s, 3] - seg[s, 1])
    t = np.sort(rng.random(n)) * 0.2
    dt = t - t[-1]
    x = x0 - u_true[0] * dt
    y = y0 - u_true[1] * dt
    p = np.where(rng.random(n) < 0.8, 1.0, -1.0)
    ev = [torch.from_numpy(c).float().cuda() for c in (x, y, t, p)]
    v = torch.zeros(2, dtype=torch.float32, device="cuda", requires_grad=True)
    opt = torch.optim.Adam([v], lr=2.0)
    sched = torch.optim.lr_scheduler.CosineAnnealingLR(opt, T_max=300, eta_min=0.02)
    for it in range(300):
        opt.zero_grad()
        f = flow_contrast_objective_torch(*ev, v.view(2, 1, 1).expand(2, H, W), blur_sigma=1.0)
        f.sum().backward()
        opt.step()
        sched.step()
    got = v.detach().cpu().numpy()
    assert np.linalg.norm(got - u_true) <= 0.05 * np.linalg.norm(u_true), (got, u_true)
