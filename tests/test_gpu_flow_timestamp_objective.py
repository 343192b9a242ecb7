"""The batched dense-flow average-timestamp loss (evk_flow_timestamp_objective_f32 / _grad_f32,
flow_timestamp_objective_torch) against the f64 reference of tests/flow_timestamp_reference.py, the unchanged
flow-warp and timestamp-image entries, and zhu_timestamp_objective."""
import ctypes

import numpy as np
import pytest
import torch

import flow_timestamp_reference as R
from conftest import assert_close_to_max
from exact_bounds import gamma

pytestmark = pytest.mark.gpu


def batch_stream(seed, sizes, H, W, mag, integer=False, leave=None):
    """concatenated samples; per sample events in the sensor with sorted stamps t over 0.1 time units (d = t - the
    sample's last stamp, so in [-0.1, 0]) and a random smooth flow of up to `mag` px per unit time.  leave: index of a
    sample whose flow sends every event off the canvas."""
    rng = np.random.default_rng(seed)
    n = sum(sizes)
    if integer:
        x = rng.integers(0, W, n).astype(np.float32)
        y = rng.integers(0, H, n).astype(np.float32)
    else:
        x = (rng.random(n) * (W - 1)).astype(np.float32)
        y = (rng.random(n) * (H - 1)).astype(np.float32)
    p = (rng.integers(0, 2, n) * 2 - 1).astype(np.float32)
    t = np.empty(n, np.float32)
    off = np.concatenate(([0], np.cumsum(sizes))).astype(np.int64)
    yy, xx = np.mgrid[0:H, 0:W]
    flows = []
    for b in range(len(sizes)):
        t[off[b]:off[b + 1]] = np.sort(rng.random(sizes[b])) * 0.1 + b
        a, c = rng.random(2) * 6.28
        f = np.stack((np.cos(xx / (W / 5.0) + a), np.sin(yy / (H / 4.0) + c))) * rng.random() * mag * 10.0
        if b == leave:
            f = np.full((2, H, W), -50.0 * (W + H), np.float64)     # d <= 0: every event moves far right and down
            t[off[b]:off[b + 1] - 1] = np.minimum(t[off[b]:off[b + 1] - 1], t[off[b + 1] - 1] - 0.02)
        flows.append(f)
    d = np.empty(n, np.float32)
    for b in range(len(sizes)):
        if sizes[b]:
            d[off[b]:off[b + 1]] = t[off[b]:off[b + 1]] - t[off[b + 1] - 1]
    return x, y, t, d, p, off, np.stack(flows).astype(np.float32)


def run_forward(x, y, d, tau, p, off, flows, sigma):
    from event_utils_b200 import _lib
    L = _lib.lib()
    B, _, H, W = flows.shape
    X, Y, D, U, P, O, F = (torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (x, y, d, tau, p, off, flows))
    f = torch.empty(B, dtype=torch.float64, device="cuda")
    T = torch.empty((B, 2, H + 1, W + 1), device="cuda")
    C = torch.empty_like(T)
    ws = torch.empty(L.evk_flow_timestamp_objective_workspace_bytes(B, H, W), dtype=torch.uint8, device="cuda")
    _lib.check(L.evk_flow_timestamp_objective_f32(X.data_ptr(), Y.data_ptr(), D.data_ptr(), U.data_ptr(), P.data_ptr(),
                                                  O.data_ptr(), B, x.shape[0], F.data_ptr(), H, W, sigma, f.data_ptr(),
                                                  T.data_ptr(), C.data_ptr(), ws.data_ptr(), ws.numel(), None))
    torch.cuda.synchronize()
    return f.cpu().numpy(), T.cpu().numpy(), C.cpu().numpy()


def torch_loss(x, y, t, p, off, flows, sigma, reverse=False, t0=None):
    from event_utils_b200.contrast_max import flow_timestamp_objective_torch
    fl = torch.from_numpy(flows).cuda().requires_grad_(True)
    ev = [torch.from_numpy(a).cuda() for a in (x, y, t, p)]
    f = flow_timestamp_objective_torch(*ev, fl, t0=t0, blur_sigma=sigma, timestamp_reverse=reverse,
                                       batch_end_indices=torch.from_numpy(off[1:]).cuda())
    return f, fl


@pytest.mark.parametrize("sigma", [0.0, 1.0, 2.0])
@pytest.mark.parametrize("reverse", [False, True])
@pytest.mark.parametrize("batch", [1, 5])
@pytest.mark.parametrize("integer", [False, True])
def test_f_and_images_against_reference(sigma, reverse, batch, integer):
    H, W = 45, 60
    sizes = [20000] if batch == 1 else [15000, 0, 9000, 20000, 12000]
    x, y, t, d, p, off, flows = batch_stream(7 + batch, sizes, H, W, 50.0, integer, leave=3 if batch == 5 else None)
    if batch == 5:
        d[off[3]:off[4]] = np.minimum(d[off[3]:off[4]], -0.02)     # the sample's last event (d = 0) leaves too
    tau = R.tau_f32(t, off, reverse)
    f, T, C = run_forward(x, y, d, tau, p, off, flows, sigma)
    fr, Tr, Cr = (a.detach().numpy() for a in R.reference(x, y, d, tau, p, off, torch.from_numpy(flows).double(), sigma))
    for b in range(batch):
        assert_close_to_max(T[b], Tr[b], 1e-5, "T %d" % b)
        assert_close_to_max(C[b], Cr[b], 1e-5, "C %d" % b)
        assert abs(f[b] - fr[b]) <= 1e-5 * max(abs(fr[b]), 1e-30), (b, f[b], fr[b])
    if batch == 5:
        for b in (1, 3):
            assert (T[b] == 0).all() and (C[b] == 1).all() and f[b] == 0


@pytest.mark.parametrize("sigma", [0.0, 1.0, 2.0])
@pytest.mark.parametrize("reverse", [False, True])
def test_gradient_against_reference(sigma, reverse):
    H, W = 45, 60
    sizes = [15000, 0, 9000, 20000, 12000]
    x, y, t, d, p, off, flows = batch_stream(3, sizes, H, W, 50.0, leave=3)
    f, fl = torch_loss(x, y, t, p, off, flows, sigma, reverse)
    g = torch.from_numpy(np.random.default_rng(5).standard_normal(len(sizes)))
    (f * g.cuda().to(f.dtype)).sum().backward()
    got = fl.grad.cpu().numpy().astype(np.float64)
    tau = R.tau_f32(t, off, reverse)
    flow64 = torch.from_numpy(flows).double().requires_grad_(True)
    fr, Tr, Cr = R.reference(x, y, d, tau, p, off, flow64, sigma)
    (fr * g).sum().backward()
    ref = flow64.grad.numpy()
    assert_close_to_max(got, ref, 1e-4, "grad_flow sigma %g reverse %s" % (sigma, reverse))
    M, cnt = R.grad_magnitude(x, y, d, tau, p, off, flow64, sigma, g.numpy(), Tr.detach().numpy(), Cr.detach().numpy())
    bound = gamma(cnt + 32) * M
    err = np.abs(got - ref)
    bad = err > bound
    assert not bad.any(), "%d cells outside the bound, e.g. err %r bound %r" % (bad.sum(), err[bad][:3], bound[bad][:3])
    assert (got[1] == 0).all() and (got[3] == 0).all()


def _entries(x, y, t, p, flow, H, W, reverse):
    """evk_warp_flow_f32 (t0 = the last stamp) followed by evk_timestamp_image_counts_f32 on the (H+1, W+1) canvas"""
    from event_utils_b200 import _lib
    L = _lib.lib()
    n = x.shape[0]
    X, Y, Tt, P, F = (torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (x, y, t, p, flow))
    xw, yw = torch.empty_like(X), torch.empty_like(X)
    ws = torch.empty(max(L.evk_warp_flow_workspace_bytes(H, W), 256), dtype=torch.uint8, device="cuda")
    _lib.check(L.evk_warp_flow_f32(X.data_ptr(), Y.data_ptr(), Tt.data_ptr(), n, F.data_ptr(), H, W, float(t[-1]), xw.data_ptr(),
                                   yw.data_ptr(), ws.data_ptr(), ws.numel(), None))
    out = [torch.empty((H + 1, W + 1), device="cuda") for _ in range(4)]
    ws2 = torch.empty(L.evk_timestamp_image_workspace_bytes(H + 1, W + 1), dtype=torch.uint8, device="cuda")
    oob = torch.zeros(1, dtype=torch.int64, device="cuda")
    _lib.check(L.evk_timestamp_image_counts_f32(xw.data_ptr(), yw.data_ptr(), Tt.data_ptr(), P.data_ptr(), n, float(t[0]),
                                                float(t[-1]), H + 1, W + 1, float(W), float(H),
                                                _lib.TS_REVERSE if reverse else 0, *(o.data_ptr() for o in out),
                                                ws2.data_ptr(), ws2.numel(), oob.data_ptr(), None))
    torch.cuda.synchronize()
    assert oob.item() == 0
    pos, neg, cpos, cneg = (o.cpu().numpy() for o in out)
    return np.stack([pos, neg]), np.stack([cpos, cneg])


@pytest.mark.parametrize("reverse", [False, True])
def test_bitwise_against_the_unchanged_entries(reverse):
    """footprints that do not overlap: T and C equal the warp + timestamp-image entries bit for bit"""
    H, W = 60, 80
    rng = np.random.default_rng(12)
    gy, gx = np.mgrid[2:H - 3:4, 2:W - 3:4]                 # one event per 4x4 cell, moved by at most 1 px
    x = (gx.ravel() + rng.random(gx.size) * 0.9).astype(np.float32)
    y = (gy.ravel() + rng.random(gy.size) * 0.9).astype(np.float32)
    n = x.shape[0]
    t = (np.sort(rng.random(n)) * 0.05 + 3.0).astype(np.float32)
    p = (rng.integers(0, 2, n) * 2 - 1).astype(np.float32)
    flow = (rng.random((2, H, W)) * 30 - 15).astype(np.float32)   # |u d| < 0.75 px
    off = np.array([0, n], np.int64)
    f, fl = torch_loss(x, y, t, p, off, flow[None], 0.0, reverse)
    d = (t - t[-1]).astype(np.float32)
    _, T, C = run_forward(x, y, d, R.tau_f32(t, off, reverse), p, off, flow[None], 0.0)
    Te, Ce = _entries(x, y, t, p, flow, H, W, reverse)
    assert (T[0].view(np.uint32) == Te.view(np.uint32)).all()
    assert (C[0].view(np.uint32) == Ce.view(np.uint32)).all()
    # the torch function's own stamp preparation feeds the kernel the same tau: the f of these images, rounded to the
    # flow's f32
    fr = float(sum((T[0, s].astype(np.float64) ** 2).sum() for s in range(2)))
    assert f.dtype == torch.float32 and abs(f.item() - fr) <= 2.0 ** -24 * fr


def test_counts_on_an_exactly_summable_stream():
    """quarter-pixel positions under a zero flow: every tap is a multiple of 1/16 and every count sum is exact in f32,
    so C equals the timestamp-image entry's count image bit for bit whatever the order of the reductions"""
    H, W = 32, 48
    rng = np.random.default_rng(13)
    n = 300000
    hot = rng.random(n) < 0.5
    x = np.where(hot, 16.25, rng.integers(0, 4 * (W - 1), n) / 4.0).astype(np.float32)
    y = np.where(hot, 10.75, rng.integers(0, 4 * (H - 1), n) / 4.0).astype(np.float32)
    t = np.sort(rng.random(n)).astype(np.float32)
    p = (rng.integers(0, 2, n) * 2 - 1).astype(np.float32)
    flow = np.zeros((2, H, W), np.float32)
    off = np.array([0, n], np.int64)
    _, T, C = run_forward(x, y, (t - t[-1]).astype(np.float32), R.tau_f32(t, off), p, off, flow[None], 0.0)
    Te, Ce = _entries(x, y, t, p, flow, H, W, False)
    assert (C[0].view(np.uint32) == Ce.view(np.uint32)).all()
    # the stamp sums are not exact: up to ~1e5 f32 additions per pixel in either order
    assert_close_to_max(T[0], Te, 1e-4)


@pytest.mark.parametrize("sigma", [0.0, 2.0])
def test_against_zhu_timestamp_objective(sigma):
    """uniform flow -v (an expanded 2-vector) on 180x240 with every event strictly inside: f = -zhu_timestamp_objective's
    f at linvel v.  That path warps and normalises in f64; this one warps in f32, which moves each x', y' < 241 by at most
    2 ulp(256) = 2^-15 px and each tap weight by as much.  T is a weighted mean of the stamps and f = sum G^2, so the
    relative difference of f stays below 4 * 2^-15 (plus the f32 sums of that path, far below)."""
    from event_utils_b200.contrast_max import flow_timestamp_objective_torch, linvel_warp, zhu_timestamp_objective
    H, W = 180, 240
    rng = np.random.default_rng(4)
    n = 200000
    x = (30 + rng.random(n) * (W - 61)).astype(np.float32).astype(np.float64)
    y = (30 + rng.random(n) * (H - 61)).astype(np.float32).astype(np.float64)
    t = np.sort(rng.random(n)) * 0.1
    p = rng.integers(0, 2, n) * 2.0 - 1
    for v0 in ((30.0, -20.0), (-55.0, 12.5)):
        v = torch.tensor(v0, dtype=torch.float64, device="cuda", requires_grad=True)
        ev = [torch.from_numpy(a).cuda() for a in (x, y, t, p)]
        f = flow_timestamp_objective_torch(*ev, (-v).view(2, 1, 1).expand(2, H, W), blur_sigma=sigma)
        fz = -zhu_timestamp_objective().evaluate_function(v0, x, y, t, p, linvel_warp(), (H, W), sigma)
        assert f.shape == (1,) and f.dtype == torch.float64
        assert abs(f.item() - fz) <= 4 * 2.0 ** -15 * abs(fz), (f.item(), fz)
        f.sum().backward()
        assert torch.isfinite(v.grad).all() and (v.grad != 0).any()


def test_batch_behaviour():
    H, W = 60, 80
    sizes = [30000, 5000, 0, 22000, 1]
    x, y, t, d, p, off, flows = batch_stream(21, sizes, H, W, 30.0)
    f, fl = torch_loss(x, y, t, p, off, flows, 2.0)
    g = torch.tensor([0.5, -2.0, 1.0, 3.0, 1.5], dtype=torch.float32, device="cuda")
    (f * g).sum().backward()
    for b in range(len(sizes)):
        sl = slice(off[b], off[b + 1])
        fb, flb = torch_loss(x[sl], y[sl], t[sl], p[sl], np.array([0, sizes[b]], np.int64), flows[b:b + 1], 2.0)
        (fb * g[b]).sum().backward()
        assert abs(f[b].item() - fb.item()) <= 1e-6 * max(abs(fb.item()), 1e-30)
        assert_close_to_max(fl.grad[b].cpu().numpy(), flb.grad[0].cpu().numpy(), 1e-5, "sample %d" % b)
    # the empty and the one-event sample: f = 0 (T = 0: tau of a lone event is 0) and a zero gradient
    for b in (2, 4):
        assert f[b].item() == 0 and (fl.grad[b] == 0).all()
    # sample b's loss puts no gradient into the other samples' flows
    f, fl = torch_loss(x, y, t, p, off, flows, 2.0)
    f[0].backward()
    assert (fl.grad[1:] == 0).all() and (fl.grad[0] != 0).any()
    # NaN in flow[b] at an event's pixel: f_b and its gradient NaN, the others finite
    bad = flows.copy()
    bad[3, 0, int(y[off[3] + 7]), int(x[off[3] + 7])] = np.nan
    f, fl = torch_loss(x, y, t, p, off, bad, 2.0)
    f.sum().backward()
    fc = f.detach().cpu().numpy()
    assert np.isnan(fc[3]) and np.isfinite(np.delete(fc, 3)).all()
    assert torch.isnan(fl.grad[3]).any()
    assert torch.isfinite(fl.grad[[0, 1, 2, 4]]).all()


def test_inputs():
    """host events, f32 / f64 / expanded flows, t0 as a number or per sample"""
    from event_utils_b200.contrast_max import flow_timestamp_objective_torch
    H, W = 45, 60
    sizes = [8000, 12000]
    x, y, t, d, p, off, flows = batch_stream(31, sizes, H, W, 20.0)
    ends = off[1:].tolist()
    dev = [torch.from_numpy(a).cuda() for a in (x, y, t, p)]
    f_dev = flow_timestamp_objective_torch(*dev, torch.from_numpy(flows).cuda(), batch_end_indices=ends)
    f_host = flow_timestamp_objective_torch(x, y, t, p, torch.from_numpy(flows).cuda(), batch_end_indices=ends)
    torch.testing.assert_close(f_host, f_dev, rtol=1e-6, atol=0)     # the reductions' order may differ
    fl64 = torch.from_numpy(flows).double().cuda().requires_grad_(True)
    f64 = flow_timestamp_objective_torch(*dev, fl64, batch_end_indices=ends)
    assert f64.dtype == torch.float64
    torch.testing.assert_close(f64.float(), f_dev, rtol=1e-6, atol=0)
    f64.sum().backward()
    assert fl64.grad.dtype == torch.float64 and torch.isfinite(fl64.grad).all()
    # expanded: one uniform 2-vector per sample
    v = torch.tensor([[3.0, -2.0], [-1.0, 4.0]], device="cuda", requires_grad=True)
    fe = flow_timestamp_objective_torch(*dev, v.view(2, 2, 1, 1).expand(2, 2, H, W), batch_end_indices=ends)
    fe.sum().backward()
    full = v.detach().view(2, 2, 1, 1).expand(2, 2, H, W).contiguous().requires_grad_(True)
    ff = flow_timestamp_objective_torch(*dev, full, batch_end_indices=ends)
    ff.sum().backward()
    torch.testing.assert_close(fe, ff, rtol=1e-6, atol=0)
    assert torch.allclose(v.grad, full.grad.sum((2, 3)), rtol=1e-5, atol=1e-6 * full.grad.abs().sum().item())
    # t0: a number, or one per sample, against the reference with d = t - t0
    for t0 in (1.5, torch.tensor([0.05, 1.02], dtype=torch.float32)):
        f = flow_timestamp_objective_torch(*dev, torch.from_numpy(flows).cuda(), t0=t0 if isinstance(t0, float) else t0.cuda(),
                                           batch_end_indices=ends)
        t0s = np.broadcast_to(np.asarray(t0, np.float32), (2,))
        dd = np.concatenate([(t[off[b]:off[b + 1]] - t0s[b]).astype(np.float32) for b in range(2)])
        fr, _, _ = R.reference(x, y, dd, R.tau_f32(t, off), p, off, torch.from_numpy(flows).double(), 2.0)
        np.testing.assert_allclose(f.cpu().numpy(), fr.detach().numpy(), rtol=1e-5)


def test_full_size_canvas():
    from event_utils_b200.contrast_max import flow_timestamp_objective_torch
    H, W = 480, 640
    sizes = [50000] * 8
    x, y, t, d, p, off, flows = batch_stream(41, sizes, H, W, 40.0)
    f, fl = torch_loss(x, y, t, p, off, flows, 2.0)
    f.sum().backward()
    assert torch.isfinite(fl.grad).all() and (fl.grad != 0).any()
    fr, _, _ = R.reference(x[:sizes[0]], y[:sizes[0]], d[:sizes[0]], R.tau_f32(t[:sizes[0]], [0, sizes[0]]), p[:sizes[0]],
                           [0, sizes[0]], torch.from_numpy(flows[:1]).double(), 2.0)
    assert abs(f[0].item() - fr.item()) <= 1e-5 * fr.item()
    f1 = flow_timestamp_objective_torch(*(torch.from_numpy(a[off[7]:]).cuda() for a in (x, y, t, p)),
                                        torch.from_numpy(flows[7]).cuda())
    assert abs(f[7].item() - f1.item()) <= 1e-6 * f1.item()


def test_no_host_round_trips_and_constant_launch_count():
    from event_utils_b200 import _lib
    from event_utils_b200.contrast_max import flow_timestamp_objective_torch
    L = _lib.lib()
    H, W = 60, 80
    counts = []
    for sizes in ([40000], [2500] * 16):
        x, y, t, d, p, off, flows = batch_stream(2, sizes, H, W, 30.0)
        torch_loss(x, y, t, p, off, flows, 2.0)     # warm-up: scratch buffers, modules
        fl = torch.from_numpy(flows).cuda().requires_grad_(True)
        ev = [torch.from_numpy(a).cuda() for a in (x, y, t, p)]
        ends = torch.from_numpy(off[1:]).cuda()
        torch.cuda.synchronize()
        L.evk_prof_enable(1)
        torch.cuda.set_sync_debug_mode("error")
        try:
            f = flow_timestamp_objective_torch(*ev, fl, blur_sigma=2.0, timestamp_reverse=True, batch_end_indices=ends)
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
    """the scene of R.edge_scene; Adam on a uniform 2-vector from zero finds u_true within 5 % (the CPU test checks that
    the reference's f is smallest there)"""
    from event_utils_b200.contrast_max import flow_timestamp_objective_torch
    H, W = 120, 160
    u_true = np.array([32.0, -21.0])
    x, y, t, p = R.edge_scene(H=H, W=W, u_true=tuple(u_true))
    ev = [torch.from_numpy(c).float().cuda() for c in (x, y, t, p)]
    v = torch.zeros(2, dtype=torch.float32, device="cuda", requires_grad=True)
    opt = torch.optim.Adam([v], lr=2.0)
    sched = torch.optim.lr_scheduler.CosineAnnealingLR(opt, T_max=300, eta_min=0.02)
    for it in range(300):
        opt.zero_grad()
        f = flow_timestamp_objective_torch(*ev, v.view(2, 1, 1).expand(2, H, W), blur_sigma=1.0)
        f.sum().backward()
        opt.step()
        sched.step()
    got = v.detach().cpu().numpy()
    assert np.linalg.norm(got - u_true) <= 0.05 * np.linalg.norm(u_true), (got, u_true)
