"""No-GPU checks of tests/flow_timestamp_reference.py, the f64 reference of the batched dense-flow average-timestamp
loss, and of the host side of flow_timestamp_objective_torch: on streams inside the canvas the reference agrees with
the ports' warp_events_flow_torch and events_to_timestamp_image_torch (pinned to the reference by tests/golden), its
gradient with central differences, the f32 stamp preparation with evk_tsimg.cu's arithmetic bit for bit, and the
scene of the GPU descent test has its minimum at the true flow."""
import numpy as np
import pytest
import scipy.ndimage
import torch

import autograd_ports as ports
import flow_timestamp_reference as R

H, W = 30, 40


def stream(seed, n, mag, margin):
    """events inside [margin, W-1-margin] x [margin, H-1-margin], sorted stamps t in [0, 0.1] and d = t - t[-1], a
    smooth flow of up to `mag` px per unit time"""
    rng = np.random.default_rng(seed)
    x = (margin + rng.random(n) * (W - 1 - 2 * margin)).astype(np.float32)
    y = (margin + rng.random(n) * (H - 1 - 2 * margin)).astype(np.float32)
    t = (np.sort(rng.random(n)) * 0.1).astype(np.float32)
    d = (t - t[-1]).astype(np.float32)
    p = (rng.integers(0, 2, n) * 2 - 1).astype(np.float32)
    yy, xx = np.mgrid[0:H, 0:W]
    flow = np.stack((np.cos(xx / 7.0 + yy / 11.0), np.sin(xx / 5.0 - yy / 9.0))) * mag
    return x, y, t, d, p, flow.astype(np.float32)


@pytest.mark.parametrize("reverse", [False, True])
@pytest.mark.parametrize("sigma", [0.0, 2.0])
def test_reference_matches_ports_inside(reverse, sigma):
    x, y, t, d, p, flow = stream(1, 4000, 40.0, 5.0)      # |u d| <= 4 px: every event stays inside
    xw, yw = R.warp_f32(x, y, d, flow)
    keep, finite = R.keep_mask(xw, yw, H, W)
    assert keep.all() and finite.all()
    tau = R.tau_f32(t, [0, len(t)], reverse)
    f, T, C = R.reference(x, y, d, tau, p, [0, len(x)], torch.from_numpy(flow).double()[None], sigma)
    xw_p, yw_p = ports.warp_events_flow_torch(torch.from_numpy(x), torch.from_numpy(y), torch.from_numpy(d), None,
                                              torch.from_numpy(flow), t0=torch.zeros(()))
    imgs = ports.events_to_timestamp_image_torch(xw_p, yw_p, torch.from_numpy(t), torch.from_numpy(p), sensor_size=(H, W),
                                                 timestamp_reverse=reverse)
    total = 0.0
    for s, img in enumerate(imgs):
        img = img.numpy()
        np.testing.assert_allclose(T[0, s].detach().numpy(), img, rtol=0, atol=1e-5 * np.abs(img).max())
        G = scipy.ndimage.gaussian_filter(img.astype(np.float64), sigma, mode="reflect", truncate=4.0) if sigma else img
        total += float((G.astype(np.float64) ** 2).sum())
    assert abs(float(f[0]) - total) <= 1e-5 * total
    # C counts every event once: 1 + sum k over the canvas is the canvas size plus the events of the polarity
    for s, sel in enumerate((p > 0, p <= 0)):
        assert abs(float(C[0, s].sum()) - (H + 1) * (W + 1) - sel.sum()) < 1e-9 * len(x)


def test_reference_gradient_matches_central_differences():
    x, y, t, d, p, flow = stream(2, 3000, 60.0, 3.0)
    offsets = [0, 1800, 3000]
    tau = R.tau_f32(t, offsets)
    flows = torch.from_numpy(np.stack([flow, -0.5 * flow])).double().requires_grad_(True)
    f, _, _ = R.reference(x, y, d, tau, p, offsets, flows, 1.0)
    g = np.array([1.0, -0.7])
    (f * torch.from_numpy(g)).sum().backward()
    grad = flows.grad.numpy()
    h = 1e-4
    for b, c, yy, xx in ((0, 0, 10, 12), (0, 1, 20, 30), (1, 0, 5, 33), (1, 1, 15, 7), (0, 0, 25, 3)):
        fp, fm = flows.detach().clone(), flows.detach().clone()
        fp[b, c, yy, xx] += h
        fm[b, c, yy, xx] -= h
        num = (float((R.reference(x, y, d, tau, p, offsets, fp, 1.0)[0] * torch.from_numpy(g)).sum()) -
               float((R.reference(x, y, d, tau, p, offsets, fm, 1.0)[0] * torch.from_numpy(g)).sum())) / (2 * h)
        assert abs(num - grad[b, c, yy, xx]) <= 1e-5 * np.abs(grad).max() + 1e-4 * abs(num), (b, c, yy, xx, num, grad[b, c, yy, xx])
    assert np.abs(grad).max() > 0


@pytest.mark.parametrize("reverse", [False, True])
def test_stamp_preparation_is_bitwise_the_timestamp_image_arithmetic(reverse):
    from event_utils_b200.contrast_max.flow_timestamp_objective import _normalised_stamps
    rng = np.random.default_rng(3)
    sizes = [5000, 0, 1, 3000, 2000]
    off = np.concatenate(([0], np.cumsum(sizes))).astype(np.int64)
    t = np.concatenate([np.sort(rng.random(s)) * rng.random() * 10 + rng.random() * 1e3 for s in sizes]).astype(np.float32)
    sample = torch.from_numpy(np.repeat(np.arange(len(sizes)), sizes))
    got = _normalised_stamps(torch.from_numpy(t), sample, torch.from_numpy(off), reverse).numpy()
    want = R.tau_f32(t, off, reverse)
    assert got.dtype == np.float32 and (got.view(np.uint32) == want.view(np.uint32)).all()
    # f64 stamps: formed in f64, then rounded to f32
    t64 = t.astype(np.float64) + rng.random(len(t)) * 1e-4
    got = _normalised_stamps(torch.from_numpy(t64), sample, torch.from_numpy(off), reverse).numpy()
    for b in range(len(sizes)):
        tb = t64[off[b]:off[b + 1]]
        if len(tb):
            den = tb[-1] - tb[0] + 1e-6
            want = (((-tb + tb[-1]) if reverse else (tb - tb[0])) / den).astype(np.float32)
            assert (got[off[b]:off[b + 1]] == want).all()


def test_reference_keep_rule_empty_and_nan_samples():
    x, y, t, d, p, flow = stream(4, 6000, 300.0, 0.0)   # up to 30 px: events leave on every side
    xw, yw = R.warp_f32(x, y, d, flow)
    keep, _ = R.keep_mask(xw, yw, H, W)
    assert 0.2 < keep.mean() < 0.95
    flows = torch.from_numpy(np.stack([flow, flow, flow])).double()
    flows[2, 0, int(y[5500]), int(x[5500])] = float("nan")
    offsets = [0, 4000, 4000, 6000]
    tau = R.tau_f32(t, offsets)
    f, T, C = R.reference(x, y, d, tau, p, offsets, flows, 2.0)
    k = keep[:4000]
    for s, sel in enumerate((p[:4000] > 0, p[:4000] <= 0)):
        # every kept event lands whole on the canvas, every other one contributes nothing
        assert abs(float(C[0, s].sum()) - (H + 1) * (W + 1) - (k & sel).sum()) < 1e-9 * len(x)
    assert float(f[1]) == 0.0 and (T[1] == 0).all() and (C[1] == 1).all()
    assert np.isnan(float(f[2])) and torch.isnan(T[2]).all()


def test_descent_scene_has_its_minimum_at_the_true_flow():
    """the premise of the GPU descent test: on its scene (one-sided loss, t0 = the last stamp, blur 1) the reference's f
    over a grid of uniform flows u_true (1 + a, 1 + b), a, b in -15 % .. 15 %, is smallest within 5 % of u_true"""
    Hs, Ws = 120, 160
    u = np.array([32.0, -21.0])
    x, y, t, p = R.edge_scene(H=Hs, W=Ws, u_true=tuple(u))
    t32 = t.astype(np.float32)
    d = (t - t[-1]).astype(np.float32)
    tau = R.tau_f32(t32, [0, len(t)])
    x, y, p = (a.astype(np.float32) for a in (x, y, p))
    best = None
    for a in np.linspace(-0.15, 0.15, 7):
        for b in np.linspace(-0.15, 0.15, 7):
            v = u * [1 + a, 1 + b]
            fl = torch.tensor(v).view(1, 2, 1, 1).expand(1, 2, Hs, Ws)
            fv = float(R.reference(x, y, d, tau, p, [0, len(t)], fl, 1.0)[0][0])
            if best is None or fv < best[0]:
                best = (fv, v)
    assert np.linalg.norm(best[1] - u) <= 0.05 * np.linalg.norm(u), best


def test_argument_errors():
    from event_utils_b200.contrast_max import flow_timestamp_objective_torch
    x = torch.zeros(10)
    with pytest.raises(ValueError, match="must not require grad"):
        flow_timestamp_objective_torch(x.clone().requires_grad_(True), x, x, x, torch.zeros(2, 4, 5))
    with pytest.raises(ValueError, match="must not require grad"):
        flow_timestamp_objective_torch(x, x, x, x, torch.zeros(2, 4, 5), t0=torch.zeros((), requires_grad=True))
    for bad in (torch.zeros(3, 4, 5), torch.zeros(1, 1, 4, 5), torch.zeros(4, 5)):
        with pytest.raises(ValueError, match="must have shape"):
            flow_timestamp_objective_torch(x, x, x, x, bad)
    with pytest.raises(ValueError, match="same length"):
        flow_timestamp_objective_torch(x, x[:9], x, x, torch.zeros(2, 4, 5))
    with pytest.raises(ValueError, match="2 samples of events for a batch of 3 flows"):
        flow_timestamp_objective_torch(x, x, x, x, torch.zeros(3, 2, 4, 5), batch_end_indices=[4, 10])
    with pytest.raises(ValueError, match="1 samples of events for a batch of 2 flows"):
        flow_timestamp_objective_torch(x, x, x, x, torch.zeros(2, 2, 4, 5), batch_end_indices=torch.tensor([10]))
