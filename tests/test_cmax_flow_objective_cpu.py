"""No-GPU checks of tests/flow_objective_reference.py, the f64 reference of the batched dense-flow contrast objective:
on streams inside the canvas it agrees with the chain the repository already trusts (the ports' warp_events_flow_torch
and bilinear events_to_image_torch, pinned to the reference by tests/golden/autograd*.npz, then the oracle's
objectives), and on streams that leave the canvas it drops exactly the events the keep rule names."""
import numpy as np
import pytest
import torch

import autograd_ports as ports
import flow_objective_reference as R

H, W = 30, 40


def stream(seed, n, mag, margin):
    """events inside [margin, W-1-margin] x [margin, H-1-margin], d in [-0.1, 0], a smooth flow of up to `mag` px per
    unit time"""
    rng = np.random.default_rng(seed)
    x = (margin + rng.random(n) * (W - 1 - 2 * margin)).astype(np.float32)
    y = (margin + rng.random(n) * (H - 1 - 2 * margin)).astype(np.float32)
    d = (-np.sort(rng.random(n))[::-1] * 0.1).astype(np.float32)
    p = (rng.integers(0, 2, n) * 2 - 1).astype(np.float32)
    yy, xx = np.mgrid[0:H, 0:W]
    flow = np.stack((np.cos(xx / 7.0 + yy / 11.0), np.sin(xx / 5.0 - yy / 9.0))) * mag
    return x, y, d, p, flow.astype(np.float32)


@pytest.mark.parametrize("name", ["variance", "sos", "soe", "sosa"])
@pytest.mark.parametrize("sigma", [0.0, 1.0, 3.0])
def test_reference_matches_ports_and_oracle_inside(oracle, name, sigma):
    x, y, d, p, flow = stream(1, 4000, 40.0, 5.0)      # |u d| <= 4 px: every event stays inside
    xw, yw = R.warp_f32(x, y, d, flow)
    keep, finite = R.keep_mask(xw, yw, H, W)
    assert keep.all() and finite.all()
    param = 0.5
    f, iwe, _ = R.reference(x, y, d, p, [0, len(x)], torch.from_numpy(flow).double()[None], sigma, name, param)
    # the trusted chain in f32, as the reference runs it
    xw_p, yw_p = ports.warp_events_flow_torch(torch.from_numpy(x), torch.from_numpy(y), torch.from_numpy(d), None,
                                              torch.from_numpy(flow), t0=torch.zeros(()))
    img = ports.events_to_image_torch(xw_p, yw_p, torch.from_numpy(p), sensor_size=(H, W), interpolation='bilinear')
    img = img.numpy()
    np.testing.assert_allclose(iwe[0].detach().numpy(), img, rtol=0, atol=1e-5 * np.abs(img).max())
    if name == "variance":
        fo = oracle.variance_f(img, sigma)
    else:
        fo, _ = oracle.objective_of_images(name, img, blur_sigma=sigma, param=param)
    assert abs(float(f[0]) - fo) <= 1e-6 * abs(fo), (name, sigma, float(f[0]), fo)


def test_reference_drops_exactly_the_events_the_keep_rule_names():
    x, y, d, p, flow = stream(2, 6000, 300.0, 0.0)     # up to 30 px: events leave on every side
    xw, yw = R.warp_f32(x, y, d, flow)
    keep, finite = R.keep_mask(xw, yw, H, W)
    assert finite.all()
    for side in (xw < 0, xw >= W, yw < 0, yw >= H):
        assert side.any()
    assert 0.2 < keep.mean() < 0.95
    _, iwe, _ = R.reference(x, y, d, p, [0, len(x)], torch.from_numpy(flow).double()[None], 0.0, "variance")
    # the kept events alone, through the trusted chain: the same image
    k = np.flatnonzero(keep)
    xw_p, yw_p = ports.warp_events_flow_torch(torch.from_numpy(x[k]), torch.from_numpy(y[k]), torch.from_numpy(d[k]), None,
                                              torch.from_numpy(flow), t0=torch.zeros(()))
    img = ports.events_to_image_torch(xw_p, yw_p, torch.from_numpy(p[k]), sensor_size=(H, W), interpolation='bilinear')
    np.testing.assert_allclose(iwe[0].detach().numpy(), img.numpy(), rtol=0, atol=1e-5 * np.abs(img.numpy()).max())
    # every kept event lands whole on the canvas, every other one contributes nothing
    assert abs(float(iwe[0].sum()) - float(p[k].astype(np.float64).sum())) < 1e-9 * len(k)


def test_reference_batches_empty_samples_and_nan():
    x, y, d, p, flow = stream(3, 3000, 40.0, 5.0)
    flows = torch.from_numpy(np.stack([flow, flow * 0.5, flow])).double()
    flows[2, 0, int(y[2500]), int(x[2500])] = float("nan")
    f, iwe, _ = R.reference(x, y, d, p, [0, 2000, 2000, 3000], flows, 1.0, "variance")
    f0, _, _ = R.reference(x[:2000], y[:2000], d[:2000], p[:2000], [0, 2000], flows[:1], 1.0, "variance")
    assert float(f[0]) == float(f0[0])
    assert float(f[1]) == 0.0 and (iwe[1] == 0).all()
    assert np.isnan(float(f[2])) and torch.isnan(iwe[2]).all()
