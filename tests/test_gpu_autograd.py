"""Gradients of the CUDA event image, timestamp images and flow warp (event_utils_b200.autograd, csrc/evk_grad.cu)
against autograd on the torch-op ports of the reference (tests/autograd_ports.py, pinned to the reference by
tests/test_autograd_port.py), on the same device.  Per-event gradients: max error <= 1e-5 of the largest one; the flow
gradient, a scatter, also cell by cell against exact f64 sums of its f32 taps (tests/exact_bounds.py)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import autograd_ports as P
from autograd_cases import CASES, forward, run, scene
from conftest import assert_close_to_max
from edge_cases import hard_cases
from exact_bounds import assert_within_exact
from grad_reference import flow_grad_exact

pytestmark = pytest.mark.gpu

PORT = (P.events_to_image_torch, P.events_to_timestamp_image_torch, P.warp_events_flow_torch)


def ours():
    from event_utils_b200.representations.image import events_to_image_torch, events_to_timestamp_image_torch
    from event_utils_b200.transforms.optic_flow import warp_events_flow_torch
    return events_to_image_torch, events_to_timestamp_image_torch, warp_events_flow_torch


def to(inputs, device):
    return {k: v.to(device) for k, v in inputs.items()}


def pinned_port():
    """The port with its warped coordinates pinned to the values of our warp by a straight-through add (the port's
    graph, our values).  The two warps may differ in the last bit, and a warped coordinate one ulp below an integer
    lands in another pixel than one at it, which changes that event's gradient by O(1): both right, not comparable."""
    warp = ours()[2]

    def warp_pinned(xt, yt, tt, pt, flow, t0=None):
        xw, yw = P.warp_events_flow_torch(xt, yt, tt, pt, flow, t0=t0)
        with torch.no_grad():
            ox, oy = warp(xt, yt, tt, pt, flow, t0=t0)
        return xw + (ox.to(xw) - xw).detach(), yw + (oy.to(yw) - yw).detach()
    return P.events_to_image_torch, P.events_to_timestamp_image_torch, warp_pinned


def compare(case, inputs, what, outputs=True):
    """Run the case through ours and the port on the inputs' device with the same loss; gradients must agree, and an
    input the port leaves without a gradient stays without one.  `outputs`: also compare the forward outputs."""
    outs, w, grads = run(case, ours(), inputs)
    p_outs, _, p_grads = run(case, pinned_port() if case["kind"] == "chain" else PORT, inputs, weights=w)
    for i, (o, po) in enumerate(zip(outs, p_outs)):
        assert o.device == po.device
        if outputs:
            assert_close_to_max(o.cpu().numpy(), po.cpu().numpy(), 1e-5, "%s out%d" % (what, i))
    for k in case["grad"]:
        if p_grads[k] is None:
            assert grads[k] is None, "%s: %s must get no gradient" % (what, k)
            continue
        g = grads[k]
        assert g is not None, "%s: no gradient for %s" % (what, k)
        assert g.dtype == inputs[k].dtype and g.device == inputs[k].device and g.shape == inputs[k].shape, (what, k)
        assert_close_to_max(g.cpu().numpy(), p_grads[k].cpu().numpy(), 1e-5, "%s grad %s" % (what, k))
    return outs, w, grads


@pytest.mark.parametrize("device", ["cuda", "cpu"])
@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_against_port(case, device):
    compare(case, to(scene(case), device), case["name"])


def check_flow_exact(inputs, grad_flow, weights, t0):
    xs, ys, ts = (inputs[k].detach().cpu().numpy().reshape(-1) for k in ("xs", "ys", "ts"))
    t_rel = (ts - np.float32(t0)).astype(np.float32)
    H, W = grad_flow.shape[-2:]
    ex = flow_grad_exact(xs, ys, t_rel, weights[0].numpy(), weights[1].numpy(), H, W)
    assert_within_exact(grad_flow.detach().cpu().numpy().reshape(2, H, W), ex, what="flow gradient")


@pytest.mark.parametrize("name", ["warp", "warp_t0"])
def test_flow_gradient_cell_by_cell(name):
    case = next(c for c in CASES if c["name"] == name)
    inputs = to(scene(case), "cuda")
    _, w, grads = run(case, ours(), inputs)
    t0 = inputs["t0"].item() if "t0" in inputs else inputs["ts"][-1].item()
    check_flow_exact(inputs, grads["flow"], w, t0)


def _hard_inputs(c, kind):
    n = c["x"].shape[0]
    rng = np.random.default_rng(int(c["k"]) + 77)
    p = c["p"].copy()
    if kind == "tsimg":
        p[rng.random(n) < 0.05] = np.nan
    inputs = dict(xs=torch.from_numpy(c["x"]), ys=torch.from_numpy(c["y"]), ts=torch.from_numpy(np.sort(c["t"])),
                  ps=torch.from_numpy(p))
    if kind == "warp":
        inputs["flow"] = torch.from_numpy((rng.standard_normal((2, c["H"], c["W"])) * 3).astype(np.float32))
    return inputs


@pytest.mark.parametrize("kind", ["image_bil", "image_nearest", "tsimg", "tsimg_reverse", "warp"])
def test_hard_cases(kind):
    """Borders, integer coordinates, clipped events, wrapped indices, NaN polarities (timestamp images)."""
    for c in hard_cases(31, 24, nonfinite=False):
        sensor = (c["H"], c["W"])
        if kind.startswith("image"):
            case = dict(name=kind, kind="image", seed=int(c["k"]), grad="xs ys ps".split(),
                        opts=dict(sensor_size=sensor, clip_out_of_range=True, padding=True,
                                  interpolation='bilinear' if kind == "image_bil" else None))
        elif kind.startswith("tsimg"):
            case = dict(name=kind, kind="tsimg", seed=int(c["k"]), grad="xs ys ts ps".split(),
                        opts=dict(sensor_size=sensor, clip_out_of_range=True, padding=c["padding"],
                                  timestamp_reverse=kind == "tsimg_reverse"))
        else:
            case = dict(name=kind, kind="warp", seed=int(c["k"]), grad="xs ys ts flow".split(), opts={})
        if kind.startswith("tsimg") and c["x"].shape[0] < 2:
            continue
        inputs = to(_hard_inputs(c, case["kind"]), "cuda")
        # the polarities span 2^-10 .. 2^20, so the image sums depend on their order: forward parity on these inputs
        # is checked cell by cell against exact sums in test_gpu_adversarial.py
        _, w, grads = compare(case, inputs, "%s k=%s" % (kind, c["k"]), outputs=case["kind"] != "image")
        if kind == "warp":
            check_flow_exact(inputs, grads["flow"], w, inputs["ts"][-1].item())


def test_outputs_unchanged_and_no_graph_without_grad():
    """The grad path runs the plain path's kernels: the warp is bit for bit the same, the scatters agree up to the
    order their atomic additions land in (which varies from run to run on either path).  Without grad mode, or when
    no differentiable input requires grad, the plain path runs and the outputs have no grad_fn."""
    for case in CASES:
        inputs = to(scene(case), "cuda")
        plain = forward(case, ours(), inputs)
        assert all(o.grad_fn is None for o in plain)
        leaves = {k: (v.clone().requires_grad_(True) if k in case["grad"] else v) for k, v in inputs.items()}
        graded = forward(case, ours(), leaves)
        with torch.no_grad():
            nograd = forward(case, ours(), leaves)
        for a, b, c in zip(plain, graded, nograd):
            assert b.grad_fn is not None and c.grad_fn is None, case["name"]
            if case["kind"] == "warp":
                assert torch.equal(a, b.detach()) and torch.equal(a, c), case["name"]
            else:
                assert_close_to_max(b.detach().cpu().numpy(), a.cpu().numpy(), 1e-6, case["name"])
                assert_close_to_max(c.cpu().numpy(), a.cpu().numpy(), 1e-6, case["name"])
    # only inputs the reference does not differentiate require grad
    c = next(c for c in CASES if c["name"] == "image_nearest_clip")
    a = to(scene(c), "cuda")
    assert forward(c, ours(), dict(a, xs=a["xs"].requires_grad_(True)))[0].grad_fn is None
    c = next(c for c in CASES if c["name"] == "tsimg_clip")
    a = to(scene(c), "cuda")
    assert all(o.grad_fn is None for o in forward(c, ours(), dict(a, ps=a["ps"].requires_grad_(True))))
    c = next(c for c in CASES if c["name"] == "warp")
    a = to(scene(c), "cuda")
    assert all(o.grad_fn is None for o in forward(c, ours(), dict(a, ps=a["ps"].requires_grad_(True))))


def test_input_forms():
    """(N,1) shapes, float64 stamps, t0 as a float and as a tensor, a `device=` move, img.sum().backward()."""
    _, tsimg, warp = ours()
    case = next(c for c in CASES if c["name"] == "warp")
    a = to(scene(case), "cuda")
    for t0_kind in ("float", "tensor"):
        xs, ys = (a[k].reshape(-1, 1).clone().requires_grad_(True) for k in ("xs", "ys"))
        ts = a["ts"].double().reshape(-1, 1).requires_grad_(True)
        flow = a["flow"].clone().requires_grad_(True)
        t0 = 0.02 if t0_kind == "float" else torch.tensor(0.02, dtype=torch.float64, device="cuda", requires_grad=True)
        res = []
        for fn in (warp, P.warp_events_flow_torch):
            for leaf in (xs, ys, ts, flow) + ((t0,) if t0_kind == "tensor" else ()):
                leaf.grad = None
            xw, yw = fn(xs, ys, ts, a["ps"], flow, t0=t0)
            ((xw.float() ** 2).sum() + (yw.float() * 3).sum()).backward()
            res.append([leaf.grad.clone() for leaf in (xs, ys, ts, flow)] + ([t0.grad.clone()] if t0_kind == "tensor" else []))
        for g, pg, what in zip(res[0], res[1], ["xs", "ys", "ts", "flow", "t0"]):
            assert g.dtype == pg.dtype and g.shape == pg.shape, (t0_kind, what)
            if what == "t0":
                # -sum over the events of ts's gradient, which cancels heavily; the reference forms the warped
                # coordinates in float64 for float64 stamps, this package in float32
                assert abs(float(g - pg)) <= 1e-5 * float(res[1][2].abs().sum()), (float(g), float(pg))
            else:
                assert_close_to_max(g.cpu().numpy(), pg.cpu().numpy(), 1e-5, "%s %s" % (t0_kind, what))
    # image on another device than the events; an expanded (stride 0) incoming gradient
    from event_utils_b200.representations.image import events_to_image_torch
    c = next(c for c in CASES if c["name"] == "image_bil_clip")
    a = to(scene(c), "cuda")
    grads = []
    for fn in (events_to_image_torch, P.events_to_image_torch):
        xs = a["xs"].clone().requires_grad_(True)
        img = fn(xs, a["ys"], a["ps"], **c["opts"]) if fn is P.events_to_image_torch else \
            fn(xs, a["ys"], a["ps"], device="cpu", **c["opts"])
        img.sum().backward()
        grads.append(xs.grad)
    assert grads[0].device == a["xs"].device
    assert_close_to_max(grads[0].cpu().numpy(), grads[1].cpu().numpy(), 1e-5, "image device=cpu")
    # only one of the two timestamp images used
    c = next(c for c in CASES if c["name"] == "tsimg_clip")
    a = to(scene(c), "cuda")
    grads = []
    for fn in (tsimg, P.events_to_timestamp_image_torch):
        ts = a["ts"].clone().requires_grad_(True)
        pos, _ = fn(a["xs"], a["ys"], ts, a["ps"], **c["opts"])
        (pos ** 2).sum().backward()
        grads.append(ts.grad)
    assert_close_to_max(grads[0].cpu().numpy(), grads[1].cpu().numpy(), 1e-5, "tsimg pos only")


def _blur_variance(img):
    """-variance of a 7x7 Gaussian blur, as f32 sums of shifted images (no TF32 convolution, whose input rounding
    would differ between two images that differ in the last bits)."""
    k = torch.exp(-torch.arange(-3.0, 4.0, device=img.device) ** 2 / 2)
    k = k / k.sum()
    b = img
    for dim, pad in ((1, (3, 3, 0, 0)), (0, (0, 0, 3, 3))):
        q = F.pad(b[None, None], pad)[0, 0]
        b = sum(k[i] * q.narrow(dim, i, b.shape[dim]) for i in range(7))
    return -((b - b.mean()) ** 2).mean()


def _chain(fns, xs, ys, ts, ps, flow, ts_images):
    image, tsimg, warp = fns
    xw, yw = warp(xs, ys, ts, ps, flow)
    if ts_images:
        pos, neg = tsimg(xw, yw, ts, ps, sensor_size=(480, 640))
        return _blur_variance(pos) + _blur_variance(neg)
    return _blur_variance(image(xw, yw, ps, sensor_size=(480, 640), interpolation='bilinear'))


@pytest.mark.parametrize("ts_images", [False, True], ids=["image", "timestamp"])
def test_chain_5m(ts_images):
    """flow (requires grad) -> warp -> bilinear image or timestamp images -> blur + variance in torch -> backward(),
    at 5 M events on a 480x640 sensor: flow, xs, ys and ts get the port's gradients.  The loss's gradient image is a
    function of the forward images, which the two sides sum in different orders (about 1e-7 of the largest cell
    apart), and each event's gradient takes differences of neighbouring cells of it: the chain agrees to 1e-4 of
    the largest gradient, each function by itself to 1e-5 (test_against_port, test_hard_cases)."""
    n, H, W = 5_000_000, 480, 640
    g = torch.Generator(device="cuda").manual_seed(5)

    def off_the_grid(size):
        # at an integer coordinate the gradient is one-sided and the side depends on the last bit of the sample
        # position, which the port forms differently (ATen divides by a scalar through its reciprocal): keep the
        # events 0.01 px away from pixel centres (integer coordinates are in the hard cases)
        whole = torch.randint(0, size - 1, (n,), device="cuda", generator=g).float()
        return whole + 0.01 + 0.98 * torch.rand(n, device="cuda", generator=g)
    xs, ys = off_the_grid(W), off_the_grid(H)
    ts = torch.sort(torch.rand(n, device="cuda", generator=g))[0] * 0.05
    ps = (torch.rand(n, device="cuda", generator=g) < 0.5).float() * 2 - 1
    flow0 = torch.randn(2, H, W, device="cuda", generator=g) * 20
    res = []
    for fns in (ours(), pinned_port()):
        leaves = [a.clone().requires_grad_(True) for a in (xs, ys, ts, flow0)]
        loss = _chain(fns, leaves[0], leaves[1], leaves[2], ps, leaves[3], ts_images)
        loss.backward()
        res.append((loss.item(), [a.grad for a in leaves]))
    assert abs(res[0][0] - res[1][0]) <= 1e-5 * abs(res[1][0])
    for g0, g1, what in zip(res[0][1], res[1][1], ["xs", "ys", "ts", "flow"]):
        assert g0 is not None
        assert_close_to_max(g0.cpu().numpy(), g1.cpu().numpy(), 1e-4, what)
