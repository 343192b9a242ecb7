"""Seeded scenes for the gradient tests (tests/test_autograd_port.py, tests/test_gpu_autograd.py) and their golden
generator (tests/golden/make_golden_autograd.py): 2 000 events on a 30x40 sensor with coordinates beyond every
border (clipped, wrapped, outside the flow field), exact integers, and a few NaN polarities where the function
allows them.  Each case names the function, its options and the inputs that require grad."""
import numpy as np
import torch

H, W, N = 30, 40, 2000


def _coords(rng, n, size, lo, hi):
    v = rng.uniform(lo, size - 1 + hi, n)
    snap = rng.random(n) < 0.1
    v[snap] = np.floor(v[snap])
    return v.astype(np.float32)


def scene(case):
    """The case's inputs as CPU tensors: xs, ys, ts, ps, and flow / t0 for the warp cases."""
    rng = np.random.default_rng(case["seed"])
    lo, hi = case["span"]
    xs, ys = _coords(rng, N, W, lo, hi), _coords(rng, N, H, lo, hi)
    ts = np.sort(rng.random(N)).astype(np.float32) * np.float32(0.05)
    ps = rng.choice(np.array([1.0, -1.0, 0.0, 0.37], np.float32), N)
    if case.get("nan_p"):
        ps[rng.random(N) < 0.02] = np.nan
    out = dict(xs=torch.from_numpy(xs), ys=torch.from_numpy(ys), ts=torch.from_numpy(ts), ps=torch.from_numpy(ps))
    if case["kind"] in ("warp", "chain"):
        out["flow"] = torch.from_numpy((rng.standard_normal((2, H, W)) * 20).astype(np.float32))
        if case.get("t0") is not None:
            out["t0"] = torch.tensor(np.float32(case["t0"]))
    return out


_BIL = dict(sensor_size=(H, W), interpolation='bilinear')
CASES = [
    dict(name="image_bil_clip", kind="image", seed=1, span=(-0.9, 1.5), grad="xs ys ps".split(),
         opts=dict(_BIL, clip_out_of_range=True, padding=True)),
    dict(name="image_bil_noclip", kind="image", seed=2, span=(-0.9, -0.01), grad="xs ys ps".split(),
         opts=dict(_BIL, clip_out_of_range=False, padding=False)),
    dict(name="image_nearest_clip", kind="image", seed=3, span=(-0.9, 1.5), grad="xs ys ps".split(),
         opts=dict(sensor_size=(H, W), clip_out_of_range=True, padding=True)),
    dict(name="image_nearest_wrap", kind="image", seed=4, span=(-2.0, 0.99), grad=["ps"],
         opts=dict(sensor_size=(H, W), clip_out_of_range=False, padding=False)),
    dict(name="tsimg_clip", kind="tsimg", seed=5, span=(-0.9, 1.5), grad="xs ys ts ps".split(), nan_p=True,
         opts=dict(sensor_size=(H, W), clip_out_of_range=True, padding=True, timestamp_reverse=False)),
    dict(name="tsimg_reverse", kind="tsimg", seed=6, span=(-0.9, -0.01), grad="xs ys ts ps".split(), nan_p=True,
         opts=dict(sensor_size=(H, W), clip_out_of_range=False, padding=False, timestamp_reverse=True)),
    dict(name="tsimg_reverse_clip", kind="tsimg", seed=7, span=(-0.9, 1.5), grad="xs ys ts".split(),
         opts=dict(sensor_size=(H, W), clip_out_of_range=True, padding=False, timestamp_reverse=True)),
    dict(name="warp", kind="warp", seed=8, span=(-1.5, 1.5), grad="xs ys ts flow".split(), opts={}),
    dict(name="warp_t0", kind="warp", seed=9, span=(-1.5, 1.5), grad="xs ys ts flow t0".split(), t0=0.02, opts={}),
    dict(name="chain", kind="chain", seed=10, span=(0.0, -0.01), grad="xs ys ts flow".split(),
         opts=dict(_BIL, clip_out_of_range=True, padding=True)),
]


def forward(case, fns, inputs):
    """The case's outputs (a tuple) through fns = (events_to_image_torch, events_to_timestamp_image_torch,
    warp_events_flow_torch) of one implementation."""
    image, tsimg, warp = fns
    kind, opts, a = case["kind"], case["opts"], inputs
    if kind == "image":
        return (image(a["xs"], a["ys"], a["ps"], **opts),)
    if kind == "tsimg":
        return tuple(tsimg(a["xs"], a["ys"], a["ts"], a["ps"], **opts))
    xw, yw = warp(a["xs"], a["ys"], a["ts"], a["ps"], a["flow"], t0=a.get("t0"))
    if kind == "warp":
        return xw, yw
    return (image(xw, yw, a["ps"], **opts),)


def loss_weights(case, outs):
    rng = np.random.default_rng(case["seed"] + 1000)
    return [torch.from_numpy(rng.standard_normal(tuple(o.shape)).astype(np.float32)) for o in outs]


def run(case, fns, inputs, weights=None):
    """Forward, loss sum(out * R) with the case's seeded R (or `weights`), backward.  Returns (outputs, weights,
    grads): grads[name] is the gradient of each input the case names, None where autograd left it without one."""
    leaves = {k: (v.detach().clone().requires_grad_(True) if k in case["grad"] else v) for k, v in inputs.items()}
    outs = forward(case, fns, leaves)
    if weights is None:
        weights = loss_weights(case, outs)
    loss = sum((o * w.to(o.device)).sum() for o, w in zip(outs, weights))
    loss.backward()
    return [o.detach() for o in outs], weights, {k: leaves[k].grad for k in case["grad"]}
