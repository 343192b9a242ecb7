"""Seeded scenes for the voxel-grid gradient tests (tests/test_autograd_voxel_port.py, tests/test_gpu_voxel_autograd.py)
and their golden generator (tests/golden/make_golden_autograd_voxel.py): 400 events on a 12x16 sensor with negative
(wrapping) coordinates, and the stamp patterns where the reference's subgradients matter: integer tn, repeated first
and last stamps, stamps one ulp off a bin, dt == 0, NaN polarities."""
import numpy as np
import torch

H, W, N = 12, 16, 400
f32 = np.float32


def _stamps(rng, kind, B):
    if kind == "dyadic":
        # quarter-bin tn, integers included: t in multiples of 1/4, t0 = 0, dt = B-1 (a power of two for B = 5, 9)
        t = np.sort(rng.integers(0, 4 * (B - 1) + 1, N)).astype(f32) / f32(4)
        t[:3], t[-3:] = 0, B - 1          # repeated first and last stamps
        return t
    if kind == "ulp":
        # dt = 1: tn = 4t, and every stamp is a bin's stamp b/4 or one ulp to either side of it
        t = rng.integers(0, 5, N).astype(f32) / f32(4)
        side = rng.integers(-1, 2, N)
        t = np.where(side < 0, np.nextafter(t, f32(-1)), np.where(side > 0, np.nextafter(t, f32(2)), t)).astype(f32)
        t = np.sort(t)
        t[0], t[-1] = 0, 1
        return t
    if kind == "dt0":
        return np.full(N, f32(0.25))
    return (np.sort(rng.random(N)) * 0.05).astype(f32)


def scene(case):
    """The case's inputs as CPU tensors xs, ys, ts, ps."""
    rng = np.random.default_rng(case["seed"])
    xs = rng.uniform(-W, W, N).astype(f32)
    ys = rng.uniform(-H, H, N).astype(f32)
    ts = _stamps(rng, case["stamps"], case["B"])
    ps = rng.choice(np.array(case.get("pols", [1.0, -1.0, 0.5]), f32), N)
    if case.get("nan_p"):
        ps[rng.random(N) < 0.03] = np.nan
    return dict(xs=torch.from_numpy(xs), ys=torch.from_numpy(ys), ts=torch.from_numpy(ts), ps=torch.from_numpy(ps))


_NP = [1.0, -1.0, 0.0, 0.37, np.nan]
CASES = [
    dict(name="b1", B=1, seed=1, stamps="uniform"),
    dict(name="b2", B=2, seed=2, stamps="uniform", nan_p=True),
    dict(name="b5", B=5, seed=3, stamps="uniform", nan_p=True),
    dict(name="b9", B=9, seed=4, stamps="uniform"),
    dict(name="b5_dyadic", B=5, seed=5, stamps="dyadic"),
    dict(name="b9_dyadic", B=9, seed=6, stamps="dyadic", nan_p=True),
    dict(name="b5_ulp", B=5, seed=7, stamps="ulp"),
    dict(name="b2_ulp", B=2, seed=8, stamps="ulp"),
    dict(name="b5_dt0", B=5, seed=9, stamps="dt0"),
    dict(name="b1_dt0", B=1, seed=10, stamps="dt0"),
    dict(name="negpos_b5", B=5, seed=11, stamps="uniform", negpos=True, pols=_NP),
    dict(name="negpos_b2_dyadic", B=2, seed=12, stamps="dyadic", negpos=True, pols=_NP),
    dict(name="negpos_b5_ulp", B=5, seed=13, stamps="ulp", negpos=True, pols=_NP),
    dict(name="negpos_b5_dt0", B=5, seed=14, stamps="dt0", negpos=True, pols=_NP),
]


def forward(case, fns, inputs):
    """The case's outputs (a tuple) through fns = (events_to_voxel_torch, events_to_neg_pos_voxel_torch)."""
    voxel, negpos = fns
    a = inputs
    if case.get("negpos"):
        return tuple(negpos(a["xs"], a["ys"], a["ts"], a["ps"], case["B"], sensor_size=(H, W)))
    return (voxel(a["xs"], a["ys"], a["ts"], a["ps"], case["B"], sensor_size=(H, W)),)


def loss_weights(case, outs):
    rng = np.random.default_rng(case["seed"] + 1000)
    return [torch.from_numpy(rng.standard_normal(tuple(o.shape)).astype(f32)) for o in outs]


def run(case, fns, inputs, weights=None, grad=("ts", "ps")):
    """Forward, loss sum(out * R), backward.  Returns (outputs, weights, grads) with grads[k] None where autograd left
    input k without a gradient."""
    leaves = {k: (v.detach().clone().requires_grad_(True) if k in grad else v) for k, v in inputs.items()}
    outs = forward(case, fns, leaves)
    if weights is None:
        weights = loss_weights(case, outs)
    loss = sum((o * w.to(o.device)).sum() for o, w in zip(outs, weights))
    loss.backward()
    return [o.detach() for o in outs], weights, {k: leaves[k].grad for k in grad}
