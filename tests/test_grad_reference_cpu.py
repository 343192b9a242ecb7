"""The f64 gradient references of tests/grad_reference.py, pinned on the CPU: against the real reference's stored
gradients (tests/golden/autograd.npz, autograd_voxel.npz) and against autograd on the torch-op ports for the
adversarial hard cases, at the tolerance of tests/test_autograd_port.py with identical NaN patterns.  Needs no GPU."""
import numpy as np
import pytest
import torch

import autograd_ports as P
import autograd_voxel_ports as PV
import grad_reference as G
from autograd_cases import CASES
from autograd_voxel_cases import CASES as VCASES
from conftest import assert_close_to_max, golden
from edge_cases import hard_cases
from exact_bounds import assert_exact



def _close(a, b, what):
    """assert_close_to_max at 1e-5 over the finite values, with the same infinities and NaNs."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    assert (np.isnan(a) == np.isnan(b)).all(), what + ": NaN pattern differs"
    inf = np.isinf(b)
    assert (np.isinf(a) == inf).all() and (a[inf] == b[inf]).all(), what + ": infinities differ"
    fin = np.isfinite(b)
    if fin.any():
        assert_close_to_max(a[fin], b[fin], 1e-5, what)


def _check(name, ref, expected):
    v = ref.sum if isinstance(ref, G.Exact) else ref.v
    _close(np.asarray(v, np.float64).reshape(np.shape(expected)), expected, name)


@pytest.mark.parametrize("case", [c for c in CASES if c["kind"] != "chain"], ids=lambda c: c["name"])
def test_reference_against_golden(case):
    """image, timestamp images and warp (the chain case composes the warp with the image and is left to the ports)."""
    g = golden("autograd")
    name = case["name"]
    a = {k[len(name) + 4:]: g[k] for k in g.files if k.startswith(name + "/in_")}
    weights = [g["%s/w%d" % (name, i)] for i in range(2 if case["kind"] == "tsimg" else 1)]
    if case["kind"] == "warp":
        weights = [weights[0], g["%s/w1" % name]]
    ref = G.public_grads(case["kind"], a, weights, case["opts"])
    for k in case["grad"]:
        expected = g["%s/grad_%s" % (name, k)]
        if expected.size == 0:
            assert ref.get(k) is None, (name, k)
            continue
        _check("%s grad %s" % (name, k), ref[k], expected)


@pytest.mark.parametrize("case", VCASES, ids=lambda c: c["name"])
def test_voxel_reference_against_golden(case):
    g = golden("autograd_voxel")
    name = case["name"]
    a = {k: g["%s/in_%s" % (name, k)] for k in ("xs", "ys", "ts", "ps")}
    weights = [g["%s/w%d" % (name, i)] for i in range(2 if case.get("negpos") else 1)]
    ref = G.public_grads("voxel", a, weights, B=case["B"], negpos=bool(case.get("negpos")))
    for k in ("ts", "ps"):
        expected = g["%s/grad_%s" % (name, k)]
        if expected.size == 0:
            assert ref[k] is None, (name, k)
        else:
            _check("%s grad %s" % (name, k), ref[k], expected)


def _port_grads(kind, a, opts, B=None, negpos=False, seed=0):
    """Autograd on the ports on the CPU: (weights, {input: grad})."""
    names = {"image": ["xs", "ys", "ps"], "tsimg": ["xs", "ys", "ts"], "warp": ["xs", "ys", "ts", "flow"],
             "voxel": ["ts", "ps"]}[kind]
    leaves = {k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in a.items()}
    for k in names:
        leaves[k].requires_grad_(True)
    if kind == "image":
        outs = (P.events_to_image_torch(leaves["xs"], leaves["ys"], leaves["ps"], **opts),)
    elif kind == "tsimg":
        outs = P.events_to_timestamp_image_torch(leaves["xs"], leaves["ys"], leaves["ts"], leaves["ps"], **opts)
    elif kind == "warp":
        outs = P.warp_events_flow_torch(leaves["xs"], leaves["ys"], leaves["ts"], leaves["ps"], leaves["flow"])
    else:
        fn = PV.events_to_neg_pos_voxel_torch if negpos else PV.events_to_voxel_torch
        outs = fn(leaves["xs"], leaves["ys"], leaves["ts"], leaves["ps"], B, sensor_size=opts["sensor_size"])
        outs = outs if negpos else (outs,)
    rng = np.random.default_rng(seed)
    weights = [rng.integers(-4, 5, tuple(o.shape)).astype(np.float32) for o in outs]
    sum((o * torch.from_numpy(w)).sum() for o, w in zip(outs, weights)).backward()
    return weights, {k: (leaves[k].grad.numpy() if leaves[k].grad is not None else None) for k in names}


def _hard_setup(c, kind):
    n = c["x"].shape[0]
    rng = np.random.default_rng(int(str(c["k"]).split("*")[0]) + 77)
    a = dict(xs=c["x"], ys=c["y"], ts=np.sort(c["t"]) if kind != "voxel" else c["t"], ps=c["p"].copy())
    sensor = (c["H"], c["W"])
    if kind == "image_bil":
        return "image", a, dict(sensor_size=sensor, clip_out_of_range=True, padding=True, interpolation='bilinear')
    if kind == "image_nearest":
        return "image", a, dict(sensor_size=sensor, clip_out_of_range=True, padding=True, interpolation=None)
    if kind.startswith("tsimg"):
        a["ps"][rng.random(n) < 0.05] = np.nan
        return "tsimg", a, dict(sensor_size=sensor, clip_out_of_range=True, padding=c["padding"],
                                timestamp_reverse=kind == "tsimg_reverse")
    if kind == "warp":
        a["flow"] = (rng.standard_normal((2, c["H"], c["W"])) * 3).astype(np.float32)
        return "warp", a, {}
    return "voxel", a, dict(sensor_size=sensor)


@pytest.mark.parametrize("kind", ["image_bil", "image_nearest", "tsimg", "tsimg_reverse", "warp", "voxel", "negpos"])
def test_reference_against_ports_hard_cases(kind):
    """Borders, integer coordinates, clipped and wrapped indices, NaN polarities (timestamp images); for the voxel
    grids also unsorted stamps (tn outside [0, B-1] and beyond 1e9), +-inf and NaN polarities, -0.0 and +-2^20, and
    B up to 17.  The image and warp kinds run the existing hard-case kinds (finite polarities)."""
    vox = kind in ("voxel", "negpos")
    for c in hard_cases(31, 24, nonfinite=vox):
        fn_kind, a, opts = _hard_setup(c, "voxel" if vox else kind)
        if fn_kind == "tsimg" and c["x"].shape[0] < 2:
            continue
        B = None
        if vox:
            B = 1 + int(c["k"]) % 17 if isinstance(c["k"], int) else c["B"]
        weights, pg = _port_grads(fn_kind, a, opts, B=B, negpos=kind == "negpos", seed=int(c["k"]))
        if fn_kind == "warp":
            weights = [weights[0], weights[1]]
        ref = G.public_grads(fn_kind, a, weights, opts, B=B, negpos=kind == "negpos")
        for k, v in pg.items():
            what = "%s k=%s grad %s" % (kind, c["k"], k)
            if v is None:
                assert ref.get(k) is None, what
                continue
            if k == "ts":
                _check_ts(what, ref[k], v)
            else:
                _check(what, ref[k], v)


def _check_ts(what, ref, expected):
    """As tests/test_gpu_voxel_autograd.py assert_grad_t: the first and last stamps, which also take the cancelling sums
    of the normalisation (or of t0 = ts[-1] for the warp), where the port rounds those sums in f32, within 1e-5 of
    sum |grad ts| plus the f32 evaluation bound of the reference; every other event at 1e-5 of the largest."""
    v, b = np.asarray(ref.v, np.float64), G.bound_of(ref) + np.zeros(np.shape(ref.v))
    n = v.shape[0]
    ends = sorted({0, n - 1})
    inner = np.ones(n, bool)
    inner[ends] = False
    _close(v[inner], expected[inner], what)
    tot = np.sum(np.abs(expected[np.isfinite(expected)]))
    for i in ends:
        assert np.isnan(v[i]) == np.isnan(expected[i]), (what, i, v[i], expected[i])
        if np.isfinite(v[i]):
            assert abs(v[i] - expected[i]) <= 1e-5 * tot + b[i], (what, i, v[i], expected[i], tot, b[i])
        elif not np.isnan(v[i]):
            assert v[i] == expected[i], (what, i)


def test_reference_exact_on_exact_streams():
    """On an exactly computable voxel stream (tests/edge_cases.py exact_grad_streams) every per-event value of the
    reference is an f32 value, and the port, which rounds every step in f32, agrees with it bit for bit (the first and
    last stamps, where the port sums in f32, excepted)."""
    from edge_cases import exact_grad_streams
    s = exact_grad_streams(5, "voxel", 3000)
    # the port raises IndexError where the kernel drops an event: keep the pixels the reference can index
    keep = (s["x"] < s["W"]) & (s["y"] < s["H"])
    keep[[0, -1]] = True
    a = dict(xs=np.where(keep, s["x"], 0)[keep], ys=np.where(keep, s["y"], 0)[keep], ts=s["t"][keep], ps=s["p"][keep])
    a["xs"][[0, -1]] = a["ys"][[0, -1]] = 0.5
    weights, pg = _port_grads("voxel", a, dict(sensor_size=(s["H"], s["W"])), B=s["B"])
    ref = G.public_grads("voxel", a, weights, B=s["B"])
    for k in ("ts", "ps"):
        got = np.asarray(ref[k].v, np.float64)[1:-1]
        assert (got.astype(np.float32).astype(np.float64) == got).all(), k
        assert_exact(pg[k][1:-1], G.Exact(got, np.abs(got), np.ones_like(got)), what="voxel exact %s" % k)
