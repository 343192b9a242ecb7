"""Gradients of the CUDA voxel grids (event_utils_b200.autograd.VoxelGrid, evk_voxel_grad_f32 in csrc/evk_grad.cu)
against autograd on the torch-op ports of the reference (tests/autograd_voxel_ports.py, pinned to the reference by
tests/test_autograd_voxel_port.py), on the same device.  Per-event gradients agree to 1e-5 of the largest one; the
gradients of a window's first and last stamps, which also carry the -sum terms of the normalisation, to 1e-5 of
sum |grad_t|."""
import numpy as np
import pytest
import torch

import autograd_voxel_ports as P
from autograd_voxel_cases import CASES, H, W, forward, run, scene
from conftest import assert_close_to_max

pytestmark = pytest.mark.gpu

PORT = (P.events_to_voxel_torch, P.events_to_neg_pos_voxel_torch)


def ours():
    from event_utils_b200.representations.voxel_grid import events_to_neg_pos_voxel_torch, events_to_voxel_torch
    return events_to_voxel_torch, events_to_neg_pos_voxel_torch


def to(inputs, device):
    return {k: v.to(device) for k, v in inputs.items()}


def assert_grad_t(g, pg, ends, what, rel=1e-5):
    """Per-event agreement (rel of the largest) away from the window ends; at the ends (which also carry the two-sum
    terms) within 1e-5 of sum |grad_t|."""
    g, pg = g.detach().cpu().numpy().reshape(-1), pg.detach().cpu().numpy().reshape(-1)
    inner = np.ones(g.shape[0], bool)
    inner[list(ends)] = False
    assert_close_to_max(g[inner], pg[inner], rel, what + " grad ts")
    tot = np.nansum(np.abs(pg))
    for i in ends:
        assert np.isnan(g[i]) == np.isnan(pg[i]), (what, i, g[i], pg[i])
        if not np.isnan(pg[i]):
            assert abs(g[i] - pg[i]) <= 1e-5 * tot, (what, i, g[i], pg[i], tot)


def compare(case, inputs, what, grad=("ts", "ps")):
    outs, w, grads = run(case, ours(), inputs, grad=grad)
    p_outs, _, p_grads = run(case, PORT, inputs, weights=w, grad=grad)
    for i, (o, po) in enumerate(zip(outs, p_outs)):
        assert o.device == po.device
        assert_close_to_max(o.cpu().numpy(), po.cpu().numpy(), 1e-5, "%s out%d" % (what, i))
    for k in grad:
        if p_grads[k] is None:
            assert grads[k] is None, "%s: %s must get no gradient" % (what, k)
            continue
        g = grads[k]
        assert g is not None, "%s: no gradient for %s" % (what, k)
        assert g.dtype == inputs[k].dtype and g.device == inputs[k].device and g.shape == inputs[k].shape, (what, k)
        if k == "ts":
            assert_grad_t(g, p_grads[k], (0, g.shape[0] - 1), what)
        else:
            assert_close_to_max(g.cpu().numpy(), p_grads[k].cpu().numpy(), 1e-5, "%s grad %s" % (what, k))


@pytest.mark.parametrize("device", ["cuda", "cpu"])
@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_against_port(case, device):
    compare(case, to(scene(case), device), "%s %s" % (case["name"], device))


@pytest.mark.parametrize("grad", [("ps",), ("ts",)], ids=["ps", "ts"])
def test_one_input_requires_grad(grad):
    for name in ("b5", "b5_dyadic") + (("negpos_b5",) if grad == ("ts",) else ()):
        case = next(c for c in CASES if c["name"] == name)
        compare(case, to(scene(case), "cuda"), "%s %s only" % (name, grad[0]), grad=grad)


def _exact_stream(n, B, seed):
    """dt = 1, stamps on a grid of 1/(4(B-1)): tn on quarter bins, integers and the two ends included; integer
    polarities and pixels.  Every tap, product and partial sum of either side's backward is exact in f32."""
    rng = np.random.default_rng(seed)
    q = 4 * (B - 1)
    ts = np.sort(rng.integers(0, q + 1, n)).astype(np.float32) / np.float32(q)
    ts[:2], ts[-2:] = 0, 1
    xs = rng.integers(-W, W, n).astype(np.float32) + 0.5
    ys = rng.integers(-H, H, n).astype(np.float32) + 0.5
    ps = rng.choice(np.array([1, -1, 2, -2], np.float32), n)
    return {k: torch.from_numpy(v).cuda() for k, v in dict(xs=xs, ys=ys, ts=ts, ps=ps).items()}


@pytest.mark.parametrize("negpos", [False, True], ids=["voxel", "negpos"])
def test_exact_bit_for_bit(negpos):
    B = 5
    case = dict(name="exact", B=B, seed=21, negpos=negpos)
    inputs = _exact_stream(20000, B, 21)
    rng = np.random.default_rng(22)
    shape = ((2,) if negpos else (1,)) + (B, H, W)
    weights = [torch.from_numpy(rng.integers(-3, 4, shape[1:]).astype(np.float32)) for _ in range(shape[0])]
    _, _, grads = run(case, ours(), inputs, weights=weights)
    _, _, p_grads = run(case, PORT, inputs, weights=weights)
    assert torch.equal(grads["ts"], p_grads["ts"])
    if negpos:
        assert grads["ps"] is None and p_grads["ps"] is None
    else:
        assert torch.equal(grads["ps"], p_grads["ps"])


def _port_windows(xs, ys, ts, ps, B, bounds):
    return [P.events_to_voxel_torch(xs[s:e], ys[s:e], ts[s:e], ps[s:e], B, sensor_size=(H, W)) for s, e in bounds]


def _windows_case(xs, ys, ts, ps, B, ours_fn, bounds, what):
    leaves, grids = [], []
    for impl in ("ours", "port"):
        t, p = ts.clone().requires_grad_(True), ps.clone().requires_grad_(True)
        g = ours_fn(xs, ys, t, p) if impl == "ours" else _port_windows(xs, ys, t, p, B, bounds)
        assert len(g) == len(bounds)
        rng = np.random.default_rng(5)
        loss = sum((v * torch.from_numpy(rng.standard_normal(v.shape).astype(np.float32)).cuda()).sum() for v in g)
        loss.backward()
        leaves.append((t.grad, p.grad))
        grids.append(g)
    for a, b in zip(*grids):
        assert_close_to_max(a.detach().cpu().numpy(), b.detach().cpu().numpy(), 1e-5, what + " grid")
    ends = sorted({i for s, e in bounds for i in (s, e - 1)})
    assert_grad_t(leaves[0][0], leaves[1][0], ends, what)
    assert_close_to_max(leaves[0][1].cpu().numpy(), leaves[1][1].cpu().numpy(), 1e-5, what + " grad ps")


def _window_events(n, seed, ts=None):
    rng = np.random.default_rng(seed)
    xs = torch.from_numpy(rng.uniform(-W, W, n).astype(np.float32)).cuda()
    ys = torch.from_numpy(rng.uniform(-H, H, n).astype(np.float32)).cuda()
    if ts is None:
        ts = np.sort(rng.random(n)).astype(np.float32)
    ps = torch.from_numpy(rng.choice(np.array([1.0, -1.0, 0.37], np.float32), n)).cuda()
    return xs, ys, torch.from_numpy(ts).cuda(), ps


def test_windows_fixed_n():
    from event_utils_b200.representations.voxel_grid import voxel_grids_fixed_n_torch
    B, n = 5, 700
    xs, ys, ts, ps = _window_events(10000, 31)
    bounds = [(i, i + n) for i in range(0, len(xs) - n, n)]
    _windows_case(xs, ys, ts, ps, B, lambda x, y, t, p: voxel_grids_fixed_n_torch(x, y, t, p, B, n, sensor_size=(H, W)),
                  bounds, "fixed_n")


def _fixed_t_bounds(ts, t):
    np_ts = ts.cpu().numpy()
    starts = np.arange(ts[0].item(), ts[-1].item() - t, t)
    return [(int(np.searchsorted(np_ts, a)), int(np.searchsorted(np_ts, a + t))) for a in starts]


@pytest.mark.parametrize("overlap", [False, True], ids=["disjoint", "overlapping"])
def test_windows_fixed_t(overlap):
    from event_utils_b200.representations.voxel_grid import voxel_grids_fixed_t_torch
    B = 5
    if overlap:
        # stamps k/1024: the searchsorted end of window 14 (0.1 * 14 + 0.1) reaches past the start of window 15
        # (0 + 15 * 0.1 in np.arange), so event 1536 belongs to both
        xs, ys, ts, ps = _window_events(4097, 32, ts=(np.arange(4097) / 1024).astype(np.float32))
        t = 0.1
    else:
        xs, ys, ts, ps = _window_events(10000, 33)
        t = 0.07
    bounds = _fixed_t_bounds(ts, t)
    overlaps = any(bounds[w][1] > bounds[w + 1][0] for w in range(len(bounds) - 1))
    assert overlaps == overlap
    _windows_case(xs, ys, ts, ps, B, lambda x, y, tt, p: voxel_grids_fixed_t_torch(x, y, tt, p, B, t, sensor_size=(H, W)),
                  bounds, "fixed_t")


def test_timesync():
    from event_utils_b200.representations.voxel_grid import events_to_voxel_timesync_torch
    B = 4
    xs, ys, ts, ps = _window_events(5000, 34)
    np_ts = ts.cpu().numpy()
    bounds = [(int(np.searchsorted(np_ts, 0.2)), int(np.searchsorted(np_ts, 0.65)))]
    _windows_case(xs, ys, ts, ps, B,
                  lambda x, y, t, p: [events_to_voxel_timesync_torch(x, y, t, p, B, 0.2, 0.65, sensor_size=(H, W))],
                  bounds, "timesync")


def test_outputs_unchanged_and_no_graph_without_grad():
    """The grad path runs the plain path's kernels (the sums agree up to the order their atomic additions land in);
    without grad mode, or when only xs / ys (or ps of the neg/pos split) require grad, no graph is recorded."""
    for case in CASES:
        for device in ("cuda", "cpu"):
            inputs = to(scene(case), device)
            plain = forward(case, ours(), inputs)
            assert all(o.grad_fn is None for o in plain)
            leaves = dict(inputs, ts=inputs["ts"].clone().requires_grad_(True))
            graded = forward(case, ours(), leaves)
            with torch.no_grad():
                nograd = forward(case, ours(), leaves)
            for a, b, c in zip(plain, graded, nograd):
                assert b.grad_fn is not None and c.grad_fn is None, case["name"]
                assert b.device == a.device
                assert_close_to_max(b.detach().cpu().numpy(), a.cpu().numpy(), 1e-6, case["name"])
                assert_close_to_max(c.cpu().numpy(), a.cpu().numpy(), 1e-6, case["name"])
            xy = dict(inputs, xs=inputs["xs"].clone().requires_grad_(True), ys=inputs["ys"].clone().requires_grad_(True))
            assert all(o.grad_fn is None for o in forward(case, ours(), xy)), case["name"]
            if case.get("negpos"):
                p = dict(inputs, ps=inputs["ps"].clone().requires_grad_(True))
                assert all(o.grad_fn is None for o in forward(case, ours(), p)), case["name"]


def test_backward_does_not_synchronise():
    """backward() of the grid, the neg/pos pair and the windows reads nothing back to the host."""
    from event_utils_b200.representations.voxel_grid import voxel_grids_fixed_n_torch
    voxel, negpos = ours()
    xs, ys, ts0, ps0 = _window_events(10000, 35)
    for what in ("voxel", "negpos", "fixed_n"):
        ts, ps = ts0.clone().requires_grad_(True), ps0.clone().requires_grad_(True)
        if what == "voxel":
            out = [voxel(xs, ys, ts, ps, 5, sensor_size=(H, W))]
        elif what == "negpos":
            out = list(negpos(xs, ys, ts, ps, 5, sensor_size=(H, W)))
        else:
            out = voxel_grids_fixed_n_torch(xs, ys, ts, ps, 5, 900, sensor_size=(H, W))
        loss = sum((o * o).sum() for o in out)
        torch.cuda.set_sync_debug_mode("error")
        try:
            loss.backward()
        finally:
            torch.cuda.set_sync_debug_mode(0)
        assert ts.grad is not None, what


def test_input_forms():
    """(N,1) shapes, a `device=` move, columns of one (N,4) tensor (the AoS path)."""
    voxel = ours()[0]
    case = next(c for c in CASES if c["name"] == "b5")
    a = to(scene(case), "cuda")
    B = case["B"]
    R = torch.randn(B, H, W, generator=torch.Generator().manual_seed(3))
    grads = []
    for fn, shape, dev in ((voxel, (-1, 1), "cpu"), (P.events_to_voxel_torch, (-1,), None)):
        ts = a["ts"].reshape(shape).clone().requires_grad_(True)
        ps = a["ps"].reshape(shape).clone().requires_grad_(True)
        xs, ys = a["xs"].reshape(shape), a["ys"].reshape(shape)
        grid = fn(xs, ys, ts, ps, B, device=dev, sensor_size=(H, W)) if fn is voxel else \
            fn(xs.reshape(-1), ys.reshape(-1), ts.reshape(-1), ps.reshape(-1), B, sensor_size=(H, W))
        assert grid.device.type == (dev or "cuda")
        (grid * R.to(grid.device)).sum().backward()
        grads.append((ts.grad, ps.grad))
    for (g, pg, what) in zip(grads[0], grads[1], ("ts", "ps")):
        assert g.shape == (pg.shape[0], 1) and g.device == pg.device
        if what == "ts":
            assert_grad_t(g, pg, (0, pg.shape[0] - 1), "(N,1)")
        else:
            assert_close_to_max(g.reshape(-1).cpu().numpy(), pg.cpu().numpy(), 1e-5, "(N,1) ps")
    # (N,4) record tensor: every column a view of it
    ev_grads = []
    for fn in (voxel, P.events_to_voxel_torch):
        ev = torch.stack([a["xs"], a["ys"], a["ts"], a["ps"]], 1).contiguous().requires_grad_(True)
        xs, ys, ts, ps = ev.unbind(1)
        grid = fn(xs, ys, ts, ps, B, sensor_size=(H, W))
        (grid * R.cuda()).sum().backward()
        ev_grads.append(ev.grad)
    g, pg = ev_grads
    assert (g[:, :2] == 0).all()
    assert_grad_t(g[:, 2], pg[:, 2], (0, g.shape[0] - 1), "aos")
    assert_close_to_max(g[:, 3].cpu().numpy(), pg[:, 3].cpu().numpy(), 1e-5, "aos ps")


def test_chain_5m():
    """learned per-event weights and time offsets -> voxel grid (5x480x640) -> loss in torch -> backward(), at 5 M
    events: both get the port's gradients.  The loss's gradient is a function of the forward grid, which the two
    sides sum in different orders, so the chain agrees to 1e-4 of the largest gradient."""
    n, B, Hs, Ws = 5_000_000, 5, 480, 640
    g = torch.Generator(device="cuda").manual_seed(7)
    xs = torch.rand(n, device="cuda", generator=g) * Ws
    ys = torch.rand(n, device="cuda", generator=g) * Hs
    ts = torch.sort(torch.rand(n, device="cuda", generator=g))[0] * 0.05
    ps = (torch.rand(n, device="cuda", generator=g) < 0.5).float() * 2 - 1
    w0 = 1 + 0.1 * torch.randn(n, device="cuda", generator=g)
    off0 = 1e-4 * torch.randn(n, device="cuda", generator=g)
    R = torch.randn(B, Hs, Ws, device="cuda", generator=g)
    res = []
    for fn in (ours()[0], P.events_to_voxel_torch):
        w, off = w0.clone().requires_grad_(True), off0.clone().requires_grad_(True)
        grid = fn(xs, ys, ts + off, ps * w, B, sensor_size=(Hs, Ws))
        loss = (grid * R).sum() + 0.01 * (grid ** 2).sum()
        loss.backward()
        res.append((loss.item(), w.grad, off.grad))
    assert abs(res[0][0] - res[1][0]) <= 1e-4 * abs(res[1][0])
    assert_close_to_max(res[0][1].cpu().numpy(), res[1][1].cpu().numpy(), 1e-4, "weights")
    assert_grad_t(res[0][2], res[1][2], (0, n - 1), "offsets", rel=1e-4)
