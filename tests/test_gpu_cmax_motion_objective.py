"""The batched parametric contrast objective (evk_cmax_motion_objective_f32 / _grad_f32, motion_contrast_objective_torch)
against the f64 reference of tests/motion_objective_reference.py and against the single-window entries
(evk_cmax_warp_objective_f32 / evk_cmax_linvel_objective_f32) it restates per sample."""
import ctypes

import numpy as np
import pytest
import torch

import motion_objective_reference as R
from conftest import assert_close_to_max
from edge_cases import exact_streams
from exact_bounds import gamma

pytestmark = pytest.mark.gpu

OBJ = {"variance": 0, "sos": 1, "soe": 2, "sosa": 5}
WARP = {"linvel": 3, "rotation": 1, "xyztheta": 2}
H, W = 60, 80
CENTRE = (40.0, 30.0)
# per model: parameters of up to five samples (the fourth sends most events off the canvas)
PARAMS = {"linvel": [(30.0, -20.0), (-55.0, 12.5), (5.0, 8.0), (900.0, -700.0), (0.0, 0.0)],
          "rotation": [(40.0, 30.0, 4.0), (35.0, 28.0, -6.0), (45.0, 33.0, 1.5), (10.0, 10.0, 40.0), (40.0, 30.0, 0.0)],
          "xyztheta": [(20.0, -10.0, 3.0, 2.0), (-30.0, 15.0, -2.0, 4.0), (5.0, 5.0, 0.5, -3.0), (600.0, -500.0, 30.0, 9.0),
                       (0.0, 0.0, 0.0, 0.0)]}


def _warp(kind, centre=CENTRE):
    from event_utils_b200.contrast_max import linvel_warp, pure_rotation_warp, xyztheta_warp
    return {"linvel": linvel_warp, "rotation": pure_rotation_warp, "xyztheta": lambda: xyztheta_warp(center=centre)}[kind]()


def batch_stream(seed, sizes, h=H, w=W):
    """concatenated samples; events in the sensor, d = t - t0 in [-0.1, 0] on a 2^-12 grid"""
    rng = np.random.default_rng(seed)
    n = sum(sizes)
    x = (rng.random(n) * (w - 1)).astype(np.float32)
    y = (rng.random(n) * (h - 1)).astype(np.float32)
    p = (rng.integers(0, 2, n) * 2 - 1).astype(np.float32)
    d = np.empty(n, np.float32)
    off = np.concatenate(([0], np.cumsum(sizes))).astype(np.int64)
    for b in range(len(sizes)):
        d[off[b]:off[b + 1]] = -np.sort(rng.integers(0, 410, sizes[b]))[::-1] / 4096.0
    return x, y, d, p, off


def torch_loss(kind, x, y, d, p, off, params, sigma, name, param=3.0, img_size=(H, W), centre=CENTRE):
    """motion_contrast_objective_torch on device inputs with ts = d and t0 = 0, so that d reaches the kernel unchanged"""
    from event_utils_b200.contrast_max import motion_contrast_objective_torch
    prm = torch.tensor(np.asarray(params, np.float64), device="cuda", requires_grad=True)
    ev = [torch.from_numpy(a).cuda() for a in (x, y, d, p)]
    f = motion_contrast_objective_torch(*ev, prm, _warp(kind, centre), t0=0.0, objective=name, blur_sigma=sigma,
                                        obj_param=param, img_size=img_size, batch_end_indices=torch.from_numpy(off[1:]).cuda())
    return f, prm


def run_forward(kind, x, y, d, p, off, params, sigma, name, param=3.0, h=H, w=W, centre=CENTRE):
    """the C entry directly: (f, iwe) as numpy"""
    from event_utils_b200 import _lib
    L = _lib.lib()
    B = len(params)
    X, Y, D, P, O = (torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (x, y, d, p, off))
    prm = torch.tensor(np.asarray(params, np.float64), device="cuda")
    f = torch.empty(B, dtype=torch.float64, device="cuda")
    iwe = torch.empty((B, h + 1, w + 1), device="cuda")
    ws = torch.empty(L.evk_cmax_motion_objective_workspace_bytes(B, h, w), dtype=torch.uint8, device="cuda")
    _lib.check(L.evk_cmax_motion_objective_f32(X.data_ptr(), Y.data_ptr(), D.data_ptr(), P.data_ptr(), O.data_ptr(), B, x.shape[0],
                                               WARP[kind], prm.data_ptr(), prm.shape[1], centre[0], centre[1], h, w, sigma,
                                               OBJ[name], param, f.data_ptr(), iwe.data_ptr(), ws.data_ptr(), ws.numel(), None))
    torch.cuda.synchronize()
    return f.cpu().numpy(), iwe.cpu().numpy()


def single_window(kind, x, y, d, p, prm, sigma, name, param, h, w, centre=CENTRE, grad=False):
    """evk_cmax_warp_objective_f32 / evk_cmax_linvel_objective_f32 on one window: (f, g or None, iwe)"""
    from event_utils_b200 import _lib
    L = _lib.lib()
    X, Y, D, P = (torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (x, y, d, p))
    ws = torch.empty(L.evk_cmax_workspace_bytes(h, w), dtype=torch.uint8, device="cuda")
    res = torch.zeros(16, dtype=torch.float64, device="cuda")
    iwe = torch.empty((h + 1, w + 1), device="cuda")
    flags = _lib.CMAX_WANT_GRAD if grad else 0
    if kind == "linvel":
        _lib.check(L.evk_cmax_linvel_objective_f32(X.data_ptr(), Y.data_ptr(), D.data_ptr(), P.data_ptr(), x.shape[0], 1.0, prm[0],
                                                   prm[1], h, w, h, w, sigma, flags, OBJ[name], param, res.data_ptr(),
                                                   iwe.data_ptr(), None, ws.data_ptr(), ws.numel(), None))
    else:
        model = np.array(list(prm) + (list(centre) if kind == "xyztheta" else []), np.float64)
        _lib.check(L.evk_cmax_warp_objective_f32(X.data_ptr(), Y.data_ptr(), D.data_ptr(), P.data_ptr(), x.shape[0], 1.0, WARP[kind],
                                                 model.ctypes.data, h, w, h, w, sigma, flags, OBJ[name], param, res.data_ptr(),
                                                 iwe.data_ptr(), ws.data_ptr(), ws.numel(), None))
    torch.cuda.synchronize()
    r = res.cpu().numpy()
    return r[0], (r[1:1 + len(prm)] if grad else None), iwe.cpu().numpy()


@pytest.mark.parametrize("kind", ["linvel", "rotation", "xyztheta"])
@pytest.mark.parametrize("name", ["variance", "sos", "soe", "sosa"])
@pytest.mark.parametrize("sigma", [0.0, 1.0, 3.0])
@pytest.mark.parametrize("batch", [1, 5])
def test_f_and_iwe_against_reference(kind, name, sigma, batch):
    sizes = [20000] if batch == 1 else [15000, 0, 9000, 20000, 1]
    x, y, d, p, off = batch_stream(7 + batch, sizes)
    params = PARAMS[kind][:batch]
    param = 0.3
    f, iwe = run_forward(kind, x, y, d, p, off, params, sigma, name, param)
    fr, iwer, _ = R.reference(kind, x, y, d, p, off, torch.tensor(params, dtype=torch.float64), sigma, name, param, (H, W), CENTRE)
    fr, iwer = fr.detach().numpy(), iwer.detach().numpy()
    for b in range(batch):
        assert_close_to_max(iwe[b], iwer[b], 1e-5, "iwe %d" % b)
        assert abs(f[b] - fr[b]) <= 1e-5 * max(abs(fr[b]), 1e-30), (b, f[b], fr[b])
    if batch == 5:
        assert (iwe[1] == 0).all()


@pytest.mark.parametrize("kind", ["linvel", "rotation", "xyztheta"])
@pytest.mark.parametrize("name", ["variance", "sos", "soe", "sosa"])
@pytest.mark.parametrize("sigma", [0.0, 1.0, 3.0])
def test_gradient_against_reference(kind, name, sigma):
    sizes = [15000, 0, 9000, 20000, 1]
    x, y, d, p, off = batch_stream(3, sizes)
    params = PARAMS[kind]
    param = 0.3
    f, prm = torch_loss(kind, x, y, d, p, off, params, sigma, name, param)
    g = torch.from_numpy(np.random.default_rng(5).standard_normal(len(sizes)))
    (f * g.cuda()).sum().backward()
    got = prm.grad.cpu().numpy()
    p64 = torch.tensor(params, dtype=torch.float64, requires_grad=True)
    fr, iwer, mag = R.reference(kind, x, y, d, p, off, p64, sigma, name, param, (H, W), CENTRE)
    (fr * g).sum().backward()
    ref = p64.grad.numpy()
    # to 1e-4 of the batch's largest component (a one-event sample's gradient is a near-total cancellation), and every
    # component within its own rounding bound
    assert_close_to_max(got, ref, 1e-4, "grad %s %s sigma %g" % (kind, name, sigma))
    M, cnt = R.grad_magnitude(kind, x, y, d, p, off, p64, sigma, name, param, g.numpy(), iwer.detach().numpy(), mag.numpy(),
                              (H, W), CENTRE)
    bound = gamma(cnt + 32) * M
    err = np.abs(got - ref)
    assert not (err > bound).any(), (err, bound)
    assert (got[1] == 0).all()


# the single-window gradient (EVK_CMAX_WANT_GRAD) is the exact derivative for these objectives; for the variance and sos
# with a blur it contracts the un-blurred IWE (objectives.py:256-264), which the batched loss does not
EXACT_SINGLE = [("variance", 0.0), ("sos", 0.0), ("soe", 0.0), ("soe", 1.0), ("sosa", 1.0), ("sosa", 3.0)]


@pytest.mark.parametrize("kind", ["linvel", "rotation", "xyztheta"])
def test_against_the_single_window_entries(kind):
    h, w = 180, 240
    centre = (120.0, 90.0)
    x, y, d, p, off = batch_stream(17, [40000, 25000, 60000], h, w)
    params = {"linvel": [(30.0, -20.0), (-55.0, 12.5), (5.0, 8.0)],
              "rotation": [(130.0, 85.0, 4.0), (100.0, 70.0, -6.0), (120.0, 90.0, 1.5)],
              "xyztheta": [(20.0, -10.0, 3.0, 2.0), (-30.0, 15.0, -2.0, 4.0), (5.0, 5.0, 0.5, -3.0)]}[kind]
    for name, sigma in EXACT_SINGLE + [("variance", 1.0), ("sos", 3.0)]:
        f, prm = torch_loss(kind, x, y, d, p, off, params, sigma, name, 0.3, (h, w), centre)
        f.sum().backward()
        _, iwe = run_forward(kind, x, y, d, p, off, params, sigma, name, 0.3, h, w, centre)
        grad = (name, sigma) in EXACT_SINGLE and kind != "linvel"
        for b in range(3):
            sl = slice(off[b], off[b + 1])
            fs, gs, iwes = single_window(kind, x[sl], y[sl], d[sl], p[sl], params[b], sigma, name, 0.3, h, w, centre, grad)
            assert_close_to_max(iwe[b], iwes, 1e-6, "iwe %s %d" % (kind, b))
            assert abs(f[b].item() - fs) <= 1e-6 * abs(fs), (kind, name, sigma, b, f[b].item(), fs)
            if grad:
                np.testing.assert_allclose(prm.grad[b].cpu().numpy(), gs, rtol=0, atol=1e-5 * np.abs(gs).max())


def test_exactly_summable_streams_bit_for_bit():
    """quarter-pixel warped coordinates (tests/edge_cases.py): every tap and pixel sum is exact, so the IWE equals the
    single-window entries' bit for bit, and so does f where its sums are exact too (variance, no blur)"""
    c = exact_streams(3, "cmax", 300001)
    h, w = c["Hs"], c["Ws"]
    x, y, t, p = (np.asarray(c[k], np.float32) for k in ("x", "y", "t", "p"))
    assert all(np.array_equal(a.astype(np.float64), c[k]) for a, k in zip((x, y, t, p), "xytp"))
    cut = [0, 100000, 100000, 300001]                 # three windows, one of them empty
    off = np.array(cut, np.int64)
    centre = (20.0, 12.0)
    models = {"linvel": [(c["vx"], c["vy"])] * 3, "xyztheta": [(c["vx"], c["vy"], 0.0, 0.0)] * 3,
              "rotation": [(20.0, 12.0, 0.0), (21.0, 13.5, 0.0), (22.25, 10.0, 0.0)]}
    for kind, params in models.items():
        for name, sigma in (("variance", 0.0), ("variance", 1.0), ("sos", 0.0), ("sos", 1.0)):   # exp(G) overflows here
            f, iwe = run_forward(kind, x, y, t, p, off, params, sigma, name, 3.0, h, w, centre)
            for b in (0, 2):
                sl = slice(off[b], off[b + 1])
                fs, _, iwes = single_window(kind, x[sl], y[sl], t[sl], p[sl], params[b], sigma, name, 3.0, h, w, centre)
                assert np.array_equal(iwe[b], iwes), (kind, name, b)
                if name == "variance" and sigma == 0.0:
                    assert f[b] == fs, (kind, b, f[b], fs)
                else:
                    assert abs(f[b] - fs) <= 1e-6 * abs(fs), (kind, name, sigma, b, f[b], fs)
            assert (iwe[1] == 0).all()


def _sparse_footprints(kind, prm, centre, h, w, seed, n=40000, gap=3):
    """Events whose warped footprints lie at least `gap` pixels apart (judged on the f32 warp of the reference, which
    is within an ulp of the kernel's): every IWE pixel then receives at most one tap, so its sum is that tap, in any
    order.  d on a 2^-12 grid in [-0.1, 0], p = +-1."""
    rng = np.random.default_rng(seed)
    x = (rng.random(n) * (w - 1)).astype(np.float32)
    y = (rng.random(n) * (h - 1)).astype(np.float32)
    d = (-rng.integers(0, 410, n) / 4096.0).astype(np.float32)
    p = (rng.integers(0, 2, n) * 2 - 1).astype(np.float32)
    xw, yw = R.warp_f32(kind, x, y, d, prm, centre)
    ok = R.contributes(xw, yw, h, w)
    taken = np.zeros((h + 1 + 2 * gap, w + 1 + 2 * gap), bool)
    pick = []
    for i in np.flatnonzero(ok):
        cx, cy = int(np.floor(xw[i])) + gap, int(np.floor(yw[i])) + gap
        if taken[cy - gap:cy + gap + 1, cx - gap:cx + gap + 1].any():
            continue
        taken[cy, cx] = True
        pick.append(i)
    pick = np.array(pick)
    return tuple(a[pick] for a in (x, y, d, p))


def test_non_overlapping_footprints_bit_for_bit_under_every_model():
    """Non-trivial rotation and 4-DoF motion (and linvel): with at most one tap per pixel the IWE equals the
    single-window entries' bit for bit whatever the warp's arithmetic, since both take their taps from model_taps"""
    h, w = 180, 240
    centre = (120.0, 90.0)
    models = {"linvel": (30.0, -20.0), "rotation": (130.0, 85.0, 4.0), "xyztheta": (20.0, -10.0, 3.0, 2.0)}
    for kind, prm in models.items():
        x, y, d, p = _sparse_footprints(kind, prm, centre, h, w, seed=37)
        assert x.shape[0] > 1200, x.shape
        xd, yd, dd, pd, offd = batch_stream(38, [30000], h, w)      # a dense second sample in the same batch
        off = np.array([0, x.shape[0], x.shape[0] + 30000], np.int64)
        cat = [np.concatenate(a) for a in ((x, xd), (y, yd), (d, dd), (p, pd))]
        for name, sigma in (("variance", 0.0), ("soe", 1.0)):
            f, iwe = run_forward(kind, *cat, off, [prm, prm], sigma, name, 0.3, h, w, centre)
            fs, _, iwes = single_window(kind, x, y, d, p, prm, sigma, name, 0.3, h, w, centre)
            assert np.array_equal(iwe[0], iwes), (kind, name)
            assert (iwe[0] != 0).sum() >= 4 * 1000          # ~4 distinct pixels per event
            assert abs(f[0] - fs) <= 1e-6 * abs(fs), (kind, name, sigma, f[0], fs)


@pytest.mark.parametrize("kind", ["linvel", "rotation", "xyztheta"])
def test_large_canvas_empty_and_one_event_samples(kind):
    """480x640 (beyond the 51 200-pixel canvas of the single-window gradient pass), with an empty and a one-event sample"""
    h, w = 480, 640
    centre = (320.0, 240.0)
    x, y, d, p, off = batch_stream(23, [200000, 0, 1, 150000], h, w)
    params = {"linvel": [(60.0, -40.0), (1.0, 1.0), (0.0, 0.0), (-20.0, 30.0)],
              "rotation": [(320.0, 240.0, 3.0), (0.0, 0.0, 0.0), (320.0, 240.0, 0.0), (300.0, 250.0, -2.0)],
              "xyztheta": [(60.0, -40.0, 2.0, 1.0), (0.0, 0.0, 0.0, 0.0), (0.0, 0.0, 0.0, 0.0), (-20.0, 30.0, -1.0, 2.0)]}[kind]
    f, prm = torch_loss(kind, x, y, d, p, off, params, 1.0, "variance", img_size=(h, w), centre=centre)
    g = torch.tensor([1.0, 2.0, 3.0, -1.0], dtype=torch.float64, device="cuda")
    (f * g).sum().backward()
    got = prm.grad.cpu().numpy()
    p64 = torch.tensor(params, dtype=torch.float64, requires_grad=True)
    fr, _, _ = R.reference(kind, x, y, d, p, off, p64, 1.0, "variance", img_size=(h, w), centre=centre)
    (fr * g.cpu()).sum().backward()
    ref = p64.grad.numpy()
    fc = f.detach().cpu().numpy()
    for b in (0, 2, 3):
        assert abs(fc[b] - fr[b].item()) <= 1e-5 * abs(fr[b].item()), (b, fc[b], fr[b].item())
        assert_close_to_max(got[b], ref[b], 1e-4, "sample %d" % b)
    assert fc[1] == 0.0 and (got[1] == 0).all()
    assert fc[2] != 0.0


def test_nan_isolation():
    sizes = [20000, 15000, 18000]
    x, y, d, p, off = batch_stream(29, sizes)
    for kind in ("linvel", "rotation", "xyztheta"):
        params = PARAMS[kind][:3]
        f0, prm0 = torch_loss(kind, x, y, d, p, off, params, 1.0, "soe")
        f0.sum().backward()
        # a NaN event in sample 1: it contributes nothing; a NaN parameter of sample 2: none of its events does
        xb = x.copy()
        xb[off[1] + 5] = np.nan
        bad = [list(q) for q in params]
        bad[2][0] = float("nan")
        f1, prm1 = torch_loss(kind, xb, y, d, p, off, bad, 1.0, "soe")
        f1.sum().backward()
        fa, fb = f0.detach().cpu().numpy(), f1.detach().cpu().numpy()
        ga, gb = prm0.grad.cpu().numpy(), prm1.grad.cpu().numpy()
        assert np.isfinite(fb).all() and np.isfinite(gb[:2]).all()
        assert abs(fb[0] - fa[0]) <= 1e-6 * abs(fa[0])
        assert_close_to_max(gb[0], ga[0], 1e-5, kind)
        assert abs(fb[1] - fa[1]) <= 1e-3 * abs(fa[1])           # one event of 15000 fewer
        e = np.zeros(0, np.float32)
        fe, _ = run_forward(kind, e, e, e, e, np.array([0, 0], np.int64), [bad[2]], 1.0, "soe")
        assert fb[2] == pytest.approx(fe[0], rel=1e-12)         # the image of no event


def test_inputs_cpu_events_dtypes_and_expanded_params():
    from event_utils_b200.contrast_max import motion_contrast_objective_torch, pure_rotation_warp
    sizes = [20000, 15000]
    x, y, d, p, off = batch_stream(31, sizes)
    t = d.astype(np.float64) + 1000.0                        # t - t0 formed in f64, then f32: d exactly
    warp = pure_rotation_warp()
    base = torch.tensor([40.0, 30.0, 4.0], dtype=torch.float64)
    ref = None
    for dtype in (torch.float64, torch.float32):
        for expanded in (False, True):
            prm = base.to(dtype).cuda().requires_grad_(True)
            arg = prm.expand(2, 3) if expanded else torch.stack([prm, prm])
            f = motion_contrast_objective_torch(x, y, t, p, arg, warp, t0=[1000.0, 1000.0], img_size=(H, W),
                                                batch_end_indices=list(off[1:]))
            assert f.shape == (2,) and f.dtype == dtype and f.device == prm.device
            f.sum().backward()
            assert prm.grad.dtype == dtype and prm.grad.shape == (3,)
            got = (f.detach().double().cpu().numpy(), prm.grad.double().cpu().numpy())
            if ref is None:
                ref = got
            else:
                np.testing.assert_allclose(got[0], ref[0], rtol=1e-6)
                np.testing.assert_allclose(got[1], ref[1], rtol=1e-4, atol=1e-4 * np.abs(ref[1]).max())
    # CPU params and events: the result and the gradient come back on the CPU
    prm = base.clone().requires_grad_(True)
    f = motion_contrast_objective_torch(torch.from_numpy(x), torch.from_numpy(y), torch.from_numpy(t), torch.from_numpy(p),
                                        prm.expand(2, 3), warp, t0=1000.0, img_size=(H, W), batch_end_indices=list(off[1:]))
    f.sum().backward()
    assert f.device.type == "cpu" and prm.grad.device.type == "cpu"
    np.testing.assert_allclose(f.detach().numpy(), ref[0], rtol=1e-6)         # f32 image sums in any order
    # one sample as a (K,) vector, t0 = None: each sample's last stamp
    f1 = motion_contrast_objective_torch(x[:sizes[0]], y[:sizes[0]], t[:sizes[0]], p[:sizes[0]], base.cuda(), warp, img_size=(H, W))
    assert f1.shape == (1,) and abs(f1.item() - ref[0][0]) <= 1e-6 * abs(ref[0][0])


def test_no_host_round_trips_and_constant_launch_count():
    from event_utils_b200 import _lib
    from event_utils_b200.contrast_max import motion_contrast_objective_torch, xyztheta_warp
    L = _lib.lib()
    counts = []
    for sizes in ([40000], [2500] * 16):
        x, y, d, p, off = batch_stream(2, sizes)
        params = np.tile(np.array([[20.0, -10.0, 3.0, 2.0]]), (len(sizes), 1))
        torch_loss("xyztheta", x, y, d, p, off, params, 1.0, "soe")       # warm-up: scratch buffers, modules
        prm = torch.tensor(params, device="cuda", requires_grad=True)
        ev = [torch.from_numpy(a).cuda() for a in (x, y, d, p)]
        ends = torch.from_numpy(off[1:]).cuda()
        warp = xyztheta_warp(center=CENTRE)
        torch.cuda.synchronize()
        L.evk_prof_enable(1)
        torch.cuda.set_sync_debug_mode("error")
        try:
            f = motion_contrast_objective_torch(*ev, prm, warp, objective="soe", blur_sigma=1.0, img_size=(H, W),
                                                batch_end_indices=ends)
            f.sum().backward()
        finally:
            torch.cuda.set_sync_debug_mode(0)
        ms, timed, launches = ctypes.c_double(), ctypes.c_longlong(), ctypes.c_longlong()
        _lib.check(L.evk_prof_collect(ctypes.byref(ms), ctypes.byref(timed), ctypes.byref(launches)))
        L.evk_prof_enable(0)
        assert torch.isfinite(prm.grad).all()
        counts.append(launches.value)
    assert counts[0] == counts[1] and counts[0] > 0, counts


def _scene(rng, n_pts, per_pt, centre, radius):
    ang, rad = rng.uniform(0, 2 * np.pi, n_pts), radius * np.sqrt(rng.uniform(0.05, 1, n_pts))
    x0, y0 = np.repeat(centre[0] + rad * np.cos(ang), per_pt), np.repeat(centre[1] + rad * np.sin(ang), per_pt)
    ps = np.repeat(rng.integers(0, 2, n_pts) * 2.0 - 1.0, per_pt)
    order = rng.permutation(x0.size)
    return x0[order], y0[order], ps[order]


def _windows(kind, truths, duration, rng):
    """one window per true motion: a scene of points seen during `duration`, moving with that motion"""
    xs, ys, ts, ps, ends = [], [], [], [], []
    for tr in truths:
        centre = (tr[0], tr[1]) if kind == "rotation" else (120.0, 90.0)
        x0, y0, p = _scene(rng, 300, 200, centre, 60.0)
        t = np.sort(rng.uniform(0, duration, x0.size))
        dt = t - t[-1]
        if kind == "linvel":
            x, y = x0 + dt * tr[0], y0 + dt * tr[1]
        elif kind == "rotation":
            a = tr[2] * dt
            u, v = x0 - tr[0], y0 - tr[1]
            x, y = tr[0] + np.cos(a) * u - np.sin(a) * v, tr[1] + np.sin(a) * u + np.cos(a) * v
        else:
            hx, hy, hz, th = tr
            bx, by = (x0 - 120.0) + dt * hx, (y0 - 90.0) + dt * hy
            m00, m01, m10, m11 = 1 - dt * hz, dt * th, -dt * th, 1 - dt * hz
            det = m00 * m11 - m01 * m10
            x, y = 120.0 + (m11 * bx - m01 * by) / det, 90.0 + (m00 * by - m10 * bx) / det
        xs.append(x), ys.append(y), ts.append(t), ps.append(p)
        ends.append(sum(len(a) for a in xs))
    return [np.concatenate(a) for a in (xs, ys, ts, ps)], ends


@pytest.mark.parametrize("kind", ["linvel", "rotation", "xyztheta"])
def test_one_optimiser_recovers_every_window(kind):
    """8 windows with distinct motions; Adam on the summed loss from a start near the truth finds each window's own"""
    from event_utils_b200.contrast_max import motion_contrast_objective_torch
    rng = np.random.default_rng({"linvel": 41, "rotation": 42, "xyztheta": 43}[kind])
    if kind == "linvel":
        truths = np.column_stack((rng.uniform(20, 60, 8) * rng.choice([-1, 1], 8), rng.uniform(20, 60, 8) * rng.choice([-1, 1], 8)))
        scale, duration = np.array([1.0, 1.0]), 0.2
    elif kind == "rotation":
        truths = np.column_stack((rng.uniform(110, 130, 8), rng.uniform(80, 100, 8), rng.uniform(3, 8, 8) * rng.choice([-1, 1], 8)))
        scale, duration = np.array([0.5, 0.5, 0.05]), 0.05
    else:
        truths = np.column_stack((rng.uniform(15, 30, 8) * rng.choice([-1, 1], 8), rng.uniform(15, 30, 8) * rng.choice([-1, 1], 8),
                                  rng.uniform(2, 4, 8), rng.uniform(2, 4, 8) * rng.choice([-1, 1], 8)))
        scale, duration = np.array([1.0, 1.0, 0.1, 0.1]), 0.2
    (x, y, t, p), ends = _windows(kind, truths, duration, rng)
    ev = [torch.from_numpy(a).float().cuda() for a in (x, y, p)]
    tt = torch.from_numpy(t).cuda()
    start = truths * (1 + rng.uniform(-0.15, 0.15, truths.shape)) if kind != "rotation" else \
        np.column_stack((truths[:, :2] + rng.uniform(-2, 2, (8, 2)), truths[:, 2] * rng.uniform(0.85, 1.15, 8)))
    base = torch.tensor(start, device="cuda")
    s = torch.tensor(scale, device="cuda")
    z = torch.zeros_like(base, requires_grad=True)
    opt = torch.optim.Adam([z], lr=0.3)
    sched = torch.optim.lr_scheduler.CosineAnnealingLR(opt, T_max=300, eta_min=0.003)
    warp = _warp(kind, (120.0, 90.0))
    for _ in range(300):
        opt.zero_grad()
        f = motion_contrast_objective_torch(ev[0], ev[1], tt, ev[2], base + s * z, warp, blur_sigma=1.0,
                                            batch_end_indices=ends)
        f.sum().backward()
        opt.step()
        sched.step()
    got = (base + s * z).detach().cpu().numpy()
    if kind == "rotation":
        assert np.all(np.abs(got[:, 2] - truths[:, 2]) <= 0.03 * np.abs(truths[:, 2])), (got, truths)
        assert np.all(np.hypot(got[:, 0] - truths[:, 0], got[:, 1] - truths[:, 1]) <= 2.0), (got, truths)
    else:
        assert np.all(np.abs(got - truths) <= 0.05 * np.abs(truths)), (got, truths)
