"""The batched parametric average-timestamp loss (evk_motion_timestamp_objective_f32 / _grad_f32,
motion_timestamp_objective_torch) against the f64 reference of tests/motion_timestamp_reference.py, the unchanged motion
contrast and timestamp-image entries, zhu_timestamp_objective and the dense-flow timestamp loss."""
import ctypes

import numpy as np
import pytest
import torch

import motion_timestamp_reference as R
from conftest import assert_close_to_max
from edge_cases import exact_streams
from exact_bounds import gamma

pytestmark = pytest.mark.gpu

WARP = {"linvel": 3, "rotation": 1, "xyztheta": 2}
H, W = 60, 80
CENTRE = (40.0, 30.0)
# per model: parameters of up to five samples (the fourth sends most events off the canvas)
PARAMS = {"linvel": [(30.0, -20.0), (-55.0, 12.5), (5.0, 8.0), (900.0, -700.0), (0.0, 0.0)],
          "rotation": [(40.0, 30.0, 4.0), (35.0, 28.0, -6.0), (45.0, 33.0, 1.5), (10.0, 10.0, 40.0), (40.0, 30.0, 0.0)],
          "xyztheta": [(20.0, -10.0, 3.0, 2.0), (-30.0, 15.0, -2.0, 4.0), (5.0, 5.0, 0.5, -3.0), (600.0, -500.0, 30.0, 9.0),
                       (0.0, 0.0, 0.0, 0.0)]}
SIZES5 = [15000, 0, 9000, 20000, 1]      # an empty and a one-event window


def _warp(kind, centre=CENTRE):
    from event_utils_b200.contrast_max import linvel_warp, pure_rotation_warp, xyztheta_warp
    return {"linvel": linvel_warp, "rotation": pure_rotation_warp, "xyztheta": lambda: xyztheta_warp(center=centre)}[kind]()


def batch_stream(seed, sizes, h=H, w=W):
    """concatenated samples; events in the sensor, sorted stamps t over 0.1 time units per sample, d = t - the sample's
    last stamp"""
    rng = np.random.default_rng(seed)
    n = sum(sizes)
    x = (rng.random(n) * (w - 1)).astype(np.float32)
    y = (rng.random(n) * (h - 1)).astype(np.float32)
    p = (rng.integers(0, 2, n) * 2 - 1).astype(np.float32)
    t = np.empty(n, np.float32)
    d = np.empty(n, np.float32)
    off = np.concatenate(([0], np.cumsum(sizes))).astype(np.int64)
    for b in range(len(sizes)):
        t[off[b]:off[b + 1]] = np.sort(rng.random(sizes[b])) * 0.1 + b
        if sizes[b]:
            d[off[b]:off[b + 1]] = t[off[b]:off[b + 1]] - t[off[b + 1] - 1]
    return x, y, t, d, p, off


def run_forward(kind, x, y, d, tau, p, off, params, sigma, h=H, w=W, centre=CENTRE):
    """the C entry directly: (f, T, C) as numpy"""
    from event_utils_b200 import _lib
    L = _lib.lib()
    B = len(params)
    X, Y, D, U, P, O = (torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (x, y, d, tau, p, off))
    prm = torch.tensor(np.asarray(params, np.float64), device="cuda")
    f = torch.empty(B, dtype=torch.float64, device="cuda")
    T = torch.empty((B, 2, h + 1, w + 1), device="cuda")
    C = torch.empty_like(T)
    ws = torch.empty(L.evk_motion_timestamp_objective_workspace_bytes(B, h, w), dtype=torch.uint8, device="cuda")
    _lib.check(L.evk_motion_timestamp_objective_f32(X.data_ptr(), Y.data_ptr(), D.data_ptr(), U.data_ptr(), P.data_ptr(),
                                                    O.data_ptr(), B, x.shape[0], WARP[kind], prm.data_ptr(), prm.shape[1],
                                                    centre[0], centre[1], h, w, sigma, f.data_ptr(), T.data_ptr(),
                                                    C.data_ptr(), ws.data_ptr(), ws.numel(), None))
    torch.cuda.synchronize()
    return f.cpu().numpy(), T.cpu().numpy(), C.cpu().numpy()


def torch_loss(kind, x, y, t, p, off, params, sigma, reverse=False, img_size=(H, W), centre=CENTRE, t0=None):
    from event_utils_b200.contrast_max import motion_timestamp_objective_torch
    prm = torch.tensor(np.asarray(params, np.float64), device="cuda", requires_grad=True)
    ev = [torch.from_numpy(a).cuda() for a in (x, y, t, p)]
    f = motion_timestamp_objective_torch(*ev, prm, _warp(kind, centre), t0=t0, blur_sigma=sigma, timestamp_reverse=reverse,
                                         img_size=img_size, batch_end_indices=torch.from_numpy(off[1:]).cuda())
    return f, prm


@pytest.mark.parametrize("kind", ["linvel", "rotation", "xyztheta"])
@pytest.mark.parametrize("sigma", [0.0, 2.0])
@pytest.mark.parametrize("reverse", [False, True])
@pytest.mark.parametrize("batch", [1, 5])
def test_against_reference(kind, sigma, reverse, batch):
    """f, T and C to 1e-5 of their largest value (f32 sums), as the dense-flow loss; the parameter gradient (through the
    torch function, whose stamps are the reference's tau bit for bit) within its per-component rounding bound"""
    sizes = [20000] if batch == 1 else SIZES5
    x, y, t, d, p, off = batch_stream(7 + batch, sizes)
    params = PARAMS[kind][:batch]
    tau = R.tau_f32(t, off, reverse)
    f, T, C = run_forward(kind, x, y, d, tau, p, off, params, sigma)
    p64 = torch.tensor(params, dtype=torch.float64, requires_grad=True)
    fr, Tr, Cr = R.reference(kind, x, y, d, tau, p, off, p64, sigma, (H, W), CENTRE)
    for b in range(batch):
        assert_close_to_max(T[b], Tr[b].detach().numpy(), 1e-5, "T %d" % b)
        assert_close_to_max(C[b], Cr[b].detach().numpy(), 1e-5, "C %d" % b)
        assert abs(f[b] - fr[b].item()) <= 1e-5 * max(abs(fr[b].item()), 1e-30), (b, f[b], fr[b].item())
    if batch == 5:
        assert (T[1] == 0).all() and (C[1] == 1).all() and f[1] == 0
        assert (T[4] == 0).all() and f[4] == 0                   # tau of a lone event is 0
        xw, yw = R.warp_f32(kind, x[off[3]:off[4]], y[off[3]:off[4]], d[off[3]:off[4]], params[3], CENTRE)
        assert R.contributes(xw, yw, H, W).mean() < 0.5          # most of window 3 leaves the canvas
    ft, prm = torch_loss(kind, x, y, t, p, off, params, sigma, reverse)
    np.testing.assert_allclose(ft.detach().cpu().numpy(), f, rtol=1e-6)
    g = torch.from_numpy(np.random.default_rng(5).standard_normal(batch))
    (ft * g.cuda()).sum().backward()
    got = prm.grad.cpu().numpy()
    (fr * g).sum().backward()
    ref = p64.grad.numpy()
    assert_close_to_max(got, ref, 1e-4, "grad %s sigma %g reverse %s" % (kind, sigma, reverse))
    M, cnt = R.grad_magnitude(kind, x, y, d, tau, p, off, p64, sigma, g.numpy(), Tr.detach().numpy(), Cr.detach().numpy(),
                              (H, W), CENTRE)
    bound = gamma(cnt + 32) * M
    err = np.abs(got - ref)
    assert not (err > bound).any(), (err, bound)
    if batch == 5:
        assert (got[1] == 0).all() and (got[4] == 0).all()


def _tsimg_entry(xw, yw, ts, p, h, w):
    """evk_timestamp_image_counts_f32 on the (h+1, w+1) canvas with t_first = 0 and t_last = 32, whose normalised stamp
    (t - 0) / (32 + 1e-6f) is t / 32 exactly in f32"""
    from event_utils_b200 import _lib
    L = _lib.lib()
    X, Y, Tt, P = (torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda() for a in (xw, yw, ts, p))
    out = [torch.empty((h + 1, w + 1), device="cuda") for _ in range(4)]
    ws = torch.empty(L.evk_timestamp_image_workspace_bytes(h + 1, w + 1), dtype=torch.uint8, device="cuda")
    oob = torch.zeros(1, dtype=torch.int64, device="cuda")
    _lib.check(L.evk_timestamp_image_counts_f32(X.data_ptr(), Y.data_ptr(), Tt.data_ptr(), P.data_ptr(), X.shape[0], 0.0, 32.0,
                                                h + 1, w + 1, float(w), float(h), 0, *(o.data_ptr() for o in out),
                                                ws.data_ptr(), ws.numel(), oob.data_ptr(), None))
    torch.cuda.synchronize()
    assert oob.item() == 0
    pos, neg, cpos, cneg = (o.cpu().numpy() for o in out)
    return np.stack([pos, neg]), np.stack([cpos, cneg])


def _motion_iwe(kind, x, y, d, p, off, params, h, w, centre):
    """the IWE of the unchanged evk_cmax_motion_objective_f32 (variance, no blur)"""
    from event_utils_b200 import _lib
    L = _lib.lib()
    B = len(params)
    X, Y, D, P, O = (torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (x, y, d, p, off))
    prm = torch.tensor(np.asarray(params, np.float64), device="cuda")
    f = torch.empty(B, dtype=torch.float64, device="cuda")
    iwe = torch.empty((B, h + 1, w + 1), device="cuda")
    ws = torch.empty(L.evk_cmax_motion_objective_workspace_bytes(B, h, w), dtype=torch.uint8, device="cuda")
    _lib.check(L.evk_cmax_motion_objective_f32(X.data_ptr(), Y.data_ptr(), D.data_ptr(), P.data_ptr(), O.data_ptr(), B, x.shape[0],
                                               WARP[kind], prm.data_ptr(), prm.shape[1], centre[0], centre[1], h, w, 0.0, 0, 0.0,
                                               f.data_ptr(), iwe.data_ptr(), ws.data_ptr(), ws.numel(), None))
    torch.cuda.synchronize()
    return iwe.cpu().numpy()


def test_exactly_summable_streams_bit_for_bit():
    """quarter-pixel warped coordinates (tests/edge_cases.py) and stamps tau on a 1/4 grid: every tap and every pixel sum
    is exact in f32, so C_s - 1 equals the IWE of the motion contrast loss over the polarity-s events with p = 1, and T
    and C equal the timestamp-image entry applied to the f32-warped positions, bit for bit"""
    c = exact_streams(3, "cmax", 300001)
    h, w = c["Hs"], c["Ws"]
    x, y, d, p = (np.asarray(c[k], np.float32) for k in ("x", "y", "t", "p"))
    n = x.shape[0]
    tau = (np.random.default_rng(8).integers(0, 5, n) / 4.0).astype(np.float32)
    off = np.array([0, 100000, 100000, n], np.int64)       # three windows, one of them empty
    centre = (20.0, 12.0)
    models = {"linvel": [(c["vx"], c["vy"])] * 3, "xyztheta": [(c["vx"], c["vy"], 0.0, 0.0)] * 3,
              "rotation": [(20.0, 12.0, 0.0), (21.0, 13.5, 0.0), (22.25, 10.0, 0.0)]}
    for kind, params in models.items():
        f, T, C = run_forward(kind, x, y, d, tau, p, off, params, 0.0, h, w, centre)
        for s, sel in enumerate((p > 0, p <= 0)):
            iwe = _motion_iwe(kind, x, y, d, sel.astype(np.float32), off, params, h, w, centre)
            assert np.array_equal(C[:, s] - 1, iwe), (kind, s)
        for b in (0, 2):
            sl = slice(off[b], off[b + 1])
            xw, yw = R.warp_f32(kind, x[sl], y[sl], d[sl], params[b], centre)
            k = R.contributes(xw, yw, h, w)
            assert k.mean() > 0.9
            Te, Ce = _tsimg_entry(xw[k], yw[k], 32.0 * tau[sl][k], p[sl][k], h, w)
            assert np.array_equal(T[b], Te) and np.array_equal(C[b], Ce), (kind, b)
        assert (T[1] == 0).all() and (C[1] == 1).all()


@pytest.mark.parametrize("kind", ["linvel", "rotation", "xyztheta"])
@pytest.mark.parametrize("sigma", [0.0, 2.0])
def test_against_zhu_timestamp_objective(kind, sigma):
    """180x240 with every event strictly inside: f = -zhu_timestamp_objective's f.  That path warps and normalises in
    f64; this one warps in f32, which moves each x', y' < 241 by a few ulp(256) = 2^-16 px and each tap weight by as
    much; T is a weighted mean of the stamps and f = sum G^2, so the relative difference of f stays below 4 * 2^-15,
    the dense-flow loss's bound."""
    from event_utils_b200.contrast_max import motion_timestamp_objective_torch, zhu_timestamp_objective
    h, w = 180, 240
    centre = (120.0, 90.0)
    rng = np.random.default_rng(4)
    n = 200000
    x = (40 + rng.random(n) * (w - 81)).astype(np.float32).astype(np.float64)
    y = (40 + rng.random(n) * (h - 81)).astype(np.float32).astype(np.float64)
    t = np.sort(rng.random(n)) * 0.1
    p = rng.integers(0, 2, n) * 2.0 - 1
    models = {"linvel": [(30.0, -20.0), (-55.0, 12.5)], "rotation": [(120.0, 90.0, 4.0), (110.0, 95.0, -6.0)],
              "xyztheta": [(20.0, -10.0, 3.0, 2.0), (-30.0, 15.0, -2.0, 4.0)]}[kind]
    warp = _warp(kind, centre)
    ev = [torch.from_numpy(a).cuda() for a in (x, y, t, p)]
    for prm0 in models:
        prm = torch.tensor(prm0, dtype=torch.float64, device="cuda", requires_grad=True)
        f = motion_timestamp_objective_torch(*ev, prm, warp, blur_sigma=sigma, img_size=(h, w))
        fz = -zhu_timestamp_objective().evaluate_function(prm0, x, y, t, p, warp, (h, w), sigma)
        assert f.shape == (1,) and f.dtype == torch.float64
        assert abs(f.item() - fz) <= 4 * 2.0 ** -15 * abs(fz), (kind, prm0, f.item(), fz)
        f.sum().backward()
        assert torch.isfinite(prm.grad).all() and (prm.grad != 0).any()


@pytest.mark.parametrize("sigma", [0.0, 2.0])
def test_linvel_against_the_flow_timestamp_loss(sigma):
    """linvel v is the expanded uniform flow -v: the same f and gradient (no event reaches x' = 0 or y' = 0, where the
    keep rules differ).  Both warps compute x + (-v) d and x - d v, equal in f32; the flow path samples its uniform
    field bilinearly, which may round u by an ulp"""
    from event_utils_b200.contrast_max import flow_timestamp_objective_torch, linvel_warp, motion_timestamp_objective_torch
    x, y, t, d, p, off = batch_stream(11, [20000, 15000, 9000])
    v0 = np.array([[30.0, -20.0], [-55.0, 12.5], [300.0, 200.0]])
    ev = [torch.from_numpy(a).cuda() for a in (x, y, t, p)]
    ends = torch.from_numpy(off[1:]).cuda()
    v = torch.tensor(v0, device="cuda", requires_grad=True)
    f = motion_timestamp_objective_torch(*ev, v, linvel_warp(), blur_sigma=sigma, img_size=(H, W), batch_end_indices=ends)
    f.sum().backward()
    u = torch.tensor(-v0, device="cuda", requires_grad=True)
    ff = flow_timestamp_objective_torch(*ev, u.view(3, 2, 1, 1).expand(3, 2, H, W), blur_sigma=sigma, batch_end_indices=ends)
    ff.sum().backward()
    torch.testing.assert_close(f, ff, rtol=1e-5, atol=0)
    assert_close_to_max(v.grad.cpu().numpy(), -u.grad.cpu().numpy(), 1e-4, "linvel vs flow")


def _exact_window(seed, n):
    """a window whose images are exactly summable under the models of EXACT0: quarter-pixel positions, p = +-1, the first
    stamp 0 (d = -32: it leaves the canvas) and the others 32 - k/64 up to a last stamp 32, so that tau = t / 32 and
    d = t - 32 are exact and every warped position is a quarter pixel"""
    rng = np.random.default_rng(seed)
    x = (rng.integers(4 * 8, 4 * (W - 8), n) / 4.0).astype(np.float32)
    y = (rng.integers(4 * 8, 4 * (H - 8), n) / 4.0).astype(np.float32)
    p = (rng.integers(0, 2, n) * 2 - 1).astype(np.float32)
    t = np.concatenate(([0.0], np.sort(32.0 - rng.integers(0, 7, n - 2) / 64.0), [32.0])).astype(np.float32)
    return x, y, t, p


EXACT0 = {"linvel": (32.0, -16.0), "rotation": (40.0, 30.25, 0.0), "xyztheta": (32.0, -16.0, 0.0, 0.0)}


def test_nan_isolation_and_batch_independence():
    """a NaN coordinate in window 1 and NaN parameters in window 2: the images of window 0 (exactly summable, so its
    sums do not depend on the order of the reductions) are bit for bit those of the clean batch, its f and gradient
    agree to the order of their f64 sums, window 1 only loses that event, window 2 is the loss of no event, and
    nothing is NaN"""
    sizes = [20000, 15000, 18000]
    x, y, t, d, p, off = batch_stream(29, sizes)
    x[:sizes[0]], y[:sizes[0]], t[:sizes[0]], p[:sizes[0]] = _exact_window(30, sizes[0])
    d[:sizes[0]] = t[:sizes[0]] - 32.0
    xb = x.copy()
    xb[off[1] + 5] = np.nan
    for kind in ("linvel", "rotation", "xyztheta"):
        params = [EXACT0[kind]] + PARAMS[kind][1:3]
        bad = [list(q) for q in params]
        bad[2] = [float("nan")] * len(bad[2])
        _, Ta, Ca = run_forward(kind, x, y, d, R.tau_f32(t, off), p, off, params, 2.0)
        _, Tb, Cb = run_forward(kind, xb, y, d, R.tau_f32(t, off), p, off, bad, 2.0)
        assert np.array_equal(Ta[0], Tb[0]) and np.array_equal(Ca[0], Cb[0]), kind
        f0, prm0 = torch_loss(kind, x, y, t, p, off, params, 2.0)
        f0.sum().backward()
        f1, prm1 = torch_loss(kind, xb, y, t, p, off, bad, 2.0)
        f1.sum().backward()
        fa, fb = f0.detach().cpu().numpy(), f1.detach().cpu().numpy()
        ga, gb = prm0.grad.cpu().numpy(), prm1.grad.cpu().numpy()
        assert np.isfinite(fb).all() and np.isfinite(gb).all()
        assert abs(fb[0] - fa[0]) <= 1e-12 * abs(fa[0]), kind
        np.testing.assert_allclose(gb[0], ga[0], rtol=1e-12, atol=1e-12 * np.abs(ga[0]).max())
        assert abs(fb[1] - fa[1]) <= 1e-3 * abs(fa[1])
        assert fb[2] == 0 and (gb[2] == 0).all()
        # each window alone gives its batched value
        for b in range(3):
            sl = slice(off[b], off[b + 1])
            fs, _ = torch_loss(kind, x[sl], y[sl], t[sl], p[sl], np.array([0, sizes[b]], np.int64), params[b:b + 1], 2.0)
            assert abs(fs.item() - fa[b]) <= 1e-6 * abs(fa[b])


def test_inputs_host_dtypes_expanded_and_large_canvas():
    from event_utils_b200.contrast_max import motion_timestamp_objective_torch, pure_rotation_warp
    sizes = [20000, 15000]
    x, y, t, d, p, off = batch_stream(31, sizes)
    t64 = t.astype(np.float64) + 1000.0
    warp = pure_rotation_warp()
    base = torch.tensor([40.0, 30.0, 4.0], dtype=torch.float64)
    ref = None
    for dtype in (torch.float64, torch.float32):
        for expanded in (False, True):
            prm = base.to(dtype).cuda().requires_grad_(True)
            arg = prm.expand(2, 3) if expanded else torch.stack([prm, prm])
            f = motion_timestamp_objective_torch(x, y, t64, p, arg, warp, img_size=(H, W), batch_end_indices=list(off[1:]))
            assert f.shape == (2,) and f.dtype == dtype and f.device == prm.device
            f.sum().backward()
            assert prm.grad.dtype == dtype and prm.grad.shape == (3,)
            got = (f.detach().double().cpu().numpy(), prm.grad.double().cpu().numpy())
            if ref is None:
                ref = got
            else:
                np.testing.assert_allclose(got[0], ref[0], rtol=1e-6)
                np.testing.assert_allclose(got[1], ref[1], rtol=1e-4, atol=1e-4 * np.abs(ref[1]).max())
    # host parameters and events: the result and the gradient come back on the host
    prm = base.clone().requires_grad_(True)
    f = motion_timestamp_objective_torch(*(torch.from_numpy(a) for a in (x, y, t64, p)), prm.expand(2, 3), warp,
                                         img_size=(H, W), batch_end_indices=list(off[1:]))
    f.sum().backward()
    assert f.device.type == "cpu" and prm.grad.device.type == "cpu"
    np.testing.assert_allclose(f.detach().numpy(), ref[0], rtol=1e-6)
    # one window as a (K,) vector with t0 = None (its last stamp); t0 as a number
    f1 = motion_timestamp_objective_torch(x[:sizes[0]], y[:sizes[0]], t64[:sizes[0]], p[:sizes[0]], base.cuda(), warp,
                                          img_size=(H, W))
    assert f1.shape == (1,) and abs(f1.item() - ref[0][0]) <= 1e-6 * abs(ref[0][0])
    f2 = motion_timestamp_objective_torch(x[:sizes[0]], y[:sizes[0]], t64[:sizes[0]], p[:sizes[0]], base.cuda(), warp,
                                          t0=float(t64[sizes[0] - 1]), img_size=(H, W))
    assert abs(f2.item() - f1.item()) <= 1e-6 * abs(f1.item())     # f32 image sums in any order
    # 480x640
    h, w = 480, 640
    centre = (320.0, 240.0)
    x, y, t, d, p, off = batch_stream(23, [200000, 0, 1, 150000], h, w)
    params = [(60.0, -40.0, 2.0, 1.0), (0.0, 0.0, 0.0, 0.0), (0.0, 0.0, 0.0, 0.0), (-20.0, 30.0, -1.0, 2.0)]
    fl, prm = torch_loss("xyztheta", x, y, t, p, off, params, 2.0, img_size=(h, w), centre=centre)
    g = torch.tensor([1.0, 2.0, 3.0, -1.0], dtype=torch.float64, device="cuda")
    (fl * g).sum().backward()
    p64 = torch.tensor(params, dtype=torch.float64, requires_grad=True)
    fr, _, _ = R.reference("xyztheta", x, y, d, R.tau_f32(t, off), p, off, p64, 2.0, (h, w), centre)
    (fr * g.cpu()).sum().backward()
    fc, got, ref = fl.detach().cpu().numpy(), prm.grad.cpu().numpy(), p64.grad.numpy()
    for b in (0, 3):
        assert abs(fc[b] - fr[b].item()) <= 1e-5 * abs(fr[b].item()), (b, fc[b], fr[b].item())
        assert_close_to_max(got[b], ref[b], 1e-4, "sample %d" % b)
    assert fc[1] == 0 and fc[2] == 0 and (got[1] == 0).all() and (got[2] == 0).all()


def test_no_host_round_trips_and_constant_launch_count():
    from event_utils_b200 import _lib
    from event_utils_b200.contrast_max import motion_timestamp_objective_torch, xyztheta_warp
    L = _lib.lib()
    counts = []
    for sizes in ([40000], [2500] * 16):
        x, y, t, d, p, off = batch_stream(2, sizes)
        params = np.tile(np.array([[20.0, -10.0, 3.0, 2.0]]), (len(sizes), 1))
        torch_loss("xyztheta", x, y, t, p, off, params, 2.0)      # warm-up: scratch buffers, modules
        prm = torch.tensor(params, device="cuda", requires_grad=True)
        ev = [torch.from_numpy(a).cuda() for a in (x, y, t, p)]
        ends = torch.from_numpy(off[1:]).cuda()
        warp = xyztheta_warp(center=CENTRE)
        torch.cuda.synchronize()
        L.evk_prof_enable(1)
        torch.cuda.set_sync_debug_mode("error")
        try:
            f = motion_timestamp_objective_torch(*ev, prm, warp, blur_sigma=2.0, timestamp_reverse=True, img_size=(H, W),
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


def _windows(kind, truths, duration, rng):
    """one window per true motion: a scene of points seen during `duration`, moving with that motion"""
    xs, ys, ts, ps, ends = [], [], [], [], []
    for tr in truths:
        centre = (tr[0], tr[1]) if kind == "rotation" else (120.0, 90.0)
        ang, rad = rng.uniform(0, 2 * np.pi, 300), 60.0 * np.sqrt(rng.uniform(0.05, 1, 300))
        x0, y0 = np.repeat(centre[0] + rad * np.cos(ang), 200), np.repeat(centre[1] + rad * np.sin(ang), 200)
        p = np.repeat(rng.integers(0, 2, 300) * 2.0 - 1.0, 200)
        order = rng.permutation(x0.size)
        x0, y0, p = x0[order], y0[order], p[order]
        t = np.sort(rng.uniform(0, duration, x0.size))
        dt = t - t[-1]
        if kind == "rotation":
            a = tr[2] * dt
            u, v = x0 - tr[0], y0 - tr[1]
            x, y = tr[0] + np.cos(a) * u - np.sin(a) * v, tr[1] + np.sin(a) * u + np.cos(a) * v
        else:
            hx, hy, hz, th = tr
            bx, by = (x0 - 120.0) + dt * hx, (y0 - 90.0) + dt * hy
            m00, m01, m10, m11 = 1 - dt * hz, dt * th, -dt * th, 1 - dt * hz
            det = m00 * m11 - m01 * m10
            x, y = 120.0 + (m11 * bx - m01 * by) / det, 90.0 + (m00 * by - m10 * bx) / det
        xs.append(x), ys.append(y), ts.append(t + len(ends)), ps.append(p)
        ends.append(sum(len(a) for a in xs))
    return [np.concatenate(a) for a in (xs, ys, ts, ps)], ends


@pytest.mark.parametrize("kind", ["rotation", "xyztheta"])
def test_one_optimiser_recovers_every_window(kind):
    """8 windows with distinct motions; Adam on the summed loss from a start near the truth finds each window's own"""
    from event_utils_b200.contrast_max import motion_timestamp_objective_torch
    rng = np.random.default_rng({"rotation": 42, "xyztheta": 43}[kind])
    if kind == "rotation":
        truths = np.column_stack((rng.uniform(110, 130, 8), rng.uniform(80, 100, 8), rng.uniform(3, 8, 8) * rng.choice([-1, 1], 8)))
        scale, duration = np.array([0.5, 0.5, 0.05]), 0.05
        start = np.column_stack((truths[:, :2] + rng.uniform(-2, 2, (8, 2)), truths[:, 2] * rng.uniform(0.85, 1.15, 8)))
    else:
        truths = np.column_stack((rng.uniform(15, 30, 8) * rng.choice([-1, 1], 8), rng.uniform(15, 30, 8) * rng.choice([-1, 1], 8),
                                  rng.uniform(2, 4, 8), rng.uniform(2, 4, 8) * rng.choice([-1, 1], 8)))
        scale, duration = np.array([1.0, 1.0, 0.1, 0.1]), 0.2
        start = truths * (1 + rng.uniform(-0.15, 0.15, truths.shape))
    (x, y, t, p), ends = _windows(kind, truths, duration, rng)
    ev = [torch.from_numpy(a).float().cuda() for a in (x, y, p)]
    tt = torch.from_numpy(t).cuda()
    base = torch.tensor(start, device="cuda")
    s = torch.tensor(scale, device="cuda")
    z = torch.zeros_like(base, requires_grad=True)
    opt = torch.optim.Adam([z], lr=0.3)
    sched = torch.optim.lr_scheduler.CosineAnnealingLR(opt, T_max=300, eta_min=0.003)
    warp = _warp(kind, (120.0, 90.0))
    for _ in range(300):
        opt.zero_grad()
        f = motion_timestamp_objective_torch(ev[0], ev[1], tt, ev[2], base + s * z, warp, blur_sigma=1.0, batch_end_indices=ends)
        f.sum().backward()
        opt.step()
        sched.step()
    got = (base + s * z).detach().cpu().numpy()
    if kind == "rotation":
        assert np.all(np.abs(got[:, 2] - truths[:, 2]) <= 0.03 * np.abs(truths[:, 2])), (got, truths)
        assert np.all(np.hypot(got[:, 0] - truths[:, 0], got[:, 1] - truths[:, 1]) <= 2.0), (got, truths)
    else:
        assert np.all(np.abs(got - truths) <= 0.05 * np.abs(truths)), (got, truths)
