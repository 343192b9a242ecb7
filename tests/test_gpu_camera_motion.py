"""The camera-motion model (camera_motion_warp, EVK_WARP_CAMERA_MOTION) through the depth entries of the contrast and
timestamp losses and their candidates passes, against the f64 references of tests/camera_motion_reference.py: f, the
images, the parameter gradient and the C-level focal-length gradient, the identity with camera_rotation_warp at v = 0
and rho = 0, events that are not kept, chunked windows, host syncs and launch counts, and the fits' recovery of the
angular and linear velocity of a camera moving through a scene with depth, from an embedded camera_rotation_warp fit."""
import ctypes
import functools

import numpy as np
import pytest
import torch

import camera_motion_reference as R
import camera_rotation_reference as CR
import candidate_checks as C
from conftest import assert_close_to_max

pytestmark = pytest.mark.gpu

H, W = 60, 80
INTR = (70.3, 64.9, 43.7, 27.2)     # fx != fy, the principal point away from the canvas' centre (40, 30)
CENTRE = INTR[2:]
# (wx, wy, wz, vx, vy, vz): phi reaches 0.56 rad and rho d |v| 0.25 at d = -0.1
PARAMS = [(2.0, -3.0, 4.0, 1.0, -0.8, 1.5), (-5.0, 1.5, -2.0, -1.5, 0.5, -1.0), (3.5, 4.0, 1.0, 0.4, 2.0, 0.6)]
# the tolerances of tests/test_gpu_camera_rotation.py: the f32 warp and the f64 one differ by a few ulps, no tap moves
F_REL, IMG_REL, GRAD_REL = 1e-4, 1e-4, 1e-3


def _warp(intr=INTR):
    from event_utils_b200.contrast_max.warps import camera_motion_warp
    return camera_motion_warp(intr)


def _rows(params, intr=INTR):
    """(..., 6) motions -> (..., 8) rows (wx, wy, wz, vx, vy, vz, fx, fy) of the C entries"""
    p = np.asarray(params, np.float64)
    return np.concatenate((p, np.broadcast_to(np.array(intr[:2]), p.shape[:-1] + (2,))), axis=-1)


def safe_stream(seed, sizes, models, intr=INTR):
    """Windows of random events in the sensor (d = t - t0 in [-0.1, 0] on a 2^-12 grid, rho in [1/8, 1]), keeping only
    the events whose f64 warp under every model of their window lies at least 1e-3 px from every integer: f32 rounding
    cannot move their taps or keep decisions.  models[b]: the (M,6) motions of window b."""
    rng = np.random.default_rng(seed)
    xs, ys, ds, ps, rs, ends = [], [], [], [], [], []
    for b, n in enumerate(sizes):
        x = (rng.random(n) * (W - 1)).astype(np.float32)
        y = (rng.random(n) * (H - 1)).astype(np.float32)
        d = (-np.sort(rng.integers(0, 410, n))[::-1] / 4096.0).astype(np.float32)
        r = rng.uniform(0.125, 1.0, n).astype(np.float32)
        ok = np.ones(n, bool)
        for m in np.atleast_2d(models[b]) if n else []:
            xw, yw = R.warp(x, y, d, r, m[:3], m[3:], intr)
            for c in (xw, yw):
                with np.errstate(invalid="ignore"):
                    ok &= np.isfinite(c) & (np.abs(c - np.round(c)) >= 1e-3)
        xs.append(x[ok]), ys.append(y[ok]), ds.append(d[ok]), rs.append(r[ok])
        ps.append((rng.integers(0, 2, int(ok.sum())) * 2 - 1).astype(np.float32))
        ends.append(sum(a.size for a in xs))
    off = np.array([0] + ends, np.int64)
    return [np.concatenate(a) for a in (xs, ys, ds, ps, rs)] + [off]


def _cuda(*arrays):
    return [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in arrays]


def _ends(off):
    return torch.from_numpy(off[1:]).cuda()


def entry(stem, events, off, rows, scalars, outs, warp=None, centre=CENTRE):
    """a forward C entry: events as device tensors, outs the shapes of its f64 f and f32 images"""
    from event_utils_b200 import _lib
    L = _lib.lib()
    B = len(off) - 1
    prm = torch.tensor(np.asarray(rows, np.float64), device="cuda")
    res = [torch.empty(s, dtype=torch.float64 if i == 0 else torch.float32, device="cuda") for i, s in enumerate(outs)]
    ws = torch.empty(getattr(L, stem + "_workspace_bytes")(B, H, W), dtype=torch.uint8, device="cuda")
    O = torch.from_numpy(off).cuda()
    lead = [a.data_ptr() for a in events] + [O.data_ptr(), B, events[0].shape[0],
                                             _lib.WARP_CAMERA_MOTION if warp is None else warp, prm.data_ptr(),
                                             prm.shape[-1], centre[0], centre[1], H, W]
    _lib.check(getattr(L, stem + "_f32")(*lead, *scalars, *[r.data_ptr() for r in res], ws.data_ptr(), ws.numel(), None))
    torch.cuda.synchronize()
    return [r.cpu() for r in res], (lead, res, ws, (events, prm, O))


def contrast_forward(x, y, d, p, rho, off, rows, sigma=1.0, name="variance"):
    B = len(off) - 1
    return entry("evk_cmax_motion_depth_objective", _cuda(x, y, d, p, rho), off, rows,
                 (sigma, {"variance": 0, "soe": 2}[name], 0.0), [(B,), (B, H + 1, W + 1)])


def ts_forward(x, y, d, tau, p, rho, off, rows, sigma=1.0):
    B = len(off) - 1
    return entry("evk_motion_timestamp_depth_objective", _cuda(x, y, d, tau, p, rho), off, rows, (sigma,),
                 [(B,), (B, 2, H + 1, W + 1), (B, 2, H + 1, W + 1)])


def c_gradient(stem, call, scalars, gf):
    """grad_params (B,8) of the gradient entry `stem`_grad_f32 after the forward `call` of entry(), at grad_f = gf"""
    from event_utils_b200 import _lib
    L = _lib.lib()
    lead, res, ws, _ = call
    g = torch.from_numpy(np.asarray(gf, np.float32)).cuda()
    out = torch.empty((len(gf), 8), dtype=torch.float64, device="cuda")
    _lib.check(getattr(L, stem + "_grad_f32")(*lead, *scalars, *[r.data_ptr() for r in res[1:]], g.data_ptr(),
                                               out.data_ptr(), ws.data_ptr(), ws.numel(), None))
    torch.cuda.synchronize()
    return out.cpu().numpy()


def loss(fn, x, y, d, p, rho, off, params, **kw):
    """(f with autograd, params leaf) of a torch loss, d reaching the kernel unchanged (t0 = 0)"""
    prm = torch.tensor(np.asarray(params, np.float64), device="cuda", requires_grad=True)
    f = fn(*_cuda(x, y, d, p), prm, _warp(), t0=0.0, blur_sigma=1.0, img_size=(H, W), batch_end_indices=_ends(off),
           inv_depth=torch.from_numpy(rho).cuda(), **kw)
    return f, prm


def _batch_params(batch):
    return PARAMS[:1] if batch == 1 else [PARAMS[0], PARAMS[1], PARAMS[1], PARAMS[2]]


SIZES = {1: [20000], 3: [15000, 0, 12000, 9000]}


@pytest.mark.parametrize("name", ["variance", "soe"])
@pytest.mark.parametrize("batch", [1, 3])
def test_contrast_loss_against_the_reference(name, batch):
    from event_utils_b200.contrast_max import motion_contrast_candidates_torch, motion_contrast_objective_torch
    params = _batch_params(batch)
    x, y, d, p, rho, off = safe_stream(7 + batch, SIZES[batch], params)
    rows = _rows(params)
    scalars = (1.0, {"variance": 0, "soe": 2}[name], 0.0)
    (f, iwe), call = contrast_forward(x, y, d, p, rho, off, rows, 1.0, name)
    p64 = torch.tensor(rows, dtype=torch.float64, requires_grad=True)
    fr, iwer = R.contrast(x, y, d, p, rho, off, p64, 1.0, name, CENTRE, img_size=(H, W))
    for b in range(len(params)):
        assert_close_to_max(iwe[b].numpy(), iwer[b].detach().numpy(), IMG_REL, "iwe %d" % b)
        assert abs(f[b].item() - fr[b].item()) <= F_REL * max(abs(fr[b].item()), 1e-30), (b, f[b], fr[b])
    g = np.random.default_rng(5).standard_normal(len(params))
    (fr * torch.from_numpy(g)).sum().backward()
    # the C entry's eight columns: w, v and the focal lengths
    gc = c_gradient("evk_cmax_motion_depth_objective", call, scalars, g)
    assert_close_to_max(gc[:, :3], p64.grad.numpy()[:, :3], GRAD_REL, "C grad w %s" % name)
    assert_close_to_max(gc[:, 3:6], p64.grad.numpy()[:, 3:6], GRAD_REL, "C grad v %s" % name)
    assert_close_to_max(gc[:, 6:], p64.grad.numpy()[:, 6:], GRAD_REL, "C grad f %s" % name)
    # the torch loss: K = 6, its gradient the first six columns
    fg, prm = loss(motion_contrast_objective_torch, x, y, d, p, rho, off, params, objective=name)
    np.testing.assert_allclose(fg.detach().cpu().numpy(), f.numpy(), rtol=1e-6, atol=0)
    (fg * torch.from_numpy(g).cuda()).sum().backward()
    assert prm.grad.shape == (len(params), 6)
    assert_close_to_max(prm.grad.cpu().numpy(), p64.grad.numpy()[:, :6], GRAD_REL, "grad %s" % name)
    cand = torch.tensor(params, dtype=torch.float64, device="cuda").unsqueeze(1).repeat(1, 3, 1)
    fc = motion_contrast_candidates_torch(*_cuda(x, y, d, p), cand, _warp(), t0=0.0, objective=name, blur_sigma=1.0,
                                          img_size=(H, W), batch_end_indices=_ends(off), inv_depth=torch.from_numpy(rho).cuda())
    # f32 image sums in another order (atomics): equal to f32 rounding
    np.testing.assert_allclose(fc.cpu().numpy(), f.unsqueeze(1).repeat(1, 3).numpy(), rtol=1e-6, atol=0)


@pytest.mark.parametrize("batch", [1, 3])
def test_timestamp_loss_against_the_reference(batch):
    from event_utils_b200.contrast_max import motion_timestamp_candidates_torch, motion_timestamp_objective_torch
    params = _batch_params(batch)
    x, y, d, p, rho, off = safe_stream(17 + batch, SIZES[batch], params)
    tau = R.tau_f32(d, off)
    rows = _rows(params)
    (f, T, C), call = ts_forward(x, y, d, tau, p, rho, off, rows)
    p64 = torch.tensor(rows, dtype=torch.float64, requires_grad=True)
    fr, Tr, Cr = R.timestamp(x, y, d, tau, p, rho, off, p64, 1.0, CENTRE, img_size=(H, W))
    for b in range(len(params)):
        assert_close_to_max(T[b].numpy(), Tr[b].detach().numpy(), IMG_REL, "T %d" % b)
        assert_close_to_max(C[b].numpy(), Cr[b].detach().numpy(), IMG_REL, "C %d" % b)
        assert abs(f[b].item() - fr[b].item()) <= F_REL * max(abs(fr[b].item()), 1e-30), (b, f[b], fr[b])
    g = np.random.default_rng(6).standard_normal(len(params))
    (fr * torch.from_numpy(g)).sum().backward()
    gc = c_gradient("evk_motion_timestamp_depth_objective", call, (1.0,), g)
    assert_close_to_max(gc[:, :3], p64.grad.numpy()[:, :3], GRAD_REL, "C ts grad w")
    assert_close_to_max(gc[:, 3:6], p64.grad.numpy()[:, 3:6], GRAD_REL, "C ts grad v")
    assert_close_to_max(gc[:, 6:], p64.grad.numpy()[:, 6:], GRAD_REL, "C ts grad f")
    fg, prm = loss(motion_timestamp_objective_torch, x, y, d, p, rho, off, params)
    np.testing.assert_allclose(fg.detach().cpu().numpy(), f.numpy(), rtol=1e-6, atol=0)
    (fg * torch.from_numpy(g).cuda()).sum().backward()
    assert_close_to_max(prm.grad.cpu().numpy(), p64.grad.numpy()[:, :6], GRAD_REL, "ts grad")
    cand = torch.tensor(params, dtype=torch.float64, device="cuda").unsqueeze(1).repeat(1, 2, 1)
    fc = motion_timestamp_candidates_torch(*_cuda(x, y, d, p), cand, _warp(), t0=0.0, blur_sigma=1.0, img_size=(H, W),
                                           batch_end_indices=_ends(off), inv_depth=torch.from_numpy(rho).cuda())
    np.testing.assert_allclose(fc.cpu().numpy(), f.unsqueeze(1).repeat(1, 2).numpy(), rtol=1e-6, atol=0)


def sparse_stream(om, seed, per_window=4000):
    """events whose footprints under the camera rotation om[b] of their window share no pixel: every canvas cell then
    sums at most one tap, in any order, so the f32 images of two runs can be compared bit for bit.  Each event lies at
    least 1e-3 px from the integers, so the f32 and f64 warps floor alike."""
    rng = np.random.default_rng(seed)
    xs, ys, ds, ps, ends = [], [], [], [], []
    for m in om:
        x = (rng.random(per_window) * (W - 1)).astype(np.float32)
        y = (rng.random(per_window) * (H - 1)).astype(np.float32)
        d = (-np.sort(rng.random(per_window))[::-1] * 0.1).astype(np.float32)
        xw, yw = CR.warp(x, y, d, m, INTR)
        with np.errstate(invalid="ignore"):
            ok = (np.isfinite(xw) & (np.abs(xw - np.round(xw)) >= 1e-3) & (np.abs(yw - np.round(yw)) >= 1e-3) &
                  (xw > 1) & (xw < W - 1) & (yw > 1) & (yw < H - 1))
        taken = np.zeros((H + 2, W + 2), bool)
        pick = []
        for e in np.flatnonzero(ok):
            cx, cy = int(xw[e]) + 1, int(yw[e]) + 1
            if not taken[cy - 1:cy + 2, cx - 1:cx + 2].any():
                taken[cy, cx] = True
                pick.append(e)
        xs.append(x[pick]), ys.append(y[pick]), ds.append(d[pick])
        ps.append((rng.integers(0, 2, len(pick)) * 2 - 1).astype(np.float32))
        ends.append(sum(a.size for a in xs))
    return [np.concatenate(a) for a in (xs, ys, ds, ps)] + [np.array([0] + ends, np.int64)]


def test_equal_to_the_camera_rotation_at_zero_translation():
    """at v = 0 and at rho = 0 the translation adds an exact zero: the images of both losses are camera_rotation_warp's
    bit for bit and f equal to the f64 atomics of the image tail, and the w gradient is its to f32 rounding"""
    from event_utils_b200 import _lib
    from event_utils_b200.contrast_max import motion_contrast_objective_torch, motion_timestamp_objective_torch, warps
    om = np.array([[2.0, -3.0, 4.0], [-5.0, 1.5, -2.0], [3.5, 4.0, 1.0]])
    x, y, d, p, off = sparse_stream(om, 31)
    assert off[1] > 300 and np.diff(off).min() > 300, off
    n = x.size
    tau = R.tau_f32(d, off)
    rot_rows = np.concatenate((om, np.tile(INTR[:2], (3, 1))), 1)
    rot = entry("evk_cmax_motion_objective", _cuda(x, y, d, p), off, rot_rows, (1.0, 0, 0.0), [(3,), (3, H + 1, W + 1)],
                warp=_lib.WARP_CAMERA_ROTATION)[0]
    rot_ts = entry("evk_motion_timestamp_objective", _cuda(x, y, d, tau, p), off, rot_rows, (1.0,),
                   [(3,), (3, 2, H + 1, W + 1), (3, 2, H + 1, W + 1)], warp=_lib.WARP_CAMERA_ROTATION)[0]
    v = np.array([[1.0, -0.8, 1.5], [-1.5, 0.5, -1.0], [0.4, 2.0, 0.6]])
    rho = np.random.default_rng(32).uniform(0.125, 1.0, n).astype(np.float32)
    for motion, r in ((np.concatenate((om, 0 * v), 1), rho), (np.concatenate((om, v), 1), np.zeros(n, np.float32))):
        for got, want in ((contrast_forward(x, y, d, p, r, off, _rows(motion))[0], rot),
                          (ts_forward(x, y, d, tau, p, r, off, _rows(motion))[0], rot_ts)):
            np.testing.assert_allclose(got[0].numpy(), want[0].numpy(), rtol=1e-12, atol=0)
            assert all(torch.equal(a, b) for a, b in zip(got[1:], want[1:]))
        vgrad = []
        for fn in (motion_contrast_objective_torch, motion_timestamp_objective_torch):
            f, prm = loss(fn, x, y, d, p, r, off, motion)
            prm0 = torch.tensor(om, device="cuda", requires_grad=True)
            f0 = fn(*_cuda(x, y, d, p), prm0, warps.camera_rotation_warp(INTR), t0=0.0, blur_sigma=1.0, img_size=(H, W),
                    batch_end_indices=_ends(off))
            np.testing.assert_allclose(f.detach().cpu().numpy(), f0.detach().cpu().numpy(), rtol=1e-12, atol=0)
            f.sum().backward()
            f0.sum().backward()
            assert_close_to_max(prm.grad[:, :3].cpu().numpy(), prm0.grad.cpu().numpy(), 1e-5, "w grad %s" % fn.__name__)
            vgrad.append(prm.grad[:, 3:].abs().max().item())
        # the v columns: rho d fx iz (1, 0, -X) is zero with rho = 0, and not with v = 0
        assert (max(vgrad) == 0.0) == (not r.any()), vgrad


def test_events_that_are_not_kept_add_nothing():
    """events behind the camera and events with a negative, NaN or infinite inverse depth add nothing to f, the images
    or the gradient of either loss: the stream of the kept events alone gives the same values, up to summation order,
    and those meet the reference"""
    from event_utils_b200.contrast_max import motion_contrast_objective_torch, motion_timestamp_objective_torch
    intr = (30.0, 30.0, 40.0, 30.0)       # a wide field of view: fast rotations take events behind the camera
    m = np.array([[11.0, -13.0, 6.0, 2.0, -1.0, 3.0]])
    rng = np.random.default_rng(51)
    n = 20000
    x = (rng.random(n) * (W - 1)).astype(np.float32)
    y = (rng.random(n) * (H - 1)).astype(np.float32)
    d = (-np.sort(rng.integers(0, 410, n))[::-1] / 4096.0).astype(np.float32)
    p = (rng.integers(0, 2, n) * 2 - 1).astype(np.float32)
    rho = rng.uniform(0.125, 1.0, n).astype(np.float32)
    bad = rng.random(n)
    rho[bad < 0.03] = -0.5
    rho[(bad >= 0.03) & (bad < 0.06)] = np.nan
    rho[(bad >= 0.06) & (bad < 0.07)] = np.inf
    xw, yw = R.warp(x, y, d, rho, m[0, :3], m[0, 3:], intr)
    out = np.isnan(xw)
    behind = out & (bad >= 0.07)
    assert 0.02 < behind.mean() < 0.5 and 0.09 < out.mean() < 0.6, (behind.mean(), out.mean())
    with np.errstate(invalid="ignore"):
        safe = out | ((np.abs(xw - np.round(xw)) >= 1e-3) & (np.abs(yw - np.round(yw)) >= 1e-3))
    x, y, d, p, rho, out = x[safe], y[safe], d[safe], p[safe], rho[safe], out[safe]
    keep = ~out
    off, offk = np.array([0, x.size]), np.array([0, int(keep.sum())])
    rows = _rows(m, intr)
    tau = R.tau_f32(d, off)
    c_all = entry("evk_cmax_motion_depth_objective", _cuda(x, y, d, p, rho), off, rows, (1.0, 0, 0.0), [(1,), (1, H + 1, W + 1)],
                  centre=intr[2:])[0]
    c_kept = entry("evk_cmax_motion_depth_objective", _cuda(x[keep], y[keep], d[keep], p[keep], rho[keep]), offk, rows,
                   (1.0, 0, 0.0), [(1,), (1, H + 1, W + 1)], centre=intr[2:])[0]
    np.testing.assert_allclose(c_all[1].numpy(), c_kept[1].numpy(), rtol=0, atol=1e-5 * c_all[1].abs().max().item())
    np.testing.assert_allclose(c_all[0].numpy(), c_kept[0].numpy(), rtol=1e-6)
    shapes = [(1,), (1, 2, H + 1, W + 1), (1, 2, H + 1, W + 1)]
    t_all = entry("evk_motion_timestamp_depth_objective", _cuda(x, y, d, tau, p, rho), off, rows, (1.0,), shapes,
                  centre=intr[2:])[0]
    t_kept = entry("evk_motion_timestamp_depth_objective", _cuda(x[keep], y[keep], d[keep], tau[keep], p[keep], rho[keep]),
                   offk, rows, (1.0,), shapes, centre=intr[2:])[0]
    np.testing.assert_allclose(t_all[0].numpy(), t_kept[0].numpy(), rtol=1e-6)
    np.testing.assert_allclose(t_all[1].numpy(), t_kept[1].numpy(), rtol=0, atol=1e-6)
    for fn in (motion_contrast_objective_torch, motion_timestamp_objective_torch):
        grads = []
        for sel, o in ((np.ones(x.size, bool), off), (keep, offk)):
            prm = torch.tensor(m, device="cuda", requires_grad=True)
            f = fn(*_cuda(x[sel], y[sel], d[sel], p[sel]), prm, _warp(intr), t0=0.0, img_size=(H, W),
                   batch_end_indices=_ends(o), inv_depth=torch.from_numpy(rho[sel]).cuda())
            f.sum().backward()
            grads.append(prm.grad.cpu().numpy())
        assert np.isfinite(grads[0]).all()
        assert_close_to_max(grads[0], grads[1], 1e-6, "not-kept grad %s" % fn.__name__)
    p64 = torch.tensor(rows, dtype=torch.float64, requires_grad=True)
    fr, _ = R.contrast(x, y, d, p, rho, off, p64, 1.0, "variance", intr[2:], img_size=(H, W))
    np.testing.assert_allclose(c_all[0].numpy(), fr.detach().numpy(), rtol=F_REL)


def test_chunked_windows_change_nothing(monkeypatch):
    """the fits' forward and gradient and both candidates passes run in chunks of windows under a small workspace
    budget, with the inverse depth read through each chunk's offsets: every value equals the one-chunk run"""
    from event_utils_b200.contrast_max import motion_fit as MF
    from event_utils_b200.contrast_max import motion_objective as MO
    from event_utils_b200.contrast_max import motion_timestamp_fit as MTF
    from event_utils_b200.contrast_max import motion_timestamp_objective as MT
    from event_utils_b200.contrast_max._batched import _batch_events, _depth_events, _model, _normalised_stamps, _ts_model
    B = 9
    params = np.array([PARAMS[b % 3] for b in range(B)])
    x, y, d, p, rho, off = safe_stream(41, [3000, 0, 2500, 4000, 1000, 3500, 2000, 0, 3000], params)
    w = _warp()
    dev = torch.device("cuda")
    X, Y, D, P, O, t, sample = _batch_events(*_cuda(x, y, d, p), 0.0, _ends(off), B, dev, "w", stamps=True)
    U = _normalised_stamps(t, sample, O, False)
    rho_d = _depth_events(torch.from_numpy(rho), dev)
    prm = torch.tensor(params, device="cuda")
    cand = prm.unsqueeze(1).repeat(1, 5, 1) + torch.linspace(0, 0.5, 5, device="cuda", dtype=torch.float64).view(1, 5, 1)
    opts, ts_opts = _model(7, w, "variance", 1.0, None, H, W), _ts_model(7, w, 1.0, H, W)

    def run():
        return (MF._objective_and_gradient(X, Y, D, P, O, opts, rho_d)(prm),
                MTF._objective_and_gradient(X, Y, D, U, P, O, ts_opts, rho_d)(prm),
                MO._candidates(X, Y, D, P, O, cand, opts, rho_d), MT._ts_candidates(X, Y, D, U, P, O, cand, ts_opts, rho_d))
    whole = run()
    per_window = (H + 1) * (W + 1) * 4
    monkeypatch.setattr(MF, "FIT_WORKSPACE_BYTES", 40 * per_window)
    monkeypatch.setattr(MTF, "FIT_WORKSPACE_BYTES", 60 * per_window)
    monkeypatch.setattr(MO, "CANDIDATES_WORKSPACE_BYTES", 40 * per_window)
    monkeypatch.setattr(MT, "TIMESTAMP_CANDIDATES_WORKSPACE_BYTES", 100 * per_window)
    chunked = run()
    # the same arithmetic per window; the atomics of the image sums may meet in another order from call to call
    for a, b in zip(whole[:2], chunked[:2]):
        np.testing.assert_allclose(a[0].cpu().numpy(), b[0].cpu().numpy(), rtol=1e-6, atol=0)
        assert_close_to_max(a[1].cpu().numpy(), b[1].cpu().numpy(), 1e-5, "chunked gradient")
    for a, b in zip(whole[2:], chunked[2:]):
        np.testing.assert_allclose(a.cpu().numpy(), b.cpu().numpy(), rtol=1e-6, atol=0)
    # and f of the forward is the reference's
    fr, _ = R.contrast(x, y, d, p, rho, off, torch.tensor(_rows(params)), 1.0, "variance", CENTRE, img_size=(H, W))
    np.testing.assert_allclose(whole[0][0].cpu().numpy(), fr.numpy(), rtol=F_REL)


def test_no_host_round_trips_and_constant_launch_count():
    from event_utils_b200 import _lib
    from event_utils_b200.contrast_max import motion_contrast_objective_torch, motion_timestamp_objective_torch
    L = _lib.lib()
    counts = []
    for sizes in ([40000], [2500] * 16):
        params = np.tile(np.array([PARAMS[0]]), (len(sizes), 1))
        x, y, d, p, rho, off = safe_stream(2, sizes, [params[:1]] * len(sizes))
        ev = _cuda(x, y, d, p)
        r = torch.from_numpy(rho).cuda()
        ends = _ends(off)
        for _ in range(2):          # the first round warms up (scratch, library load)
            prm = torch.tensor(params, device="cuda", requires_grad=True)
            torch.cuda.synchronize()
            L.evk_prof_enable(1)
            torch.cuda.set_sync_debug_mode("error")
            try:
                f = motion_contrast_objective_torch(*ev, prm, _warp(), objective="soe", img_size=(H, W), batch_end_indices=ends,
                                                    inv_depth=r)
                g = motion_timestamp_objective_torch(*ev, prm, _warp(), img_size=(H, W), batch_end_indices=ends, inv_depth=r)
                (f.sum() + g.sum()).backward()
            finally:
                torch.cuda.set_sync_debug_mode(0)
            ms, timed, launches = ctypes.c_double(), ctypes.c_longlong(), ctypes.c_longlong()
            _lib.check(L.evk_prof_collect(ctypes.byref(ms), ctypes.byref(timed), ctypes.byref(launches)))
            L.evk_prof_enable(0)
        assert torch.isfinite(prm.grad).all() and prm.grad.shape == (len(sizes), 6)
        counts.append(launches.value)
    assert counts[0] == counts[1] and counts[0] > 0, counts


# ---- the candidates passes with distinct candidates (tests/candidate_checks.py) -------------------------------------
SPREAD = (0.3, 0.3, 0.3, 0.1, 0.1, 0.1)
# GONE turns every bearing by phi = |w| |d| in [1.25, 2.5] rad about the y axis, past the 59 degree field of view or
# behind the camera, at |d| >= 0.05.  PARTIAL moves the camera forward: Pz = 1 - 12 rho |d| takes the events of large
# rho |d| behind the camera and zooms the others out of the canvas, so what it keeps depends on every event's rho.
GONE_M, PARTIAL_M = (0.0, 25.0, 0.0, 0.0, 0.0, 0.0), (0.0, 0.0, 0.0, 0.0, 0.0, 12.0)
CAND_SIZES = {1: [12000], 5: [9000, 0, 6000, 12000, 1], 6: [5000, 0, 4000, 7000, 1, 3000]}


def cand_warp(intr=INTR):
    """the reference warp of candidate_stream, NaN for the events that are not kept"""
    return lambda x, y, d, rho, prm: R.warp(x, y, d, rho, prm[:3], prm[3:6], intr)


@functools.lru_cache(maxsize=None)
def candidate_case(batch):
    """(B,70,6) distinct candidates with GONE and PARTIAL, and the windows CAND_SIZES[batch] safe under every one; the
    events' rho spread over [1/8, 1] in every window"""
    base = np.array([PARAMS[b % 3] for b in range(batch)])
    cand = C.distinct_sets(base, 70, np.random.default_rng(700 + batch), SPREAD, GONE_M, PARTIAL_M)
    return cand, C.candidate_stream(batch, CAND_SIZES[batch], cand, cand_warp(), H, W)


# three candidates of the sparse stream, on the 180 x 240 camera CAMERA: their v differ, and rho varies per event
SPARSE = [(1.0, -0.8, 0.6, 1.5, 0.0, 0.5), (0.8, -1.0, 0.7, -1.0, 1.0, 1.5), (1.2, -0.6, 0.5, 2.0, -0.5, -1.0)]


@functools.lru_cache(maxsize=None)
def sparse_case():
    """window 0: events whose footprints lie 3 px apart under each of SPARSE; window 1: 30000 dense events.  x, y, d, p,
    rho, offsets."""
    rng = np.random.default_rng(37)
    x, y, d, p, rho = C.draw(rng, 40000, 180, 240, (-0.1, 0.0))
    pick = C.sparse_pick([cand_warp(CAMERA)(x, y, d, rho, q) for q in SPARSE], 180, 240)
    dense = C.draw(rng, 30000, 180, 240, (-0.1, 0.0))
    off = np.array([0, pick.size, pick.size + 30000], np.int64)
    return [np.concatenate((a[pick], b)) for a, b in zip((x, y, d, p, rho), dense)] + [off]


def contrast_candidates(ev, rho, off, cand, sigma, name, img_size=(H, W), intr=INTR):
    from event_utils_b200.contrast_max import motion_contrast_candidates_torch
    return motion_contrast_candidates_torch(*ev, torch.tensor(cand, device="cuda"), _warp(intr), t0=0.0, objective=name,
                                            blur_sigma=sigma, obj_param=0.3, img_size=img_size, batch_end_indices=_ends(off),
                                            inv_depth=rho).cpu().numpy()


def contrast_per_candidate(ev, rho, off, cand, sigma, name, img_size=(H, W), intr=INTR):
    """motion_contrast_objective_torch once per candidate index j: (B,J)"""
    from event_utils_b200.contrast_max import motion_contrast_objective_torch
    return np.stack([motion_contrast_objective_torch(*ev, torch.tensor(cand[:, j], device="cuda"), _warp(intr), t0=0.0,
                                                     objective=name, blur_sigma=sigma, obj_param=0.3, img_size=img_size,
                                                     batch_end_indices=_ends(off), inv_depth=rho).cpu().numpy()
                     for j in range(cand.shape[1])], 1)


def ts_candidates(ev, rho, off, cand, sigma, reverse):
    from event_utils_b200.contrast_max import motion_timestamp_candidates_torch
    return motion_timestamp_candidates_torch(*ev, torch.tensor(cand, device="cuda"), _warp(), t0=0.0, blur_sigma=sigma,
                                             timestamp_reverse=reverse, img_size=(H, W), batch_end_indices=_ends(off),
                                             inv_depth=rho).cpu().numpy()


def ts_per_candidate(ev, rho, off, cand, sigma, reverse):
    from event_utils_b200.contrast_max import motion_timestamp_objective_torch
    return np.stack([motion_timestamp_objective_torch(*ev, torch.tensor(cand[:, j], device="cuda"), _warp(), t0=0.0,
                                                      blur_sigma=sigma, timestamp_reverse=reverse, img_size=(H, W),
                                                      batch_end_indices=_ends(off), inv_depth=rho).cpu().numpy()
                     for j in range(cand.shape[1])], 1)


@pytest.mark.parametrize("name", ["variance", "sos", "soe", "sosa"])
@pytest.mark.parametrize("sigma", [0.0, 1.0, 3.0])
@pytest.mark.parametrize("batch", [1, 5])
def test_contrast_candidates_distinct_against_the_forward_and_the_reference(name, sigma, batch):
    master, (x, y, d, p, rho, off) = candidate_case(batch)
    ev, r = _cuda(x, y, d, p), torch.from_numpy(rho).cuda()

    def reference(cand):
        return np.stack([R.contrast(x, y, d, p, rho, off, torch.from_numpy(_rows(cand[:, j])), sigma, name, CENTRE, 0.3, (H, W))[0]
                         .numpy() for j in range(cand.shape[1])], 1), F_REL
    C.check_sets(master, lambda c: contrast_candidates(ev, r, off, c, sigma, name),
                 lambda c: contrast_per_candidate(ev, r, off, c, sigma, name), reference, C.no_event_value(name, H, W),
                 [1] if batch == 5 else [], "%s %g" % (name, sigma))


@pytest.mark.parametrize("sigma", [0.0, 1.0, 2.0, 3.0])
@pytest.mark.parametrize("reverse", [False, True])
@pytest.mark.parametrize("batch", [1, 5])
def test_timestamp_candidates_distinct_against_the_forward_and_the_reference(sigma, reverse, batch):
    """the stamps are d (t0 = 0 lies 0.05 or more after every window's last stamp); a lone event has tau = 0"""
    master, (x, y, d, p, rho, off) = candidate_case(batch)
    ev, r = _cuda(x, y, d, p), torch.from_numpy(rho).cuda()
    tau = R.tau_f32(d, off, reverse)

    def reference(cand):
        return np.stack([R.timestamp(x, y, d, tau, p, rho, off, torch.from_numpy(_rows(cand[:, j])), sigma, CENTRE, (H, W))[0]
                         .numpy() for j in range(cand.shape[1])], 1), F_REL
    C.check_sets(master, lambda c: ts_candidates(ev, r, off, c, sigma, reverse),
                 lambda c: ts_per_candidate(ev, r, off, c, sigma, reverse), reference, C.no_event_value(None, H, W),
                 [1, 4] if batch == 5 else [], "%g %s" % (sigma, reverse))


def test_candidates_of_sparse_footprints_bit_for_bit():
    """at most one tap per pixel under each candidate: the images equal the forward's bit for bit, so f agrees to the
    f64 rounding of the statistics' reduction order (a dense second window to f32 summation order)"""
    x, y, d, p, rho, off = sparse_case()
    assert off[1] > 500, off
    ev, r = _cuda(x, y, d, p), torch.from_numpy(rho).cuda()
    cand = np.array([SPARSE] * 2, np.float64)
    for name, sigma in (("variance", 0.0), ("soe", 1.0)):
        kw = dict(img_size=(180, 240), intr=CAMERA)
        f = contrast_candidates(ev, r, off, cand, sigma, name, **kw)
        ref = contrast_per_candidate(ev, r, off, cand, sigma, name, **kw)
        np.testing.assert_allclose(f[0], ref[0], rtol=1e-12, atol=0, err_msg=name)
        np.testing.assert_allclose(f[1], ref[1], rtol=1e-6, atol=0, err_msg=name)


def test_window_chunks_with_distinct_candidates(monkeypatch):
    """six skewed windows x 70 distinct candidates in chunks of two windows (three J passes each), rho read through
    each chunk's offsets: every entry equals the one-chunk run and the per-candidate forward"""
    from event_utils_b200 import _lib
    from event_utils_b200.contrast_max import motion_objective as MO
    from event_utils_b200.contrast_max import motion_timestamp_objective as MT
    L = _lib.lib()
    cand, (x, y, d, p, rho, off) = candidate_case(6)
    ev, r = _cuda(x, y, d, p), torch.from_numpy(rho).cuda()
    budgets = [(MO, "CANDIDATES_WORKSPACE_BYTES", 2 * L.evk_cmax_motion_depth_candidates_workspace_bytes(1, 32, H, W) + 1),
               (MT, "TIMESTAMP_CANDIDATES_WORKSPACE_BYTES",
                2 * L.evk_motion_timestamp_depth_candidates_workspace_bytes(1, 32, H, W) + 1)]
    C.check_chunks(monkeypatch, budgets, lambda c: contrast_candidates(ev, r, off, c, 1.0, "variance"),
                   lambda c: contrast_per_candidate(ev, r, off, c, 1.0, "variance"), cand, "contrast")
    C.check_chunks(monkeypatch, budgets, lambda c: ts_candidates(ev, r, off, c, 1.0, False),
                   lambda c: ts_per_candidate(ev, r, off, c, 1.0, False), cand, "timestamp")


# ---- recovery on a scene with depth -----------------------------------------------------------------------------
CAMERA = (199.1, 198.7, 132.1, 110.8)        # fx, fy, cx, cy of a 180 x 240 camera
# (wx, wy, wz) rad/s and (vx, vy, vz) m/s per window; the points lie 1-8 m away
TRUTHS = np.array([(1.0, -0.8, 0.6, 1.5, 0.0, 0.5), (-2.0, 1.0, 0.5, -1.0, 1.0, 1.5), (0.5, 2.5, -1.0, 2.0, -0.5, -1.0),
                   (3.0, 1.5, 0.8, 0.5, 1.5, 2.0), (-1.5, -2.5, 1.5, -2.0, -1.0, 0.5), (1.5, -3.0, -2.0, 1.0, 2.0, -1.5)])
DURATION = 0.05


def motion_windows(seed):
    rng = np.random.default_rng(seed)
    parts = [R.motion_scene(m[:3], m[3:], CAMERA, rng, t_end=DURATION, duration=DURATION) for m in TRUTHS]
    ends = np.cumsum([a[0].size for a in parts])
    return [np.concatenate(a) for a in zip(*parts)], ends


def recover(loss_name, seed=81):
    """(rotation-only w, camera-motion (w, v)) fitted on the scene's windows: the rotation from a grid search, then the
    camera motion from the rotation's w embedded with v = 0"""
    from event_utils_b200.contrast_max import motion_contrast_fit_torch, motion_timestamp_fit_torch
    from event_utils_b200.contrast_max.warps import camera_rotation_warp
    (x, y, t, p, rho), ends = motion_windows(seed)
    ev = [torch.from_numpy(x).float().cuda(), torch.from_numpy(y).float().cuda(), torch.from_numpy(t).cuda(),
          torch.from_numpy(p).float().cuda()]
    kw = dict(batch_end_indices=torch.tensor(ends, device="cuda"), t0=DURATION, blur_sigma=[4.0, 2.0, 1.0])
    fit_fn = motion_contrast_fit_torch if loss_name == "contrast" else motion_timestamp_fit_torch
    rot = fit_fn(*ev, camera_rotation_warp(CAMERA), param_ranges=[[-10.0, 10.0]] * 3, num_samples_per_param=5,
                 grid_levels=3, **kw).params
    x0 = torch.cat((rot, torch.zeros_like(rot)), 1)
    extra = {}
    if loss_name == "timestamp":     # this loss's degenerate minima lie outside a box (motion_timestamp_fit_torch)
        extra["bounds"] = torch.stack((x0 - 5.0, x0 + 5.0), -1)
    fit = fit_fn(*ev, _warp(CAMERA), x0=x0, inv_depth=torch.from_numpy(rho).float().cuda(), **kw, **extra)
    assert fit.params.shape == (len(TRUTHS), 6)
    return rot.cpu().numpy(), fit.params.cpu().numpy()


# largest |w_fit - w_true| (rad/s) and |v_fit - v_true| (m/s) over the windows; observed on an H100 (80 GB HBM3, 700 W):
# contrast 0.053 rad/s and 0.151 m/s, timestamp 0.0041 rad/s and 0.0104 m/s over three runs, against 0.31-0.49 rad/s for
# the w of the rotation-only fits (DESIGN section 6)
RECOVERY = {"contrast": (0.12, 0.3), "timestamp": (0.02, 0.05)}


@pytest.mark.parametrize("loss_name", ["contrast", "timestamp"])
def test_fits_recover_the_angular_and_linear_velocity(loss_name):
    rot, got = recover(loss_name)
    err_rot = np.linalg.norm(rot - TRUTHS[:, :3], axis=1)
    err_w = np.linalg.norm(got[:, :3] - TRUTHS[:, :3], axis=1)
    err_v = np.linalg.norm(got[:, 3:] - TRUTHS[:, 3:], axis=1)
    print("%s: rotation-only |w - w_true| %s, camera motion |w - w_true| %s rad/s, |v - v_true| %s m/s (|v_true| %s)"
          % (loss_name, np.round(err_rot, 4), np.round(err_w, 4), np.round(err_v, 4),
             np.round(np.linalg.norm(TRUTHS[:, 3:], axis=1), 3)))
    # the scene needs the translation: the rotation-only fit's w is measurably worse in every window
    assert (err_w < err_rot).all() and err_rot.min() > 0.1, (err_w, err_rot)
    # the recovered v is closer to the truth than zero
    assert (err_v < 0.5 * np.linalg.norm(TRUTHS[:, 3:], axis=1)).all(), err_v
    tol_w, tol_v = RECOVERY[loss_name]
    assert err_w.max() <= tol_w and err_v.max() <= tol_v, (err_w, err_v)
