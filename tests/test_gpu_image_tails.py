"""The contrast objectives' image-space tails (csrc/evk_cmax.cu) against the f64 reference of tests/tail_reference.py, at
every radius of the sweep (0, 1, 4, 8 | 9, 12, 32, 64: both sides of the fused tail's limit and the largest radius) and
on canvases below, at and past one 8x32 tile, a radius far beyond the canvas included.  Every path reaches the tail:

  evk_gaussian_blur_f32                 the blur alone
  evk_iwe_objective_f32                 the separate tail (launch_tail), six objectives, with and without channel mixing
  evk_cmax_linvel_objective_f32 / _f64  the fused variance tail (r <= 8) and the separate one (r >= 9)
  *_batch_f64                           the candidate batches, against their single-candidate calls
  evk_cmax_peer_tail_f32                the fused tail over peer images
  the three batched torch losses        the batched blur, statistics and adjoint blur

Each value is compared with the reference applied to the image the kernel returns, so the event passes (checked by
their own exact-sum tests) drop out, and within a bound carried from the blur's per-cell rounding bound -- not a flat
tolerance."""
import ctypes

import numpy as np
import pytest
import torch

import tail_reference as T

pytestmark = pytest.mark.gpu

SIGMAS = [0.0, 0.1, 0.125, 1.0, 1.875, 2.1249, 2.125, 3.0, 7.9, 15.875, 16.0]
LEGACY = [(1, 1), (1, 300), (300, 1), (6, 30), (7, 31), (8, 32), (180, 240), (255, 255)]
BATCHED = [(2, 2), (3, 70), (8, 31), (45, 60), (130, 7)]
OBJ = {"variance": 0, "sos": 1, "soe": 2, "moa": 3, "isoa": 4, "sosa": 5}
PARAM = {"variance": 0.0, "sos": 0.0, "soe": 0.0, "moa": 0.0, "isoa": 0.1, "sosa": 0.3}


def _L():
    from event_utils_b200 import _lib
    return _lib, _lib.lib()


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _ws(nbytes):
    return torch.empty(max(int(nbytes), 256), dtype=torch.uint8, device="cuda")


def _image(rng, shape, name="variance"):
    scale = 0.3 if name in ("soe", "sosa") else 1.0        # keeps exp(G) and exp(-p G) of order one
    return (rng.standard_normal(shape) * scale).astype(np.float32)


def _assert_within(res, ref, layout, what, exact_zero=()):
    bad = T.violations(res, ref, layout, exact_zero)
    assert not bad, "%s: (index, key, got, want, bound) %r" % (what, bad)


# ---- 1. the blur --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", LEGACY)
def test_gaussian_blur(shape):
    _lib, L = _L()
    rng = np.random.default_rng(sum(shape))
    I = rng.standard_normal(shape).astype(np.float32)
    a = _dev(I)
    out, tmp = torch.empty_like(a), torch.empty_like(a)
    for sigma in SIGMAS:
        out.fill_(float("nan"))
        _lib.check(L.evk_gaussian_blur_f32(a.data_ptr(), shape[0], shape[1], sigma, out.data_ptr(), tmp.data_ptr(), None))
        G = out.cpu().numpy()
        if sigma == 0:
            assert (G == I).all()
        err = np.abs(G.astype(np.float64) - T.blur64(I, sigma))
        bound = T.blur_bound(I, sigma)
        assert (err <= bound).all(), "sigma %g: %d cells outside, worst err %r" % (sigma, (err > bound).sum(), err.max())


# ---- 2. the separate tail on precomputed images ---------------------------------------------------------------------------
@pytest.mark.parametrize("shape", LEGACY)
@pytest.mark.parametrize("mix", [True, False])
def test_iwe_objective(shape, mix):
    _lib, L = _L()
    Hc, Wc = shape[0] + 1, shape[1] + 1
    rng = np.random.default_rng(Hc * 1000 + Wc)
    ws = _ws(L.evk_cmax_workspace_bytes(Hc - 1, Wc - 1))
    res = torch.zeros(12, dtype=torch.float64, device="cuda")
    D = np.stack([rng.standard_normal((Hc, Wc)), 2.0 * rng.standard_normal((Hc, Wc)) + 0.5]).astype(np.float32)
    d = _dev(D)
    flags = _lib.CMAX_WANT_GRAD | (0 if mix else _lib.CMAX_NO_CHANNEL_MIX)
    for name in OBJ:
        I = _image(rng, (Hc, Wc), name)
        a = _dev(I)
        for sigma in SIGMAS:
            res.fill_(float("nan"))
            _lib.check(L.evk_iwe_objective_f32(a.data_ptr(), d.data_ptr(), Hc, Wc, sigma, flags, OBJ[name], PARAM[name],
                                               res.data_ptr(), ws.data_ptr(), ws.numel(), None))
            r = res.cpu().numpy()
            ref = T.tail(I, D, sigma, name, PARAM[name], mix)
            _assert_within(r, ref, T.legacy_layout(name, True), "%s sigma %g" % (name, sigma), exact_zero=(4,))


# ---- 3. the fused (r <= 8) and separate (r >= 9) variance tails of the linvel entries ------------------------------------
def _events(rng, n, Hs, Ws):
    x = rng.random(n) * Ws
    y = rng.random(n) * Hs
    t = np.sort(rng.random(n)) * 0.01
    p = (rng.integers(0, 2, n) * 2 - 1).astype(np.float64)
    return x, y, t, p


@pytest.mark.parametrize("shape", LEGACY)
def test_linvel_variance_tails(shape):
    _lib, L = _L()
    Hs, Ws = shape
    Hc, Wc = Hs + 1, Ws + 1
    rng = np.random.default_rng(Hs * 7 + Ws)
    x, y, t, p = _events(rng, 3000, Hs, Ws)
    t_ref = float(t[-1])
    ev64 = [_dev(a) for a in (x, y, t, p)]
    ev32 = [_dev(a.astype(np.float32)) for a in (x, y, t - t_ref, p)]
    ws = _ws(L.evk_cmax_workspace_bytes(Hs, Ws))
    res = torch.zeros(12, dtype=torch.float64, device="cuda")
    iwe = torch.empty((Hc, Wc), device="cuda")
    diwe = torch.empty((2, Hc, Wc), device="cuda")
    # the on-chip event pass where the canvas fits in shared memory; the 256x256 canvas takes the L2 pass
    flags = _lib.CMAX_WANT_GRAD | _lib.VARIANT_SMEM_TILE
    v = (30.0, -20.0)
    for sigma in SIGMAS:
        for prec in ("f64", "f32"):
            res.fill_(float("nan"))
            if prec == "f64":
                rc = L.evk_cmax_linvel_objective_f64(*(e.data_ptr() for e in ev64), len(x), 1.0, v[0], v[1], t_ref, Hs, Ws, Hs, Ws,
                                                     sigma, flags, 0, 0.0, res.data_ptr(), iwe.data_ptr(), diwe.data_ptr(),
                                                     ws.data_ptr(), ws.numel(), None)
            else:
                rc = L.evk_cmax_linvel_objective_f32(*(e.data_ptr() for e in ev32), len(x), 1.0, v[0], v[1], Hs, Ws, Hs, Ws,
                                                     sigma, flags, 0, 0.0, res.data_ptr(), iwe.data_ptr(), diwe.data_ptr(),
                                                     ws.data_ptr(), ws.numel(), None)
            _lib.check(rc)
            r = res.cpu().numpy()
            I, D = iwe.cpu().numpy(), diwe.cpu().numpy()
            assert np.abs(I).sum() > 0
            ref = T.tail(I, D, sigma, "variance", 0.0, True)
            _assert_within(r, ref, T.legacy_layout("variance", True), "%s sigma %g (radius %d)" % (prec, sigma, T.radius(sigma)))


# ---- 4. candidate batches against their single-candidate calls -----------------------------------------------------------
def _sparse_events(rng, Hs, Ws, gap=4):
    """events on a grid `gap` pixels apart that move less than half a pixel: the 2x2 footprints never overlap, so every
    IWE pixel receives at most one term and the images of the batched and the single pass are the same numbers"""
    gy, gx = np.mgrid[0:max(Hs - 1, 1):gap, 0:max(Ws - 1, 1):gap]
    n = gy.size
    x = gx.ravel() + 0.25 + 0.5 * rng.random(n)
    y = gy.ravel() + 0.25 + 0.5 * rng.random(n)
    t = np.sort(rng.random(n)) * 0.005
    p = (rng.integers(0, 2, n) * 2 - 1).astype(np.float64)
    return x, y, t, p


def _rel_equal(a, b, tol=1e-12):
    scale = max(np.abs(b).max(), 1e-300)
    return np.abs(a - b).max() <= tol * scale


@pytest.mark.parametrize("shape", [(7, 31), (180, 240)])
@pytest.mark.parametrize("n_params", [1, 7, 32])
def test_linvel_candidate_batch(shape, n_params):
    _lib, L = _L()
    Hs, Ws = shape
    rng = np.random.default_rng(n_params)
    x, y, t, p = _sparse_events(rng, Hs, Ws)
    t_ref = float(t[-1])
    ev = [_dev(a) for a in (x, y, t, p)]
    ws = _ws(L.evk_cmax_workspace_bytes(Hs, Ws))
    params = np.stack([30.0 - 2.0 * np.arange(n_params), -20.0 + 1.5 * np.arange(n_params)], 1).astype(np.float64)
    results = torch.zeros((n_params, 12), dtype=torch.float64, device="cuda")
    one = torch.zeros(12, dtype=torch.float64, device="cuda")
    iwe = torch.empty((Hs + 1, Ws + 1), device="cuda")
    diwe = torch.empty((2, Hs + 1, Ws + 1), device="cuda")
    # r <= 8: one fused launch for every candidate; r >= 9 and sos: one separate tail per candidate
    for name, sigma in (("variance", 0.0), ("variance", 1.875), ("variance", 2.1249), ("variance", 2.125), ("sos", 1.0)):
        _lib.check(L.evk_cmax_linvel_objective_batch_f64(*(e.data_ptr() for e in ev), len(x), 1.0, params.ctypes.data, n_params,
                                                          t_ref, Hs, Ws, Hs, Ws, sigma, _lib.CMAX_WANT_GRAD, OBJ[name], 0.0,
                                                          results.data_ptr(), ws.data_ptr(), ws.numel(), None))
        batch = results.cpu().numpy()
        for k in range(n_params):
            _lib.check(L.evk_cmax_linvel_objective_f64(*(e.data_ptr() for e in ev), len(x), 1.0, params[k, 0], params[k, 1], t_ref,
                                                       Hs, Ws, Hs, Ws, sigma, _lib.CMAX_WANT_GRAD, OBJ[name], 0.0, one.data_ptr(),
                                                       iwe.data_ptr(), diwe.data_ptr(), ws.data_ptr(), ws.numel(), None))
            single = one.cpu().numpy()
            lay = T.legacy_layout(name, True)
            idx = sorted(lay)
            assert _rel_equal(batch[k][idx], single[idx]), (name, sigma, k, batch[k][idx], single[idx])
            ref = T.tail(iwe.cpu().numpy(), diwe.cpu().numpy(), sigma, name, 0.0, True)
            _assert_within(batch[k], ref, lay, "%s sigma %g candidate %d" % (name, sigma, k))


@pytest.mark.parametrize("n_models", [1, 7, 32])
def test_warp_candidate_batch(n_models):
    _lib, L = _L()
    Hs, Ws = 45, 60
    rng = np.random.default_rng(10 + n_models)
    x, y, t, p = _sparse_events(rng, Hs, Ws)
    t_ref = float(t[-1])
    ev = [_dev(a) for a in (x, y, t, p)]
    ws = _ws(L.evk_cmax_workspace_bytes(Hs, Ws))
    models = np.stack([np.full(n_models, 30.0), np.full(n_models, 22.0), np.linspace(-1.0, 1.0, n_models)], 1)
    models = np.ascontiguousarray(models, np.float64)
    results = torch.zeros((n_models, 16), dtype=torch.float64, device="cuda")
    one = torch.zeros(16, dtype=torch.float64, device="cuda")
    iwe = torch.empty((Hs + 1, Ws + 1), device="cuda")
    for name, sigma in (("variance", 1.875), ("sos", 2.125), ("isoa", 0.125), ("sosa", 7.9), ("moa", 16.0)):
        _lib.check(L.evk_cmax_warp_objective_batch_f64(*(e.data_ptr() for e in ev), len(x), 1.0, _lib.WARP_ROTATION,
                                                        models.ctypes.data, n_models, t_ref, Hs, Ws, Hs, Ws, sigma, 0, OBJ[name],
                                                        PARAM[name], results.data_ptr(), ws.data_ptr(), ws.numel(), None))
        batch = results.cpu().numpy()
        lay = T.model_layout(name)
        idx = sorted(lay)
        for k in range(n_models):
            m = np.ascontiguousarray(models[k])
            _lib.check(L.evk_cmax_warp_objective_f64(*(e.data_ptr() for e in ev), len(x), 1.0, _lib.WARP_ROTATION, m.ctypes.data,
                                                     t_ref, Hs, Ws, Hs, Ws, sigma, 0, OBJ[name], PARAM[name], one.data_ptr(),
                                                     iwe.data_ptr(), ws.data_ptr(), ws.numel(), None))
            single = one.cpu().numpy()
            assert _rel_equal(batch[k][idx], single[idx]), (name, sigma, k, batch[k][idx], single[idx])
            ref = T.tail(iwe.cpu().numpy(), None, sigma, name, PARAM[name])
            _assert_within(batch[k], ref, lay, "%s sigma %g model %d" % (name, sigma, k))


def test_model_gradient_past_the_shared_memory_canvas_is_unsupported():
    """the 256x256 canvas (256 KB of f32) is above the 200 KB the model gradient pass holds in shared memory"""
    _lib, L = _L()
    Hs, Ws = 255, 255
    x, y, t, p = (_dev(a) for a in _events(np.random.default_rng(3), 100, Hs, Ws))
    ws = _ws(L.evk_cmax_workspace_bytes(Hs, Ws))
    res = torch.zeros(16, dtype=torch.float64, device="cuda")
    model = np.array([128.0, 128.0, 0.5])
    rc = L.evk_cmax_warp_objective_f64(x.data_ptr(), y.data_ptr(), t.data_ptr(), p.data_ptr(), 100, 1.0, _lib.WARP_ROTATION,
                                       model.ctypes.data, 0.01, Hs, Ws, Hs, Ws, 1.0, _lib.CMAX_WANT_GRAD, 0, 0.0, res.data_ptr(),
                                       None, ws.data_ptr(), ws.numel(), None)
    assert rc == -5 and b"shared memory" in L.evk_last_error()


# ---- 5. the peer tail -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("world", [1, 3])
def test_peer_tail(world):
    _lib, L = _L()
    oob = torch.zeros(1, dtype=torch.int64, device="cuda")
    res = torch.zeros(12, dtype=torch.float64, device="cuda")
    for Hs, Ws in [(1, 1), (1, 300), (300, 1), (6, 30), (7, 31), (8, 32), (255, 255)]:
        Hc, Wc = Hs + 1, Ws + 1
        rng = np.random.default_rng(Hc + 3 * Wc)
        img = np.concatenate([_image(rng, (1, Hc, Wc)), rng.standard_normal((2, Hc, Wc)).astype(np.float32)])
        d = _dev(img)
        peers = (ctypes.c_void_p * world)(*([d.data_ptr()] * world))
        oobs = (ctypes.c_void_p * world)(*([oob.data_ptr()] * world))
        # the tail sums the ranks' images in rank order in f32
        tot = np.zeros_like(img)
        for _ in range(world):
            tot = (tot + img).astype(np.float32)
        ws = _ws(L.evk_cmax_workspace_bytes(Hs, Ws))
        for sigma in [s for s in SIGMAS if T.radius(s) <= T.FUSED_MAX_R]:
            res.fill_(float("nan"))
            _lib.check(L.evk_cmax_peer_tail_f32(peers, oobs, world, Hc, Wc, sigma, _lib.CMAX_WANT_GRAD, res.data_ptr(),
                                                ws.data_ptr(), ws.numel(), None))
            ref = T.tail(tot[0], tot[1:], sigma, "variance", 0.0, True)
            _assert_within(res.cpu().numpy(), ref, T.legacy_layout("variance", True), "%dx%d sigma %g" % (Hc, Wc, sigma),
                           exact_zero=(4,))
        rc = L.evk_cmax_peer_tail_f32(peers, oobs, world, Hc, Wc, 2.125, _lib.CMAX_WANT_GRAD, res.data_ptr(), ws.data_ptr(),
                                      ws.numel(), None)
        assert rc == -5 and b"radius 9" in L.evk_last_error()


# ---- 6. the batched losses -------------------------------------------------------------------------------------------------
def _sizes(batch, n=300):
    """per-sample event counts with empty samples in between"""
    return [0 if b % 3 == 1 else n for b in range(batch)]


@pytest.mark.parametrize("shape", BATCHED)
@pytest.mark.parametrize("batch", [1, 3, 37])
def test_batched_losses_forward(shape, batch):
    import test_gpu_cmax_flow_objective as FO
    import test_gpu_cmax_motion_objective as MO
    import test_gpu_flow_timestamp_objective as TO
    import flow_timestamp_reference as TR
    H, W = shape
    sizes = _sizes(batch)
    names = ["variance", "sos", "soe", "sosa"] if batch < 37 else ["variance", "sosa"]
    x, y, d, p, off, flows = FO.batch_stream(batch, sizes, H, W, 0.2)
    mx, my, md, mp, moff = MO.batch_stream(batch, sizes, H, W)
    params = [(30.0 - 3.0 * b, -20.0 + 2.0 * b) for b in range(batch)]
    tx, ty, tt, td, tp, toff, tflows = TO.batch_stream(batch, sizes, H, W, 0.2)
    tau = TR.tau_f32(tt, toff)
    for sigma in SIGMAS:
        for name in names:
            f, iwe = FO.run_forward(x, y, d, p, off, flows, sigma, name, PARAM[name])
            fm, iwem = MO.run_forward("linvel", mx, my, md, mp, moff, params, sigma, name, PARAM[name], H, W)
            for b in range(batch):
                for what, got, img in (("flow", f[b], iwe[b]), ("motion", fm[b], iwem[b])):
                    want, bound = T.batched_f(img, sigma, name, PARAM[name])
                    assert abs(got - want) <= bound, (what, name, sigma, b, got, want, bound)
                    if sizes[b] == 0:
                        assert (img == 0).all()
        ft, Ti, Ci = TO.run_forward(tx, ty, td, tau, tp, toff, tflows, sigma)
        for b in range(batch):
            want, bound = T.timestamp_f(Ti[b], sigma)
            assert abs(ft[b] - want) <= bound, ("timestamp", sigma, b, ft[b], want, bound)


GRAD_SIGMAS = [0.1, 1.875, 2.125, 15.875]


@pytest.mark.parametrize("shape", [(8, 31), (3, 70)])
@pytest.mark.parametrize("sigma", GRAD_SIGMAS)
def test_batched_losses_gradient(shape, sigma):
    from exact_bounds import gamma
    import flow_objective_reference as FR
    import motion_objective_reference as MR
    import flow_timestamp_reference as TR
    import test_gpu_cmax_flow_objective as FO
    import test_gpu_cmax_motion_objective as MO
    import test_gpu_flow_timestamp_objective as TO
    H, W = shape
    sizes = [400, 0, 300]
    g = torch.from_numpy(np.random.default_rng(5).standard_normal(len(sizes)))

    def check(got, ref, M, cnt, what):
        bound = gamma(cnt + 32) * M
        err = np.abs(got - ref)
        bad = err > bound
        assert not bad.any(), "%s: %d outside, e.g. err %r bound %r" % (what, bad.sum(), err[bad][:3], bound[bad][:3])

    for name in ("variance", "sosa"):
        x, y, d, p, off, flows = FO.batch_stream(1, sizes, H, W, 0.2)
        f, fl = FO.torch_loss(x, y, d, p, off, flows, sigma, name, PARAM[name])
        (f * g.cuda().to(f.dtype)).sum().backward()
        flow64 = torch.from_numpy(flows).double().requires_grad_(True)
        fr, iwer, mag = FR.reference(x, y, d, p, off, flow64, sigma, name, PARAM[name])
        (fr * g).sum().backward()
        M, cnt = FR.grad_magnitude(x, y, d, p, off, flow64, sigma, name, PARAM[name], g.numpy(), iwer.detach().numpy(), mag.numpy())
        check(fl.grad.cpu().numpy().astype(np.float64), flow64.grad.numpy(), M, cnt, "flow %s" % name)

        mx, my, md, mp, moff = MO.batch_stream(2, sizes, H, W)
        params = [(30.0, -20.0), (0.0, 0.0), (-12.0, 7.5)]
        fm, prm = MO.torch_loss("linvel", mx, my, md, mp, moff, params, sigma, name, PARAM[name], img_size=(H, W))
        (fm * g.cuda()).sum().backward()
        p64 = torch.tensor(params, dtype=torch.float64, requires_grad=True)
        fr, iwer, mag = MR.reference("linvel", mx, my, md, mp, moff, p64, sigma, name, PARAM[name], (H, W), MO.CENTRE)
        (fr * g).sum().backward()
        M, cnt = MR.grad_magnitude("linvel", mx, my, md, mp, moff, p64, sigma, name, PARAM[name], g.numpy(),
                                   iwer.detach().numpy(), mag.numpy(), (H, W), MO.CENTRE)
        check(prm.grad.cpu().numpy(), p64.grad.numpy(), M, cnt, "motion %s" % name)

    tx, ty, tt, td, tp, toff, tflows = TO.batch_stream(3, sizes, H, W, 0.2)
    ft, fl = TO.torch_loss(tx, ty, tt, tp, toff, tflows, sigma)
    (ft * g.cuda().to(ft.dtype)).sum().backward()
    tau = TR.tau_f32(tt, toff)
    flow64 = torch.from_numpy(tflows).double().requires_grad_(True)
    fr, Tr, Cr = TR.reference(tx, ty, td, tau, tp, toff, flow64, sigma)
    (fr * g).sum().backward()
    M, cnt = TR.grad_magnitude(tx, ty, td, tau, tp, toff, flow64, sigma, g.numpy(), Tr.detach().numpy(), Cr.detach().numpy())
    check(fl.grad.cpu().numpy().astype(np.float64), flow64.grad.numpy(), M, cnt, "timestamp")


# ---- 7. a bad sigma through the Python API ------------------------------------------------------------------------------
@pytest.mark.parametrize("sigma", [float("inf"), float("nan"), 1e9])
def test_bad_sigma_raises_through_python(sigma):
    from event_utils_b200 import _lib
    from event_utils_b200.contrast_max import (flow_contrast_objective_torch, flow_timestamp_objective_torch, linvel_warp,
                                               motion_contrast_objective_torch)
    from event_utils_b200.contrast_max.objectives import rms_objective, variance_objective, zhu_timestamp_objective
    rng = np.random.default_rng(1)
    n = 2000
    xs, ys = rng.random(n) * 239, rng.random(n) * 179
    ts, ps = np.sort(rng.random(n)) * 0.1, rng.integers(0, 2, n) * 2.0 - 1
    warp = linvel_warp()
    for obj in (variance_objective(), rms_objective(), zhu_timestamp_objective()):
        with pytest.raises(_lib.EvkError, match="blur sigma"):
            obj.evaluate_function((30.0, -20.0), xs, ys, ts, ps, warp, (180, 240), sigma)
    ev = [torch.from_numpy(a).float().cuda() for a in (xs, ys, ts, ps)]
    flow = torch.zeros((2, 180, 240), device="cuda", requires_grad=True)
    prm = torch.tensor([30.0, -20.0], device="cuda", requires_grad=True)
    with pytest.raises(_lib.EvkError, match="blur sigma"):
        flow_contrast_objective_torch(*ev, flow, blur_sigma=sigma)
    with pytest.raises(_lib.EvkError, match="blur sigma"):
        motion_contrast_objective_torch(*ev, prm, warp, blur_sigma=sigma)
    with pytest.raises(_lib.EvkError, match="blur sigma"):
        flow_timestamp_objective_torch(*ev, flow, blur_sigma=sigma)
