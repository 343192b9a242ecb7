"""Motion segmentation (evk_cmax_motion_segment_*, contrast_max/motion_segmentation.py) against the single-model loss it
restates per model, against the f64 reference of tests/motion_segmentation_reference.py, and the EM fit: recovery of
several known motions per window with their events' labels, and no host synchronisation."""
import ctypes

import numpy as np
import pytest
import torch

import motion_segmentation_reference as S
from conftest import assert_close_to_max
from edge_cases import exact_streams
from test_gpu_cmax_motion_objective import CENTRE, H, PARAMS, W, _warp, batch_stream, run_forward, torch_loss
from test_gpu_motion_fit import _scene, recovered

pytestmark = pytest.mark.gpu

SIZES = {1: [6000], 5: [5000, 0, 3000, 6000, 1]}      # an empty and a one-event window


def models(kind, B, M):
    """(B,M,K): window b's model m is PARAMS[kind][(b + m) % 5] scaled by 1 + 0.1 m (the fourth sends most events off)"""
    return np.array([[np.array(PARAMS[kind][(b + m) % 5]) * (1 + 0.1 * m) for m in range(M)] for b in range(B)], np.float64)


def memberships(n, M, seed):
    """random weights in [0, 1) with exact zeros in every column"""
    w = np.random.default_rng(seed).random((n, M)).astype(np.float32)
    w[::17] = 0.0
    return w


def seg_loss(kind, x, y, d, p, w, off, params, sigma, name, param=0.3, img_size=(H, W), centre=CENTRE, grad_w=True):
    from event_utils_b200.contrast_max import motion_segmentation_objective_torch
    prm = torch.tensor(params, device="cuda", requires_grad=True)
    wt = torch.tensor(w, device="cuda", requires_grad=grad_w)
    ev = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (x, y, d, p)]
    f = motion_segmentation_objective_torch(*ev, wt, prm, _warp(kind, centre), t0=0.0, objective=name, blur_sigma=sigma,
                                            obj_param=param, img_size=img_size, batch_end_indices=torch.from_numpy(off[1:]).cuda())
    return f, prm, wt


def seg_forward(kind, x, y, d, p, w, off, params, sigma, name, param=0.3, h=H, w_=W, centre=CENTRE):
    """the C entry directly: (f (B,M), iwe (B,M,h+1,w+1)) as numpy"""
    from event_utils_b200 import _lib
    L = _lib.lib()
    B, M, K = params.shape
    X, Y, D, P, O = (torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (x, y, d, p, off))
    Wt = torch.from_numpy(np.ascontiguousarray(w)).cuda()
    prm = torch.tensor(params, device="cuda")
    f = torch.empty((B, M), dtype=torch.float64, device="cuda")
    iwe = torch.empty((B, M, h + 1, w_ + 1), device="cuda")
    ws = torch.empty(L.evk_cmax_motion_segment_workspace_bytes(B, M, h, w_), dtype=torch.uint8, device="cuda")
    _lib.check(L.evk_cmax_motion_segment_f32(X.data_ptr(), Y.data_ptr(), D.data_ptr(), P.data_ptr(), Wt.data_ptr(), M, O.data_ptr(),
                                             B, x.shape[0], {"linvel": 3, "rotation": 1, "xyztheta": 2}[kind], prm.data_ptr(), K,
                                             centre[0], centre[1], h, w_, sigma, {"variance": 0, "sos": 1, "soe": 2, "sosa": 5}[name],
                                             param, f.data_ptr(), iwe.data_ptr(), ws.data_ptr(), ws.numel(), None))
    torch.cuda.synchronize()
    return f.cpu().numpy(), iwe.cpu().numpy()


def test_one_model_of_weight_one_is_the_motion_objective():
    """M = 1, weights 1: f, the IWE and the parameter gradient are motion_contrast_objective_torch's -- bit for bit on
    exactly summable streams (tests/edge_cases.py) where the sums are exact, else to the existing tolerances"""
    c = exact_streams(3, "cmax", 300001)
    h, w = c["Hs"], c["Ws"]
    x, y, t, p = (np.asarray(c[k], np.float32) for k in ("x", "y", "t", "p"))
    off = np.array([0, 100000, 100000, 300001], np.int64)
    centre = (20.0, 12.0)
    ones = np.ones((x.shape[0], 1), np.float32)
    sets = {"linvel": [(c["vx"], c["vy"])] * 3, "xyztheta": [(c["vx"], c["vy"], 0.0, 0.0)] * 3,
            "rotation": [(20.0, 12.0, 0.0), (21.0, 13.5, 0.0), (22.25, 10.0, 0.0)]}
    for kind, prm in sets.items():
        params = np.array(prm, np.float64)
        for name, sigma in (("variance", 0.0), ("variance", 1.0), ("sos", 0.0), ("sos", 1.0)):
            f, iwe = seg_forward(kind, x, y, t, p, ones, off, params[:, None], sigma, name, 3.0, h, w, centre)
            f0, iwe0 = run_forward(kind, x, y, t, p, off, prm, sigma, name, 3.0, h, w, centre)
            assert np.array_equal(iwe[:, 0], iwe0), (kind, name, sigma)
            if name == "variance" and sigma == 0.0:
                assert np.array_equal(f[:, 0], f0), (kind, f[:, 0], f0)
            else:
                np.testing.assert_allclose(f[:, 0], f0, rtol=1e-12, atol=0)
            # the parameter gradient from the same images: the same per-thread f64 sums, which only the f64 atomics
            # of the CTAs add in another order
            g = torch.tensor([1.0, 2.0, -0.5], dtype=torch.float64, device="cuda")
            f0, prm0 = torch_loss(kind, x, y, t, p, off, prm, sigma, name, 3.0, (h, w), centre)
            (f0 * g).sum().backward()
            f1, prm1, _ = seg_loss(kind, x, y, t, p, ones, off, params[:, None], sigma, name, 3.0, (h, w), centre, grad_w=False)
            (f1[:, 0] * g).sum().backward()
            assert_close_to_max(prm1.grad[:, 0].cpu().numpy(), prm0.grad.cpu().numpy(), 1e-12, "%s %s %g" % (kind, name, sigma))
    # random streams: f32 image sums in another order, so f to 1e-6 and the gradient to the f32 rounding of W
    sizes = [15000, 0, 9000, 20000, 1]
    x, y, d, p, off = batch_stream(3, sizes)
    for kind in ("linvel", "rotation", "xyztheta"):
        for name, sigma in (("variance", 1.0), ("soe", 0.0), ("sosa", 3.0)):
            g = torch.from_numpy(np.random.default_rng(5).standard_normal(len(sizes))).cuda()
            f0, prm0 = torch_loss(kind, x, y, d, p, off, PARAMS[kind], sigma, name, 0.3)
            (f0 * g).sum().backward()
            f1, prm1, _ = seg_loss(kind, x, y, d, p, np.ones((x.shape[0], 1), np.float32), off, np.array(PARAMS[kind])[:, None],
                                   sigma, name, grad_w=False)
            (f1[:, 0] * g).sum().backward()
            np.testing.assert_allclose(f1[:, 0].detach().cpu().numpy(), f0.detach().cpu().numpy(), rtol=1e-6, atol=0)
            assert_close_to_max(prm1.grad[:, 0].cpu().numpy(), prm0.grad.cpu().numpy(), 1e-5, "%s %s" % (kind, name))


@pytest.mark.parametrize("kind", ["linvel", "rotation", "xyztheta"])
@pytest.mark.parametrize("name", ["variance", "sos", "soe", "sosa"])
@pytest.mark.parametrize("sigma", [0.0, 1.0, 3.0])
@pytest.mark.parametrize("batch", [1, 5])
@pytest.mark.parametrize("M", [1, 2, 4, 8])
def test_images_and_f_against_the_single_model_loss_and_the_reference(kind, name, sigma, batch, M):
    sizes = SIZES[batch]
    x, y, d, p, off = batch_stream(7 + batch, sizes)
    w = memberships(x.shape[0], M, seed=M)
    params = models(kind, batch, M)
    f, iwe = seg_forward(kind, x, y, d, p, w, off, params, sigma, name)
    fr, iwer = S.reference(kind, x, y, d, p, torch.from_numpy(w.astype(np.float64)), off, torch.from_numpy(params), sigma, name,
                           0.3, (H, W), CENTRE)
    fr, iwer = fr.detach().numpy(), iwer.detach().numpy()
    for m in range(M):
        fm, iwem = run_forward(kind, x, y, d, (p * w[:, m]).astype(np.float32), off, params[:, m], sigma, name, 0.3)
        for b in range(batch):
            assert_close_to_max(iwe[b, m], iwem[b], 1e-6, "iwe %d %d" % (b, m))
            assert abs(f[b, m] - fm[b]) <= 1e-6 * max(abs(fm[b]), 1e-30), (b, m, f[b, m], fm[b])
            assert_close_to_max(iwe[b, m], iwer[b, m], 1e-5, "iwe %d %d vs reference" % (b, m))
            assert abs(f[b, m] - fr[b, m]) <= 1e-5 * max(abs(fr[b, m]), 1e-30), (b, m, f[b, m], fr[b, m])
    if batch == 5:
        assert (iwe[1] == 0).all()


@pytest.mark.parametrize("kind", ["linvel", "rotation", "xyztheta"])
@pytest.mark.parametrize("name", ["variance", "sos", "soe", "sosa"])
@pytest.mark.parametrize("sigma", [0.0, 1.0, 3.0])
def test_gradients_against_the_reference(kind, name, sigma):
    """parameter and membership gradients event by event, including events of weight 0, of p = 0 and events that are
    not kept (the fourth model sends most events off the canvas)"""
    sizes = [4000, 0, 3000, 5000, 1]
    x, y, d, p, off = batch_stream(3, sizes)
    p = p.copy()
    p[5::23] = 0.0
    M = 3
    w = memberships(x.shape[0], M, seed=11)
    params = models(kind, len(sizes), M)
    f, prm, wt = seg_loss(kind, x, y, d, p, w, off, params, sigma, name)
    g = torch.from_numpy(np.random.default_rng(5).standard_normal((len(sizes), M)))
    (f * g.cuda()).sum().backward()
    p64 = torch.tensor(params, requires_grad=True)
    w64 = torch.tensor(w.astype(np.float64), requires_grad=True)
    fr, _ = S.reference(kind, x, y, d, p, w64, off, p64, sigma, name, 0.3, (H, W), CENTRE)
    (fr * g).sum().backward()
    np.testing.assert_allclose(f.detach().cpu().numpy(), fr.detach().numpy(), rtol=1e-5, atol=0)
    assert_close_to_max(prm.grad.cpu().numpy(), p64.grad.numpy(), 1e-4, "params %s %s %g" % (kind, name, sigma))
    gw, gwr = wt.grad.cpu().numpy(), w64.grad.numpy()
    assert_close_to_max(gw, gwr, 1e-4, "weights %s %s %g" % (kind, name, sigma))
    zero_w = (w == 0) & (p[:, None] != 0)
    assert (gwr[zero_w] != 0).any() and (gw[zero_w] != 0).any()          # a weight of 0 still has a gradient
    assert (gw[p == 0] == 0).all()
    assert (prm.grad[1] == 0).all()


def test_candidates_equal_the_forward_and_splits_change_no_value():
    from event_utils_b200.contrast_max import motion_segmentation as MS
    from event_utils_b200.contrast_max import motion_segmentation_candidates_torch
    from event_utils_b200 import _lib
    sizes = [9000, 0, 7000, 12000, 1, 5000]
    x, y, d, p, off = batch_stream(51, sizes)
    for kind, M in (("rotation", 2), ("linvel", 4), ("xyztheta", 3)):
        B = len(sizes)
        w = memberships(x.shape[0], M, seed=M)
        rng = np.random.default_rng(M)
        base = models(kind, B, M)
        J = 37
        cand = base[:, :, None, :] * (1 + rng.uniform(-0.2, 0.2, (B, M, J, base.shape[2])))
        cand[:, :, 0] = base
        ev = [torch.from_numpy(a).cuda() for a in (x, y, d, p)]
        kw = dict(t0=0.0, objective="variance", blur_sigma=1.0, img_size=(H, W), batch_end_indices=torch.from_numpy(off[1:]).cuda())
        wt = torch.from_numpy(w).cuda()
        one = motion_segmentation_candidates_torch(*ev, torch.tensor(cand, device="cuda"), wt, _warp(kind), **kw).cpu().numpy()
        assert one.shape == (B, M, J) and one.dtype == np.float64
        for j in (0, 5, 36):
            f, _ = seg_forward(kind, x, y, d, p, w, off, np.ascontiguousarray(cand[:, :, j]), 1.0, "variance")
            np.testing.assert_allclose(one[:, :, j], f, rtol=1e-6, atol=0, err_msg="%s j=%d" % (kind, j))
        per = _lib.load().evk_cmax_motion_segment_candidates_workspace_bytes(1, M, 32 // M, H, W)
        saved = MS.SEGMENT_CANDIDATES_WORKSPACE_BYTES
        try:
            MS.SEGMENT_CANDIDATES_WORKSPACE_BYTES = 2 * per + 1       # two windows per chunk
            many = motion_segmentation_candidates_torch(*ev, torch.tensor(cand, device="cuda"), wt, _warp(kind), **kw).cpu().numpy()
        finally:
            MS.SEGMENT_CANDIDATES_WORKSPACE_BYTES = saved
        np.testing.assert_allclose(many, one, rtol=1e-6, atol=0)


def test_assignment_against_the_reference_and_its_rules():
    from event_utils_b200.contrast_max import motion_segmentation_assign_torch
    sizes = [6000, 0, 5000, 7000]
    x, y, d, p, off = batch_stream(61, sizes)
    n = x.shape[0]
    outside = 500                                   # events after the last window
    x, y, d, p = (np.concatenate((a, a[:outside])) for a in (x, y, d, p))
    for kind in ("linvel", "rotation", "xyztheta"):
        for M, sigma in ((2, 1.0), (4, 0.0), (8, 3.0)):
            w = memberships(x.shape[0], M, seed=3)
            params = models(kind, len(sizes), M)
            pa = np.abs(p)
            kw = dict(t0=0.0, blur_sigma=sigma, img_size=(H, W), batch_end_indices=torch.from_numpy(off[1:]).cuda())
            args = [torch.from_numpy(a).cuda() for a in (x, y, d, pa)]
            got = motion_segmentation_assign_torch(*args, torch.tensor(params, device="cuda"), _warp(kind), torch.from_numpy(w).cuda(),
                                                   eps=1e-6, **kw).cpu().numpy()
            _, iwe = seg_forward(kind, x, y, d, pa, w, off, params, sigma, "variance")
            ref = S.assign(kind, x, y, d, off, params, iwe, sigma, 1e-6, (H, W), CENTRE)
            # to 1e-5 of the row sum: the reference's bilinear fractions come from numpy's f32 sin / cos, within an ulp of
            # the kernel's sincosf
            np.testing.assert_allclose(got, ref, rtol=1e-5, atol=1e-5, err_msg="%s M=%d" % (kind, M))
            np.testing.assert_allclose(got.sum(1), 1.0, rtol=1e-5)
            assert (got[n:] == np.float32(1.0 / M)).all()                       # outside every window
            # events no model keeps: 1/M
            kept_any = np.zeros(off[1], bool)
            for m in range(M):
                xw, yw = S.R.warp_f32(kind, x[:off[1]], y[:off[1]], d[:off[1]], params[0, m], CENTRE)
                kept_any |= S.R.contributes(xw, yw, H, W)
            if (~kept_any).any():
                assert np.allclose(got[:off[1]][~kept_any], 1.0 / M, rtol=1e-6)
    # a NaN event changes its own row only (its weight is 0 in both runs, so the images are the same)
    M = 3
    w = memberships(x.shape[0], M, seed=4)
    e = int(off[2]) + 17
    w[e] = 0.0
    params = models("rotation", len(sizes), M)
    kw = dict(t0=0.0, blur_sigma=1.0, img_size=(H, W), batch_end_indices=torch.from_numpy(off[1:]).cuda())
    outs = []
    for xx in (x, np.where(np.arange(x.shape[0]) == e, np.float32(np.nan), x).astype(np.float32)):
        args = [torch.from_numpy(a).cuda() for a in (xx, y, d, np.abs(p))]
        outs.append(motion_segmentation_assign_torch(*args, torch.tensor(params, device="cuda"), _warp("rotation"),
                                                     torch.from_numpy(w).cuda(), **kw).cpu().numpy())
    other = np.arange(x.shape[0]) != e
    np.testing.assert_allclose(outs[1][other], outs[0][other], rtol=1e-6, atol=1e-7)
    assert np.allclose(outs[1][e], 1.0 / M)


# ---- the fit ------------------------------------------------------------------------------------------------------------
def seg_windows(kind, B, rng, n_pts=150, per_pt=100):
    """B windows, each of 3 (linvel) or 2 (rotation) disjoint point scenes side by side, every scene moving with its own
    motion; returns the events (|p| = 1), the window ends, the truths (B,M,K) and every event's scene"""
    S_ = 3 if kind == "linvel" else 2
    centres = [(60.0, 90.0), (120.0, 90.0), (180.0, 90.0)] if S_ == 3 else [(65.0, 90.0), (175.0, 90.0)]
    radius = 25.0 if S_ == 3 else 40.0          # a rotation's centre needs a wider scene to be pinned down
    xs, ys, ts, labels, ends, truths = [], [], [], [], [], []
    duration = 0.2 if kind == "linvel" else 0.05
    for b in range(B):
        if kind == "linvel":
            signs = np.array([[1, 1], [-1, 1], [1, -1]]) * rng.choice([-1, 1])
            tr = signs * rng.uniform(25, 60, (3, 2))
        else:
            om = rng.uniform(3, 8, 2) * np.array([1, -1]) * rng.choice([-1, 1])
            tr = np.array([[c[0] + rng.uniform(-5, 5), c[1] + rng.uniform(-5, 5), o] for c, o in zip(centres, om)])
        truths.append(tr)
        parts = []
        for s in range(S_):
            x0, y0, _ = _scene(rng, n_pts, per_pt, centres[s], radius)
            t = rng.uniform(0, duration, x0.size)
            parts.append((x0, y0, t, np.full(x0.size, s)))
        x0, y0, t, lab = (np.concatenate(a) for a in zip(*parts))
        order = np.argsort(t, kind="stable")
        x0, y0, t, lab = x0[order], y0[order], t[order], lab[order]
        dt = t - t[-1]
        x, y = np.empty_like(x0), np.empty_like(y0)
        for s in range(S_):
            k = lab == s
            if kind == "linvel":
                x[k], y[k] = x0[k] + dt[k] * tr[s, 0], y0[k] + dt[k] * tr[s, 1]
            else:
                a = tr[s, 2] * dt[k]
                u, v = x0[k] - tr[s, 0], y0[k] - tr[s, 1]
                x[k], y[k] = tr[s, 0] + np.cos(a) * u - np.sin(a) * v, tr[s, 1] + np.sin(a) * u + np.cos(a) * v
        xs.append(x), ys.append(y), ts.append(t), labels.append(lab)
        ends.append(sum(len(a) for a in xs))
    ev = [np.concatenate(a) for a in (xs, ys, ts)]
    return ev, ends, np.array(truths), np.concatenate(labels)


def _start(kind, truths, rng):
    if kind == "rotation":
        return np.concatenate((truths[..., :2] + rng.uniform(-2, 2, truths[..., :2].shape),
                               truths[..., 2:] * rng.uniform(0.85, 1.15, truths[..., 2:].shape)), axis=-1)
    return truths * (1 + rng.uniform(-0.15, 0.15, truths.shape))


def _run_fit(kind, B, seed, **kw):
    from event_utils_b200.contrast_max import motion_segmentation_fit_torch
    rng = np.random.default_rng(seed)
    (x, y, t), ends, truths, labels = seg_windows(kind, B, rng)
    ev = [torch.from_numpy(x).float().cuda(), torch.from_numpy(y).float().cuda(), torch.from_numpy(t).cuda(),
          torch.ones(x.shape[0], device="cuda")]
    x0 = torch.tensor(_start(kind, truths, rng), device="cuda")
    fit = motion_segmentation_fit_torch(*ev, _warp(kind, (120.0, 90.0)), x0, batch_end_indices=torch.tensor(ends, device="cuda"),
                                        **kw)
    return fit, truths, labels, ev, ends


# share of events whose argmax label is their scene's; observed on an H100 (80 GB HBM3, 700 W): linvel 0.9993,
# rotation 0.9997
LABEL_SHARE = {"linvel": 0.99, "rotation": 0.99}
# models within the tolerance; observed: linvel 95 of 96, rotation 58 of 64 (each other one at an f below the truth's)
RECOVERED_SHARE = {"linvel": 0.95, "rotation": 0.85}


@pytest.mark.parametrize("kind", ["linvel", "rotation"])
def test_fit_recovers_every_motion_and_labels_the_events(kind):
    """every model within test_gpu_motion_fit.recovered's tolerance of its scene's motion, or at an f below the
    objective's value at the true motion (with the fit's memberships): the objective's own minimum then lies outside
    the tolerance, so no minimiser of f meets it (a few small scenes per window pin a rotation's centre loosely)"""
    from event_utils_b200.contrast_max import motion_segmentation_objective_torch
    fit, truths, labels, ev, ends = _run_fit(kind, 32, {"linvel": 91, "rotation": 92}[kind], blur_sigma=1.0, em_iters=8,
                                             max_iter=20, param_scale=[1.0, 1.0] if kind == "linvel" else [0.5, 0.5, 0.05])
    got = fit.params.cpu().numpy()
    B, M, K = got.shape
    ok = recovered(kind, got.reshape(B * M, K), truths.reshape(B * M, K))
    f_true = motion_segmentation_objective_torch(*ev, fit.weights, torch.tensor(truths, device="cuda"), _warp(kind, (120.0, 90.0)),
                                                 blur_sigma=1.0, batch_end_indices=torch.tensor(ends, device="cuda"))
    beyond = ~ok & (fit.f.cpu().numpy().reshape(-1) < f_true.cpu().numpy().reshape(-1))
    share = float((fit.weights.argmax(1).cpu().numpy() == labels).mean())
    print("%s: label share %.4f, %d of %d models recovered, %d beyond at a lower f" % (kind, share, ok.sum(), ok.size, beyond.sum()))
    assert (ok | beyond).all() and ok.mean() >= RECOVERED_SHARE[kind], \
        (np.flatnonzero(~ok), got.reshape(B * M, K)[~ok], truths.reshape(B * M, K)[~ok])
    assert share >= LABEL_SHARE[kind], share
    assert fit.weights.dtype == torch.float32 and fit.f.shape == (B, M) and fit.status.dtype == torch.int8
    assert fit.iterations.dtype == torch.int32 and fit.params.dtype == torch.float64
    # f is each model's objective at the returned params and weights
    f = motion_segmentation_objective_torch(*ev, fit.weights, fit.params, _warp(kind, (120.0, 90.0)), blur_sigma=1.0,
                                            batch_end_indices=torch.tensor(ends, device="cuda"))
    np.testing.assert_allclose(fit.f.cpu().numpy(), f.cpu().numpy(), rtol=1e-6, atol=0)


def test_fit_empty_and_nan_windows_change_no_other_window():
    from event_utils_b200.contrast_max import motion_segmentation_fit_torch
    rng = np.random.default_rng(81)
    (x, y, t), ends, truths, _ = seg_windows("rotation", 4, rng, n_pts=80, per_pt=60)
    e = np.array(ends)
    keep = np.ones(x.shape[0], bool)
    keep[e[0]:e[1]] = False                                   # window 1 is empty
    n1 = e[1] - e[0]
    ends2 = torch.tensor([e[0], e[0], e[2] - n1, e[3] - n1], device="cuda")
    ev = [torch.from_numpy(x[keep]).float().cuda(), torch.from_numpy(y[keep]).float().cuda(), torch.from_numpy(t[keep]).cuda(),
          torch.ones(int(keep.sum()), device="cuda")]
    x0 = _start("rotation", truths, rng)
    kw = dict(batch_end_indices=ends2, param_scale=[0.5, 0.5, 0.05], em_iters=3, max_iter=10)
    base = motion_segmentation_fit_torch(*ev, _warp("rotation"), torch.tensor(x0, device="cuda"), **kw)
    start = x0.copy()
    start[3, 0, 2] = np.nan
    bad = motion_segmentation_fit_torch(*ev, _warp("rotation"), torch.tensor(start, device="cuda"), **kw)
    assert (base.f[1] == base.f[1, 0]).all() and np.array_equal(base.params[1].cpu().numpy(), x0[1])
    assert np.isnan(bad.params[3, 0, 2].item()) and bad.status[3, 0].item() == 3
    assert np.isfinite(bad.params[:3].cpu().numpy()).all() and np.isfinite(bad.f[:3].cpu().numpy()).all()
    assert (bad.status[:3] != 3).all()
    # windows 0 and 2 have the same inputs in both fits; their f32 images sum in any order, and EM carries that rounding
    # into which step each line search takes, so the two fits agree to about a percent, not bit for bit
    fb, fa = bad.f[:3].cpu().numpy(), base.f[:3].cpu().numpy()
    np.testing.assert_allclose(fb[[0, 2]], fa[[0, 2]], rtol=0.03)
    wb = bad.weights.cpu().numpy()
    assert np.isfinite(wb).all()
    np.testing.assert_allclose(wb.sum(1), 1.0, rtol=1e-5)


def test_fit_no_host_sync_and_constant_launch_count():
    from event_utils_b200 import _lib
    from event_utils_b200.contrast_max import motion_segmentation_fit_torch
    L = _lib.lib()
    counts = []
    for B in (1, 16):
        rng = np.random.default_rng(90 + B)
        (x, y, t), ends, truths, _ = seg_windows("rotation", B, rng, n_pts=40, per_pt=30)
        ev = [torch.from_numpy(x).float().cuda(), torch.from_numpy(y).float().cuda(), torch.from_numpy(t).cuda(),
              torch.ones(x.shape[0], device="cuda")]
        x0 = torch.tensor(_start("rotation", truths, rng), device="cuda")
        kw = dict(batch_end_indices=torch.tensor(ends, device="cuda"), em_iters=2, max_iter=3)
        motion_segmentation_fit_torch(*ev, _warp("rotation"), x0, **kw)          # warm-up: scratch buffers, modules
        torch.cuda.synchronize()
        L.evk_prof_enable(1)
        torch.cuda.set_sync_debug_mode("error")
        try:
            fit = motion_segmentation_fit_torch(*ev, _warp("rotation"), x0, **kw)
        finally:
            torch.cuda.set_sync_debug_mode(0)
        ms, timed, launches = ctypes.c_double(), ctypes.c_longlong(), ctypes.c_longlong()
        _lib.check(L.evk_prof_collect(ctypes.byref(ms), ctypes.byref(timed), ctypes.byref(launches)))
        L.evk_prof_enable(0)
        assert torch.isfinite(fit.f).all()
        counts.append(launches.value)
    assert counts[0] == counts[1] and counts[0] > 0, counts
