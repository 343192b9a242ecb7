"""The batched losses, their candidate passes and the motion fits at their window-count limits and on skewed windows
(tests/batch_limit_streams.py: a 7x11 canvas, mostly windows of 0 to 7 events and one giant window of 2^21 + 3).

The entries map windows to grid dimensions (blockIdx.y = window in the event passes, blockIdx.z = window, candidate or
image in the image-space tails) up to the hardware limit of those dimensions, and size the event grid from the MEAN
window, so the giant window runs on one CTA in a batch and on hundreds alone.  On the exact (linvel) streams every image
is exact in f32, so images and the variance's f compare bit for bit; f of the timestamp loss to 1e-13 (an f64 sum of
f32 squares in atomic order).  Gradients compare with the f64 references within their rounding bounds, with a random
incoming gradient per window, so that reading another window's g_b shows."""
import ctypes

import numpy as np
import pytest
import torch

import batch_limit_streams as S
from batch_limit_streams import sampled_windows
import flow_objective_reference as FR
import flow_timestamp_reference as FTR
import motion_objective_reference as MR
import motion_timestamp_reference as MTR
from conftest import assert_close_to_max
from exact_bounds import gamma

pytestmark = pytest.mark.gpu

E_ARG = -1
WARP = {"linvel": 3, "rotation": 1, "xyztheta": 2}
H, W, HC, WC = S.H, S.W, S.HC, S.WC


def _L():
    from event_utils_b200 import _lib
    return _lib.lib()


def _check(rc):
    from event_utils_b200 import _lib
    _lib.check(rc)


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


class Stream:
    """a batch_limit_streams dict on the device"""

    def __init__(self, s):
        self.s = s
        self.B = len(s["sizes"])
        self.n = int(s["off"][-1])
        self.X, self.Y, self.D, self.U, self.P, self.O = (_dev(s[k]) for k in ("x", "y", "d", "tau", "p", "off"))

    def window(self, b):
        """window b alone, as a one-window stream"""
        lo, hi = int(self.s["off"][b]), int(self.s["off"][b + 1])
        s = {k: self.s[k][lo:hi] for k in ("x", "y", "d", "tau", "p")}
        s["sizes"] = np.array([hi - lo], np.int64)
        s["off"] = np.array([0, hi - lo], np.int64)
        return Stream(s)

    def select(self, idx):
        """the windows idx (host numpy), concatenated"""
        off = self.s["off"]
        ev = np.concatenate([np.arange(off[b], off[b + 1]) for b in idx]) if len(idx) else np.zeros(0, np.int64)
        s = {k: self.s[k][ev] for k in ("x", "y", "d", "tau", "p")}
        s["sizes"] = self.s["sizes"][idx]
        s["off"] = np.concatenate(([0], np.cumsum(s["sizes"]))).astype(np.int64)
        return s


# ---- the entries, called directly ----------------------------------------------------------------------------------------
def motion_contrast(st, kind, params, sigma, g=None, name=0, centre=S.CENTRE):
    """evk_cmax_motion_objective_f32 (and _grad_f32 with incoming gradient g): (f, iwe[, grad]) as device tensors"""
    L = _L()
    B = params.shape[0]
    prm = torch.as_tensor(params, dtype=torch.float64, device="cuda").contiguous()
    f = torch.full((B,), float("nan"), dtype=torch.float64, device="cuda")
    iwe = torch.empty((B, HC, WC), device="cuda")
    ws = torch.empty(max(L.evk_cmax_motion_objective_workspace_bytes(B, H, W), 256), dtype=torch.uint8, device="cuda")
    args = (st.X.data_ptr(), st.Y.data_ptr(), st.D.data_ptr(), st.P.data_ptr(), st.O.data_ptr(), B, st.n, WARP[kind],
            prm.data_ptr(), prm.shape[1], centre[0], centre[1], H, W, sigma, name, 0.0)
    rc = L.evk_cmax_motion_objective_f32(*args, f.data_ptr(), iwe.data_ptr(), ws.data_ptr(), ws.numel(), None)
    if rc:
        return rc, f
    if g is None:
        return f, iwe
    gf = torch.as_tensor(g, dtype=torch.float32, device="cuda").contiguous()
    grad = torch.empty((B, prm.shape[1]), dtype=torch.float64, device="cuda")
    _check(L.evk_cmax_motion_objective_grad_f32(*args, iwe.data_ptr(), gf.data_ptr(), grad.data_ptr(), ws.data_ptr(),
                                                ws.numel(), None))
    return f, iwe, grad


def motion_timestamp(st, kind, params, sigma, g=None, centre=S.CENTRE):
    """evk_motion_timestamp_objective_f32 (and _grad_f32): (f, T, C[, grad])"""
    L = _L()
    B = params.shape[0]
    prm = torch.as_tensor(params, dtype=torch.float64, device="cuda").contiguous()
    f = torch.full((B,), float("nan"), dtype=torch.float64, device="cuda")
    T = torch.empty((B, 2, HC, WC), device="cuda")
    C = torch.empty_like(T)
    ws = torch.empty(max(L.evk_motion_timestamp_objective_workspace_bytes(B, H, W), 256), dtype=torch.uint8, device="cuda")
    args = (st.X.data_ptr(), st.Y.data_ptr(), st.D.data_ptr(), st.U.data_ptr(), st.P.data_ptr(), st.O.data_ptr(), B, st.n,
            WARP[kind], prm.data_ptr(), prm.shape[1], centre[0], centre[1], H, W, sigma)
    rc = L.evk_motion_timestamp_objective_f32(*args, f.data_ptr(), T.data_ptr(), C.data_ptr(), ws.data_ptr(), ws.numel(), None)
    if rc:
        return rc, f
    if g is None:
        return f, T, C
    gf = torch.as_tensor(g, dtype=torch.float32, device="cuda").contiguous()
    grad = torch.empty((B, prm.shape[1]), dtype=torch.float64, device="cuda")
    _check(L.evk_motion_timestamp_objective_grad_f32(*args, T.data_ptr(), C.data_ptr(), gf.data_ptr(), grad.data_ptr(),
                                                     ws.data_ptr(), ws.numel(), None))
    return f, T, C, grad


def flow_contrast(st, flow, sigma, g=None, name=0):
    L = _L()
    B = flow.shape[0]
    fl = torch.as_tensor(flow, dtype=torch.float32, device="cuda").contiguous()
    f = torch.full((B,), float("nan"), dtype=torch.float64, device="cuda")
    iwe = torch.empty((B, HC, WC), device="cuda")
    ws = torch.empty(max(L.evk_cmax_flow_objective_workspace_bytes(B, H, W), 256), dtype=torch.uint8, device="cuda")
    args = (st.X.data_ptr(), st.Y.data_ptr(), st.D.data_ptr(), st.P.data_ptr(), st.O.data_ptr(), B, st.n, fl.data_ptr(), H, W,
            sigma, name, 0.0)
    rc = L.evk_cmax_flow_objective_f32(*args, f.data_ptr(), iwe.data_ptr(), ws.data_ptr(), ws.numel(), None)
    if rc:
        return rc, f
    if g is None:
        return f, iwe
    gf = torch.as_tensor(g, dtype=torch.float32, device="cuda").contiguous()
    grad = torch.empty((B, 2, H, W), device="cuda")
    _check(L.evk_cmax_flow_objective_grad_f32(*args, iwe.data_ptr(), gf.data_ptr(), grad.data_ptr(), ws.data_ptr(),
                                              ws.numel(), None))
    return f, iwe, grad


def flow_timestamp(st, flow, sigma, g=None):
    L = _L()
    B = flow.shape[0]
    fl = torch.as_tensor(flow, dtype=torch.float32, device="cuda").contiguous()
    f = torch.full((B,), float("nan"), dtype=torch.float64, device="cuda")
    T = torch.empty((B, 2, HC, WC), device="cuda")
    C = torch.empty_like(T)
    ws = torch.empty(max(L.evk_flow_timestamp_objective_workspace_bytes(B, H, W), 256), dtype=torch.uint8, device="cuda")
    args = (st.X.data_ptr(), st.Y.data_ptr(), st.D.data_ptr(), st.U.data_ptr(), st.P.data_ptr(), st.O.data_ptr(), B, st.n,
            fl.data_ptr(), H, W, sigma)
    rc = L.evk_flow_timestamp_objective_f32(*args, f.data_ptr(), T.data_ptr(), C.data_ptr(), ws.data_ptr(), ws.numel(), None)
    if rc:
        return rc, f
    if g is None:
        return f, T, C
    gf = torch.as_tensor(g, dtype=torch.float32, device="cuda").contiguous()
    grad = torch.empty((B, 2, H, W), device="cuda")
    _check(L.evk_flow_timestamp_objective_grad_f32(*args, T.data_ptr(), C.data_ptr(), gf.data_ptr(), grad.data_ptr(),
                                                   ws.data_ptr(), ws.numel(), None))
    return f, T, C, grad


def np_(t):
    return t.cpu().numpy()


# ---- streams, parameters and the sampled windows ------------------------------------------------------------------------
def exact_params(B, seed):
    """a velocity of the exact grid per window (window-dependent, so that reading another window's parameters shows)"""
    vel = S.exact_velocities()
    return vel[np.random.default_rng(seed).integers(0, len(vel), B)]


def random_params(kind, B, seed):
    rng = np.random.default_rng(seed)
    if kind == "rotation":
        return np.column_stack((S.CENTRE[0] + rng.uniform(-2, 2, B), S.CENTRE[1] + rng.uniform(-2, 2, B), rng.uniform(-6, 6, B)))
    return np.column_stack((rng.uniform(-20, 20, B), rng.uniform(-20, 20, B), rng.uniform(-2, 2, B), rng.uniform(-3, 3, B)))


def incoming(B, seed):
    return np.random.default_rng(seed).standard_normal(B).astype(np.float32)


def _rtol(b, giant):
    """f of a random stream's window computed twice, its images summed in different orders: to 1e-6, and the giant
    window to 1e-5 (its variance cancels the f32 rounding of 2^21 events' sums by a few 1e-6)"""
    return 1e-5 if b == giant else 1e-6


def _assert_same_f(got, f, giant):
    rest = np.arange(len(f)) != giant
    np.testing.assert_allclose(got[rest], f[rest], rtol=1e-6, atol=0)
    assert abs(got[giant] - f[giant]) <= _rtol(giant, giant) * abs(f[giant]), (got[giant], f[giant])


def _assert_grad_bound(got, ref, M, cnt, what):
    bound = gamma(cnt + 32) * M
    err = np.abs(got - ref)
    bad = err > bound
    assert not bad.any(), "%s: %d components outside the bound, e.g. err %r bound %r" % (what, bad.sum(), err[bad][:3],
                                                                                         bound[bad][:3])


# ---- 1. every batched loss at its cap, forward and backward -------------------------------------------------------------
CAP_GIANT = {S.MOTION_CAP: 40000, S.TIMESTAMP_CAP: 20000}


def _motion_reference_grad(loss, kind, sub, params, sigma, g):
    """f64 reference f and parameter gradient of the windows of `sub` (a batch_limit_streams dict), and the bound's
    magnitudes"""
    x, y, d, tau, p, off = (sub[k] for k in ("x", "y", "d", "tau", "p", "off"))
    p64 = torch.tensor(params, dtype=torch.float64, requires_grad=True)
    if loss == "contrast":
        fr, iwer, mag = MR.reference(kind, x, y, d, p, off, p64, sigma, "variance", 0.0, (H, W), S.CENTRE)
        (fr * torch.from_numpy(g.astype(np.float64))).sum().backward()
        M, cnt = MR.grad_magnitude(kind, x, y, d, p, off, p64, sigma, "variance", 0.0, g, iwer.detach().numpy(), mag.numpy(),
                                   (H, W), S.CENTRE)
    else:
        fr, Tr, Cr = MTR.reference(kind, x, y, d, tau, p, off, p64, sigma, (H, W), S.CENTRE)
        (fr * torch.from_numpy(g.astype(np.float64))).sum().backward()
        M, cnt = MTR.grad_magnitude(kind, x, y, d, tau, p, off, p64, sigma, g, Tr.detach().numpy(), Cr.detach().numpy(),
                                    (H, W), S.CENTRE)
    return fr.detach().numpy(), p64.grad.numpy(), M, cnt


MOTION_CASES = [("contrast", "linvel"), ("contrast", "rotation"), ("contrast", "xyztheta"),
                ("timestamp", "linvel"), ("timestamp", "rotation"), ("timestamp", "xyztheta")]


@pytest.mark.parametrize("loss,kind", MOTION_CASES)
def test_motion_loss_at_its_cap(loss, kind):
    cap = S.MOTION_CAP if loss == "contrast" else S.TIMESTAMP_CAP
    giant = CAP_GIANT[cap]
    exact = kind == "linvel"
    s = S.exact_stream(cap, giant, seed=11) if exact else S.random_stream(cap, giant, seed=12)
    st = Stream(s)
    params = exact_params(cap, 13) if exact else random_params(kind, cap, 14)
    sigma = 0.0 if exact else 1.0
    g = incoming(cap, 15)
    run = motion_contrast if loss == "contrast" else motion_timestamp
    out = [np_(t) for t in run(st, kind, params, sigma, g)]
    f, grad = out[0], out[-1]
    assert np.isfinite(f).all() and np.isfinite(grad).all()
    empty = s["sizes"] == 0
    assert (f[empty] == 0).all() and (grad[empty] == 0).all()
    # every window's images and f against the host's exact images (exact streams)
    if exact and loss == "contrast":
        iwe = S.linvel_iwe(s, params)
        assert np.array_equal(out[1], iwe.astype(np.float32))
        assert np.array_equal(f, S.variance_f(iwe))
    elif exact:
        Si, Ci = S.linvel_ts_images(s, params)
        fh, Th = S.timestamp_f(Si, Ci)
        assert np.array_equal(out[1], Th.astype(np.float32)) and np.array_equal(out[2], Ci.astype(np.float32))
        np.testing.assert_allclose(f, fh, rtol=1e-13, atol=0)
    # window order: the same windows reversed give the same f in reversed order
    r = S.reversed_stream(s)
    fr = np_(run(Stream(r), kind, params[::-1].copy(), sigma)[0])
    _assert_same_f(fr[::-1], f, giant)
    # the sampled windows: batch-1 calls and the f64 reference
    tail = 1 if loss == "contrast" else 2
    idx = sampled_windows(s["sizes"], giant, tail)
    for b in idx:
        one = [np_(t) for t in run(st.window(b), kind, params[b:b + 1], sigma, g[b:b + 1])]
        if exact:
            for a, c in zip(one[1:-1], out[1:-1]):
                assert np.array_equal(a[0], c[b]), b
            if loss == "contrast":
                assert one[0][0] == f[b], b
            else:
                assert abs(one[0][0] - f[b]) <= 1e-13 * abs(f[b]), b
        else:
            for a, c in zip(one[1:-1], out[1:-1]):
                assert_close_to_max(c[b], a[0], 1e-5, "window %d" % b)
            assert abs(one[0][0] - f[b]) <= _rtol(b, giant) * abs(f[b]), (b, one[0][0], f[b])
    f64, g64, M, cnt = _motion_reference_grad(loss, kind, st.select(idx), params[idx], sigma, g[idx])
    np.testing.assert_allclose(f[idx], f64, rtol=1e-5, atol=1e-30)
    _assert_grad_bound(grad[idx], g64, M, cnt, "%s %s" % (loss, kind))


@pytest.mark.parametrize("loss", ["contrast", "timestamp"])
def test_flow_loss_at_its_cap(loss):
    cap = S.MOTION_CAP if loss == "contrast" else S.TIMESTAMP_CAP
    giant = CAP_GIANT[cap]
    s = S.random_stream(cap, giant, seed=21)
    st = Stream(s)
    rng = np.random.default_rng(22)
    flow = (rng.uniform(-20, 20, (cap, 2, 1, 1)) + rng.uniform(-2, 2, (cap, 2, H, W))).astype(np.float32)
    g = incoming(cap, 23)
    sigma = 1.0
    run = flow_contrast if loss == "contrast" else flow_timestamp
    out = [np_(t) for t in run(st, flow, sigma, g)]
    f, grad = out[0], out[-1]
    assert np.isfinite(f).all() and np.isfinite(grad).all()
    empty = s["sizes"] == 0
    assert (f[empty] == 0).all() and (grad[empty] == 0).all()
    r = S.reversed_stream(s)
    fr = np_(run(Stream(r), flow[::-1].copy(), sigma)[0])
    _assert_same_f(fr[::-1], f, giant)
    idx = sampled_windows(s["sizes"], giant, 1 if loss == "contrast" else 2, seed=1)
    for b in idx:
        one = [np_(t) for t in run(st.window(b), flow[b:b + 1], sigma)]
        for a, c in zip(one[1:], out[1:-1]):
            assert_close_to_max(c[b], a[0], 1e-5, "window %d" % b)
        assert abs(one[0][0] - f[b]) <= _rtol(b, giant) * abs(f[b]), (b, one[0][0], f[b])
    sub = st.select(idx)
    x, y, d, tau, p, off = (sub[k] for k in ("x", "y", "d", "tau", "p", "off"))
    fl64 = torch.tensor(flow[idx], dtype=torch.float64, requires_grad=True)
    gs = g[idx]
    if loss == "contrast":
        f64, iwer, mag = FR.reference(x, y, d, p, off, fl64, sigma, "variance", 0.0)
        (f64 * torch.from_numpy(gs.astype(np.float64))).sum().backward()
        M, cnt = FR.grad_magnitude(x, y, d, p, off, fl64, sigma, "variance", 0.0, gs, iwer.detach().numpy(), mag.numpy())
    else:
        f64, Tr, Cr = FTR.reference(x, y, d, tau, p, off, fl64, sigma)
        (f64 * torch.from_numpy(gs.astype(np.float64))).sum().backward()
        M, cnt = FTR.grad_magnitude(x, y, d, tau, p, off, fl64, sigma, gs, Tr.detach().numpy(), Cr.detach().numpy())
    np.testing.assert_allclose(f[idx], f64.detach().numpy(), rtol=1e-5, atol=1e-30)
    _assert_grad_bound(grad[idx], fl64.grad.numpy(), M, cnt, "flow %s" % loss)


def test_cap_plus_one_is_refused():
    """batch = cap + 1 is EVK_E_ARG before any launch: the NaN-filled f stays untouched"""
    s = S.exact_stream(S.MOTION_CAP + 1, None, seed=31)
    st = Stream(s)
    ps = exact_params(S.MOTION_CAP + 1, 32)
    flow = np.zeros((S.MOTION_CAP + 1, 2, H, W), np.float32)
    for rc, f in (motion_contrast(st, "linvel", ps, 0.0), flow_contrast(st, flow, 0.0)):
        assert rc == E_ARG and torch.isnan(f).all()
    t = S.TIMESTAMP_CAP + 1
    sub = Stream(st.select(np.arange(t)))
    for rc, f in (motion_timestamp(sub, "linvel", ps[:t], 0.0), flow_timestamp(sub, flow[:t], 0.0)):
        assert rc == E_ARG and torch.isnan(f).all()
    # one window fewer runs
    assert motion_contrast(Stream(st.select(np.arange(S.MOTION_CAP))), "linvel", ps[:-1], 0.0)[0].shape == (S.MOTION_CAP,)


# ---- 2. the candidate passes at their caps, and the Python chunking -----------------------------------------------------
def candidates_entry(loss, st, cand, sigma):
    """evk_cmax_motion_candidates_f32 / evk_motion_timestamp_candidates_f32 (linvel) directly: (rc, f (B,J))"""
    L = _L()
    B, J, K = cand.shape
    c = torch.as_tensor(cand, dtype=torch.float64, device="cuda").contiguous()
    f = torch.full((B, J), float("nan"), dtype=torch.float64, device="cuda")
    if loss == "contrast":
        ws = torch.empty(max(L.evk_cmax_motion_candidates_workspace_bytes(B, J, H, W), 256), dtype=torch.uint8, device="cuda")
        rc = L.evk_cmax_motion_candidates_f32(st.X.data_ptr(), st.Y.data_ptr(), st.D.data_ptr(), st.P.data_ptr(), st.O.data_ptr(),
                                              B, st.n, WARP["linvel"], c.data_ptr(), J, K, 0.0, 0.0, H, W, sigma, 0, 0.0,
                                              f.data_ptr(), ws.data_ptr(), ws.numel(), None)
    else:
        ws = torch.empty(max(L.evk_motion_timestamp_candidates_workspace_bytes(B, J, H, W), 256), dtype=torch.uint8,
                         device="cuda")
        rc = L.evk_motion_timestamp_candidates_f32(st.X.data_ptr(), st.Y.data_ptr(), st.D.data_ptr(), st.U.data_ptr(),
                                                   st.P.data_ptr(), st.O.data_ptr(), B, st.n, WARP["linvel"], c.data_ptr(), J, K,
                                                   0.0, 0.0, H, W, sigma, f.data_ptr(), ws.data_ptr(), ws.numel(), None)
    return rc, f


def exact_candidates(B, J, seed):
    vel = S.exact_velocities()
    return vel[np.random.default_rng(seed).integers(0, len(vel), (B, J))]


def _per_candidate_forward(loss, st, cand):
    run = motion_contrast if loss == "contrast" else motion_timestamp
    return np.stack([np_(run(st, "linvel", cand[:, j].copy(), 0.0)[0]) for j in range(cand.shape[1])], axis=1)


def _assert_equal_f(loss, got, ref, what):
    if loss == "contrast":
        assert np.array_equal(got, ref), what
    else:
        np.testing.assert_allclose(got, ref, rtol=1e-13, atol=0, err_msg=what)


@pytest.mark.parametrize("loss,B,J", [("contrast", 65535, 1), ("contrast", 2047, 32), ("timestamp", 32767, 1),
                                      ("timestamp", 1023, 32)])
def test_candidates_entry_at_its_cap(loss, B, J):
    s = S.exact_stream(B, B // 2, seed=41)
    st = Stream(s)
    cand = exact_candidates(B, J, 42)
    rc, f = candidates_entry(loss, st, cand, 0.0)
    _check(rc)
    f = np_(f)
    _assert_equal_f(loss, f, _per_candidate_forward(loss, st, cand), "%s (%d, %d)" % (loss, B, J))
    # the f64 value of the exact images, every window and candidate
    for j in range(J):
        if loss == "contrast":
            ref = S.variance_f(S.linvel_iwe(s, cand[:, j]))
        else:
            ref = S.timestamp_f(*S.linvel_ts_images(s, cand[:, j]))[0]
        _assert_equal_f(loss, f[:, j], ref, "%s host j=%d" % (loss, j))
    # one more window (J more canvases, past the cap) is refused before any launch
    st2 = Stream(st.select(np.concatenate((np.arange(B), [0]))))
    rc, f2 = candidates_entry(loss, st2, np.concatenate((cand, cand[:1]), axis=0), 0.0)
    assert rc == E_ARG and torch.isnan(f2).all()


@pytest.mark.parametrize("loss,B", [("contrast", 4095), ("timestamp", 2047)])
def test_candidates_through_the_window_chunks(loss, B):
    """motion_contrast_candidates_torch / motion_timestamp_candidates_torch at B = 4095 (2047 + 2047 + 1 windows) /
    2047 (1023 + 1023 + 1) with J = 70 (passes of 32 + 32 + 6), the giant window at the first chunk boundary.  Every
    f[b, j] equals the torch forward at params[b] = candidates[b, j] (contrast: bit for bit; timestamp, whose stamps the
    torch functions normalise and are not exact: to 1e-6, the giant window to 1e-5), and the sampled windows match the
    host's f64 value of their images"""
    from event_utils_b200.contrast_max import (linvel_warp, motion_contrast_candidates_torch, motion_contrast_objective_torch,
                                               motion_timestamp_candidates_torch, motion_timestamp_objective_torch)
    wb = 2047 if loss == "contrast" else 1023
    s = S.exact_stream(B, wb, seed=51)
    st = Stream(s)
    cand = exact_candidates(B, 70, 52)
    ev, ends = (st.X, st.Y, st.D, st.P), st.O[1:]
    if loss == "contrast":
        kw = dict(t0=0.0, objective="variance", blur_sigma=0.0, img_size=(H, W), batch_end_indices=ends)
        f = np_(motion_contrast_candidates_torch(*ev, torch.tensor(cand, device="cuda"), linvel_warp(), **kw))
        ref = np.stack([np_(motion_contrast_objective_torch(*ev, torch.tensor(cand[:, j], device="cuda"), linvel_warp(), **kw))
                        for j in range(cand.shape[1])], axis=1)
        assert np.array_equal(f, ref)
    else:
        kw = dict(t0=0.0, blur_sigma=0.0, img_size=(H, W), batch_end_indices=ends)
        f = np_(motion_timestamp_candidates_torch(*ev, torch.tensor(cand, device="cuda"), linvel_warp(), **kw))
        ref = np.stack([np_(motion_timestamp_objective_torch(*ev, torch.tensor(cand[:, j], device="cuda"), linvel_warp(), **kw))
                        for j in range(cand.shape[1])], axis=1)
        for j in range(cand.shape[1]):
            _assert_same_f(f[:, j], ref[:, j], wb)
    idx = sampled_windows(s["sizes"], wb, 1 if loss == "contrast" else 2, count=24)
    sub = st.select(idx)
    if loss == "timestamp":
        sub["tau"] = FTR.tau_f32(sub["d"], sub["off"])                 # the stamps the torch functions form
    for j in range(cand.shape[1]):
        if loss == "contrast":
            assert np.array_equal(f[idx, j], S.variance_f(S.linvel_iwe(sub, cand[idx, j]))), j
        else:
            Si, Ci = S.linvel_ts_images(sub, cand[idx, j])
            host = ((Si / Ci) ** 2).sum(axis=(1, 2, 3))
            # f32 sums against f64 ones: 1e-5, and the giant window's 2^21 taps to 1e-4
            tol = np.where(idx == wb, 1e-4, 1e-5) * np.abs(host)
            assert (np.abs(f[idx, j] - host) <= tol).all(), (j, idx, f[idx, j], host)


# ---- 3. skew: the giant window at the start, in the middle and at the end -----------------------------------------------
@pytest.mark.parametrize("loss", ["contrast", "timestamp"])
@pytest.mark.parametrize("where", ["first", "middle", "last"])
def test_giant_window_in_a_batch_equals_it_alone(loss, where):
    B = 4095
    giant = {"first": 0, "middle": B // 2, "last": B - 1}[where]
    s = S.exact_stream(B, giant, seed=61)
    st = Stream(s)
    params = exact_params(B, 62)
    g = incoming(B, 63)
    run = motion_contrast if loss == "contrast" else motion_timestamp
    out = [np_(t) for t in run(st, "linvel", params, 0.0, g)]
    one = [np_(t) for t in run(st.window(giant), "linvel", params[giant:giant + 1], 0.0, g[giant:giant + 1])]
    for a, c in zip(one[1:-1], out[1:-1]):
        assert np.array_equal(a[0], c[giant])
    _assert_equal_f(loss, np.array([out[0][giant]]), one[0], "f")
    _, g64, M, cnt = _motion_reference_grad(loss, "linvel", st.select([giant]), params[giant:giant + 1], 0.0, g[giant:giant + 1])
    _assert_grad_bound(out[-1][giant:giant + 1], g64, M, cnt, "batched")
    _assert_grad_bound(one[-1], g64, M, cnt, "alone")


def _voxel_dev(s):
    return [_dev(s[k]) for k in ("x", "y", "t", "p")]


def voxel_windows(ev, off, n, grads=None):
    """evk_voxel_windows_f32 on the windows of `off` (host), n_events_hint = n; with `grads` (the incoming gradient
    (n_windows, B, H, W)) also the windowed evk_voxel_grad_f32: (grid[, grad_p, grad_t]) as numpy"""
    L = _L()
    nw, B = len(off) - 1, S.VOXEL_BINS
    X, Y, T, P = ev
    O = _dev(off)
    out = torch.full((nw, B, H, W), float("nan"), device="cuda")
    oob = torch.zeros(1, dtype=torch.int64, device="cuda")
    _check(L.evk_voxel_windows_f32(X.data_ptr(), Y.data_ptr(), T.data_ptr(), P.data_ptr(), O.data_ptr(), nw, n, B, H, W, 0,
                                   out.data_ptr(), oob.data_ptr(), None))
    if grads is None:
        return np_(out)
    pairs = _dev(np.stack((off[:-1], off[1:]), axis=1))
    gp = torch.full((n,), float("nan"), device="cuda")
    gt = torch.full((n,), float("nan"), device="cuda")
    ws = torch.empty(L.evk_voxel_grad_workspace_bytes(nw, B, H, W, 0), dtype=torch.uint8, device="cuda")
    g = _dev(grads)
    _check(L.evk_voxel_grad_f32(X.data_ptr(), Y.data_ptr(), T.data_ptr(), P.data_ptr(), n, pairs.data_ptr(), nw, B, H, W, 0,
                                g.data_ptr(), gp.data_ptr(), gt.data_ptr(), ws.data_ptr(), ws.numel(), None))
    return np_(out), np_(gp), np_(gt)


VOXEL_WINDOWS = 100000


@pytest.mark.parametrize("where", ["first", "middle", "last"])
def test_voxel_windows_giant_window_in_a_batch_equals_it_alone(where):
    """100 k windows of 0 to 7 events and one giant window on exact stamps (tests/batch_limit_streams.voxel_stream):
    every window's grid equals the host's exact grid, the giant's and the sampled windows' grids and per-event
    gradients (grad_p, grad_t) equal their single-window build and backward bit for bit, and the windows in reverse
    order give the same grids and per-event gradients"""
    nw = VOXEL_WINDOWS
    giant = {"first": 0, "middle": nw // 2, "last": nw - 1}[where]
    s = S.voxel_stream(nw, giant, seed=101)
    off, sizes, n = s["off"], s["sizes"], int(s["off"][-1])
    g = S.voxel_incoming(nw, 102)
    grid, gp, gt = voxel_windows(_voxel_dev(s), off, n, g)
    host = S.voxel_grids(s)
    ok = sizes != 1                                    # a one-event window has dt = 0: NaN in its event's pixel
    assert np.array_equal(grid[ok], host[ok].astype(np.float32))
    assert np.isnan(grid[sizes == 1]).any(axis=(1, 2, 3)).all()
    m = sizes[S.window_ids(off)] >= 2
    assert np.array_equal(gp[m], S.voxel_grad_p(s, g)[m].astype(np.float32))
    assert np.isfinite(gt[m]).all()
    for b in sampled_windows(sizes, giant, 1, seed=103):
        lo, hi = int(off[b]), int(off[b + 1])
        if hi == lo:
            assert (grid[b] == 0).all()
            continue
        alone = {k: s[k][lo:hi] for k in ("x", "y", "t", "p")}
        g1, gp1, gt1 = voxel_windows(_voxel_dev(alone), np.array([0, hi - lo], np.int64), hi - lo, g[b:b + 1])
        assert np.array_equal(g1[0], grid[b], equal_nan=True), b
        assert np.array_equal(gp1, gp[lo:hi], equal_nan=True), b
        assert np.array_equal(gt1, gt[lo:hi], equal_nan=True), b
    r = S.reversed_stream(s)
    rgrid, rgp, rgt = voxel_windows(_voxel_dev(r), r["off"], n, g[::-1].copy())
    assert np.array_equal(rgrid[::-1], grid, equal_nan=True)
    order = np.concatenate([np.arange(off[b], off[b + 1]) for b in range(nw - 1, -1, -1)])
    assert np.array_equal(rgp, gp[order], equal_nan=True) and np.array_equal(rgt, gt[order], equal_nan=True)


# ---- 4. the fits across the window chunks and past the entries' caps ----------------------------------------------------
def _fit(loss, st, B, t0=0.0, **kw):
    from event_utils_b200.contrast_max import linvel_warp, motion_contrast_fit_torch, motion_timestamp_fit_torch
    ends = st.O[1:]
    if loss == "contrast":
        return motion_contrast_fit_torch(st.X, st.Y, st.D, st.P, linvel_warp(), batch_end_indices=ends, t0=t0,
                                         objective="variance", blur_sigma=0.0, img_size=(H, W), **kw)
    return motion_timestamp_fit_torch(st.X, st.Y, st.D, st.P, linvel_warp(), batch_end_indices=ends, t0=t0, blur_sigma=0.0,
                                      img_size=(H, W), **kw)


def _f_at(loss, s, params, t0=0.0):
    """the loss at params, in calls of at most the entries' cap, each on its own sub-stream"""
    cap = S.MOTION_CAP if loss == "contrast" else S.TIMESTAMP_CAP
    from event_utils_b200.contrast_max import linvel_warp, motion_contrast_objective_torch, motion_timestamp_objective_torch
    B = len(s["sizes"])
    whole = Stream(s)
    out = []
    for b0 in range(0, B, cap):
        idx = np.arange(b0, min(B, b0 + cap))
        sub = Stream(whole.select(idx))
        ev = (sub.X, sub.Y, sub.D, sub.P)
        prm = torch.tensor(params[b0:b0 + len(idx)], dtype=torch.float64, device="cuda")
        if loss == "contrast":
            f = motion_contrast_objective_torch(*ev, prm, linvel_warp(), t0=t0, objective="variance", blur_sigma=0.0,
                                                img_size=(H, W), batch_end_indices=sub.O[1:])
        else:
            f = motion_timestamp_objective_torch(*ev, prm, linvel_warp(), t0=t0, blur_sigma=0.0, img_size=(H, W),
                                                 batch_end_indices=sub.O[1:])
        out.append(np_(f))
    return np.concatenate(out)


@pytest.mark.parametrize("loss,B", [("contrast", 2622), ("timestamp", 1311)])
def test_grid_start_across_window_chunks(loss, B):
    """max_iter = 0 returns the grid start; B is one window past the grid level's candidates chunk (J = 25).  Every
    window's start equals the one it gets in a fit of at most 64 windows (for the timestamp loss, whose stamps are not
    exact, a different start only where the two f tie to 1e-13)"""
    s = S.exact_stream(B, None, seed=71)
    st = Stream(s)
    kw = dict(param_ranges=S.EXACT_RANGES, num_samples_per_param=5, max_iter=0)
    fit = _fit(loss, st, B, **kw)
    start, f = np_(fit.params), np_(fit.f)
    assert (np_(fit.iterations) == 0).all()
    for b0 in range(0, B, 64):
        idx = np.arange(b0, min(B, b0 + 64))
        part = _fit(loss, Stream(st.select(idx)), len(idx), **kw)
        ps, pf = np_(part.params), np_(part.f)
        same = (ps == start[idx]).all(1)
        if loss == "contrast":
            assert same.all() and np.array_equal(pf, f[idx]), np.flatnonzero(~same) + b0
        else:
            tie = np.abs(pf - f[idx]) <= 1e-13 * np.abs(f[idx])
            assert (same | tie).all(), np.flatnonzero(~(same | tie)) + b0


def _launches(fn):
    from event_utils_b200 import _lib
    L = _lib.lib()
    torch.cuda.synchronize()
    L.evk_prof_enable(1)
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = fn()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    ms, timed, launches = ctypes.c_double(), ctypes.c_longlong(), ctypes.c_longlong()
    _lib.check(L.evk_prof_collect(ctypes.byref(ms), ctypes.byref(timed), ctypes.byref(launches)))
    L.evk_prof_enable(0)
    return out, launches.value


def _unit_launches(loss):
    """the launches of one candidates entry call and of one forward + gradient pair (sigma 0)"""
    from event_utils_b200.contrast_max import motion_fit as MF
    from event_utils_b200.contrast_max import motion_objective as MO
    from event_utils_b200.contrast_max import motion_timestamp_fit as MTF
    from event_utils_b200.contrast_max import motion_timestamp_objective as MT
    one = Stream(S.exact_stream(1, None, seed=90))
    c1 = torch.zeros((1, 1, 2), dtype=torch.float64, device="cuda")
    if loss == "contrast":
        opts = (WARP["linvel"], (0.0, 0.0), H, W, 0, 0.0, 0.0)
        cand = lambda: MO._candidates(one.X, one.Y, one.D, one.P, one.O, c1, opts)
        fg = MF._objective_and_gradient(one.X, one.Y, one.D, one.P, one.O, opts)
    else:
        opts = (WARP["linvel"], (0.0, 0.0), H, W, 0.0)
        cand = lambda: MT._ts_candidates(one.X, one.Y, one.D, one.U, one.P, one.O, c1, opts)
        fg = MTF._objective_and_gradient(one.X, one.Y, one.D, one.U, one.P, one.O, opts)
    cand()
    fg(c1[0])
    Lc, Lf = _launches(cand)[1], _launches(lambda: fg(c1[0]))[1]
    assert Lc > 0 and Lf > 0
    return Lc, Lf


def _ceil(a, b):
    return -(-a // b)


@pytest.mark.parametrize("loss,B", [("contrast", 65536), ("timestamp", 32768)])
def test_short_fit_past_the_entry_cap(loss, B):
    """B one past the forward and gradient entries' cap: the fit runs them in two chunks of windows, without a host
    synchronisation, with the launches that chunk count predicts, and every window's f is the loss at its params"""
    cap = S.MOTION_CAP if loss == "contrast" else S.TIMESTAMP_CAP
    Lc, Lf = _unit_launches(loss)
    s = S.exact_stream(B, None, seed=81)
    st = Stream(s)
    x0 = torch.tensor(exact_params(B, 82), dtype=torch.float64, device="cuda")
    max_iter = 3
    kw = dict(x0=x0, param_scale=torch.tensor([16.0, 16.0], dtype=torch.float64, device="cuda"), max_iter=max_iter)
    if loss == "timestamp":
        kw["bounds"] = torch.tensor(S.EXACT_RANGES, dtype=torch.float64, device="cuda")
    _fit(loss, st, B, t0=None, **kw)                                       # warm-up: scratch buffers
    fit, n = _launches(lambda: _fit(loss, st, B, t0=None, **kw))
    assert n == max_iter * _ceil(B, cap // 8) * Lc + (1 + max_iter) * _ceil(B, cap) * Lf, n
    f = np_(fit.f)
    assert f.shape == (B,) and np.isfinite(f).all()
    np.testing.assert_allclose(f, _f_at(loss, s, np_(fit.params), t0=None), rtol=1e-6, atol=0)
    assert (np_(fit.params)[s["sizes"] == 0] == np_(x0)[s["sizes"] == 0]).all()


@pytest.mark.parametrize("loss", ["contrast", "timestamp"])
def test_launch_count_follows_the_window_chunks(loss):
    """launches = grid chunks x (launches of one candidates call) + max_iter x line-search chunks x (the same) +
    (1 + max_iter) x forward/gradient chunks x (launches of one forward + gradient), with no host synchronisation"""
    cap = S.MOTION_CAP if loss == "contrast" else S.TIMESTAMP_CAP
    grid_wb, ls_wb = cap // 25, cap // 8
    max_iter = 2
    Lc, Lf = _unit_launches(loss)
    for B in (1, 64, grid_wb + 1, 2 * grid_wb + 1):
        st = Stream(S.exact_stream(B, None, seed=91 + B))
        kw = dict(param_ranges=torch.tensor(S.EXACT_RANGES, dtype=torch.float64, device="cuda"), num_samples_per_param=5,
                  max_iter=max_iter)
        _fit(loss, st, B, t0=None, **kw)                                   # warm-up: scratch buffers
        fit, n = _launches(lambda: _fit(loss, st, B, t0=None, **kw))
        want = _ceil(B, grid_wb) * Lc + max_iter * _ceil(B, ls_wb) * Lc + (1 + max_iter) * _ceil(B, cap) * Lf
        assert n == want, (B, n, want)
        assert torch.isfinite(fit.f).all()
