"""The newer families' batched entries, candidate passes and fits at their window-count limits and on skewed windows
(tests/batch_limit_streams.py: a 7x11 canvas, mostly windows of 0 to 7 events and one giant window of 2^21 + 3): the
affine and homography models, the camera rotation and camera motion, the grid flow, the depth grid and the
segmentation, each through the window-dependent code of its own entries (per-window rows, focal lengths, motion rows,
per-event inverse depth, node grids, memberships, per-candidate NaN masks).

Exact variant: each family's parameters that reproduce the linvel warp (batch_limit_streams.exact_rows, proved exact by
tests/test_batch_limits_models_cpu.py), one velocity per window, so every image and the variance's f equal the host's
f64 images bit for bit, and the timestamp loss's f to 1e-13.  Random variant: every parameter in play, checked against
the f64 references; events of the checked windows that lie within 1e-3 px of an integer add no term.  Gradients are
checked per component against the rounding bounds of tests/model_grad_bounds.py with a random incoming gradient per
window (mixed signs, one zero), so that a kernel reading another window's values shows.  The f64 references run on the
sampled windows; the giant window's own reference runs in the giant-window tests."""
import ctypes

import numpy as np
import pytest
import torch

import batch_limit_streams as S
import camera_motion_reference as CM
import camera_rotation_reference as CR
import candidate_checks as CC
import depth_grid_reference as DR
import depth_grid_timestamp_reference as DTR
import grid_flow_reference as GR
import grid_flow_timestamp_reference as GTR
import model_grad_bounds as MB
import planar_motion_reference as P

pytestmark = pytest.mark.gpu

E_ARG = -1
H, W, HC, WC = S.H, S.W, S.HC, S.WC
MOTION_CAP, TS_CAP = S.MOTION_CAP, S.TIMESTAMP_CAP
WARP = {"affine": 4, "homography": 5, "camera_rotation": 6, "camera_motion": 7, "segmentation": 4}
GIANT_AT = {MOTION_CAP: 40000, TS_CAP: 20000}
EVENT_KEYS = ("x", "y", "d", "tau", "p", "r", "w")


def _L():
    from event_utils_b200 import _lib
    return _lib.lib()


def _check(rc):
    from event_utils_b200 import _lib
    _lib.check(rc)


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def np_(t):
    return t.cpu().numpy()


class Stream:
    """a batch_limit_streams dict on the device, with its inverse depth r and memberships w"""

    def __init__(self, s):
        self.s = s
        self.B = len(s["sizes"])
        self.n = int(s["off"][-1])
        self.t = {k: _dev(s[k]) for k in EVENT_KEYS + ("off",) if k in s}

    def select(self, idx):
        """the windows idx, concatenated, as a host dict"""
        off = self.s["off"]
        ev = np.concatenate([np.arange(off[b], off[b + 1]) for b in idx]) if len(idx) else np.zeros(0, np.int64)
        s = {k: self.s[k][ev] for k in EVENT_KEYS if k in self.s}
        s["sizes"] = self.s["sizes"][np.asarray(idx)]
        s["off"] = np.concatenate(([0], np.cumsum(s["sizes"]))).astype(np.int64)
        return s

    def window(self, b):
        return Stream(self.select([b]))


# ---- the families' parameters ----------------------------------------------------------------------------------------
class Params:
    """one family's per-window parameters: `rows` (B,K) f64 ((B,M,K) for the segmentation) of the motion entries, or
    `grids` f32 node grids with, for the depth grid, `rows` the (B,8) motion rows"""

    def __init__(self, family, rows=None, grids=None):
        self.family, self.rows, self.grids = family, rows, grids

    def take(self, idx):
        idx = np.asarray(idx)
        return Params(self.family, None if self.rows is None else self.rows[idx].copy(),
                      None if self.grids is None else self.grids[idx].copy())

    def reversed(self):
        return self.take(np.arange(self.B - 1, -1, -1))

    @property
    def B(self):
        return (self.rows if self.rows is not None else self.grids).shape[0]

    def of(self, b):
        """window b's parameter sets, one per model, as batch_limit_streams.family_warp takes them"""
        if self.family == "segmentation":
            return list(self.rows[b])
        if self.family == "grid_flow":
            return [self.grids[b]]
        if self.family == "depth_grid":
            return [(self.rows[b], self.grids[b])]
        return [self.rows[b]]


def exact_params(family, B, stream_seed, seed, M=None):
    """(Params, vel): a velocity of EXACT_VELOCITIES per window (and model) embedded in the family, with the window
    rhos of the sensor_stream of `stream_seed`"""
    vel = S.exact_velocity_set((B,) if M is None else (B, M), seed)
    out = S.exact_rows(family, vel, S.window_rhos(B, stream_seed))
    if family == "grid_flow":
        return Params(family, grids=np.ascontiguousarray(out)), vel
    if family == "depth_grid":
        return Params(family, rows=out[0], grids=np.ascontiguousarray(out[1])), vel
    return Params(family, rows=out), vel


def random_params(family, B, seed, M=None):
    out = S.random_rows(family, B, seed, M)
    if family == "grid_flow":
        return Params(family, grids=out)
    if family == "depth_grid":
        return Params(family, rows=out[0], grids=out[1])
    return Params(family, rows=out)


def make_stream(exact, B, giant, seed, M=None):
    return S.sensor_stream(B, giant, seed, M) if exact else S.random_stream_models(B, giant, seed, M)


def centre(family):
    return S.INTR[2:] if family in ("camera_rotation", "camera_motion", "depth_grid") else S.CENTRE


def incoming(shape, seed, zero_in=None):
    """g_b of mixed sign and magnitude, f32 values, zero at `zero_in`"""
    rng = np.random.default_rng(seed)
    g = (rng.standard_normal(shape) * 10.0 ** rng.uniform(-1, 1, shape)).astype(np.float32)
    if zero_in is not None:
        g[zero_in] = 0.0
    return g


# ---- the entries, called directly --------------------------------------------------------------------------------------
def _stem(family, loss):
    if family == "grid_flow":
        return "evk_cmax_grid_flow" if loss == "contrast" else "evk_grid_flow_timestamp"
    if family == "depth_grid":
        return "evk_cmax_depth_grid" if loss == "contrast" else "evk_depth_grid_timestamp"
    if family == "segmentation":
        return "evk_cmax_motion_segment"
    depth = "_depth" if family == "camera_motion" else ""
    return ("evk_cmax_motion" if loss == "contrast" else "evk_motion_timestamp") + depth


def _front(family, loss, st):
    t = st.t
    ev = [t["x"], t["y"], t["d"]] + ([] if loss == "contrast" else [t["tau"]]) + [t["p"]]
    if family == "camera_motion":
        ev.append(t["r"])
    ptrs = [a.data_ptr() for a in ev]
    if family == "segmentation":
        ptrs += [t["w"].data_ptr(), t["w"].shape[1]]
    return ptrs + [t["off"].data_ptr(), st.B, st.n]


def _model_args(family, prm, keep):
    """the arguments between n_events and (H, W), as device tensors kept alive in `keep`"""
    cx, cy = centre(family)
    if family == "grid_flow":
        g = _dev(prm.grids)
        keep.append(g)
        return [g.data_ptr(), g.shape[-2], g.shape[-1]]
    if family == "depth_grid":
        r, g = _dev(prm.rows), _dev(prm.grids)
        keep += [r, g]
        return [r.data_ptr(), cx, cy, g.data_ptr(), g.shape[-2], g.shape[-1]]
    r = _dev(np.asarray(prm.rows, np.float64))
    keep.append(r)
    return [WARP[family], r.data_ptr(), r.shape[-1], cx, cy]


def _names(family, loss):
    """(forward, gradient, candidates) entry names, without _f32"""
    stem = _stem(family, loss)
    if family == "segmentation":
        return stem, stem + "_grad", stem + "_candidates"
    return stem + "_objective", stem + "_objective_grad", stem + "_candidates"


def _query(name, B, prm, M, J=None):
    js = () if J is None else (J,)
    ms = () if M is None else (M,)
    grid = tuple(prm.grids.shape[-2:]) if prm.grids is not None else ()
    return max(getattr(_L(), name + "_workspace_bytes")(B, *ms, *js, *grid, H, W), 256)


def run(family, loss, st, prm, sigma, g=None):
    """the forward (and with g, the gradient) entry: [f, images..., grad(s)] as numpy, or (rc, f) when refused.  The
    segmentation returns f (B,M), the IWEs (B,M,HC,WC), and the parameter and weight gradients."""
    L = _L()
    B = st.B
    M = st.t["w"].shape[1] if family == "segmentation" else None
    keep = []
    fwd, grd, _ = _names(family, loss)
    ws = torch.empty(_query(fwd, B, prm, M), dtype=torch.uint8, device="cuda")
    fshape = (B, M) if M else (B,)
    f = torch.full(fshape, float("nan"), dtype=torch.float64, device="cuda")
    cnt = B * (M or 1)
    imgs = [torch.empty((cnt, HC, WC), device="cuda")] if loss == "contrast" else \
        [torch.empty((cnt, 2, HC, WC), device="cuda") for _ in range(2)]
    sc = [sigma, 0, 0.0] if loss == "contrast" else [sigma]
    args = _front(family, loss, st) + _model_args(family, prm, keep) + [H, W] + sc
    rc = getattr(L, fwd + "_f32")(*args, f.data_ptr(), *[i.data_ptr() for i in imgs], ws.data_ptr(), ws.numel(), None)
    if rc:
        return rc, f
    out = [np_(f)] + [np_(i).reshape(fshape + i.shape[1:]) for i in imgs]
    if g is None:
        return out
    gf = _dev(np.asarray(g, np.float32))
    if family in ("grid_flow", "depth_grid"):
        grad = torch.full(prm.grids.shape, float("nan"), device="cuda")
    else:
        grad = torch.full(np.shape(prm.rows), float("nan"), dtype=torch.float64, device="cuda")
    extra = []
    if M:
        gw = torch.zeros((st.n, M), device="cuda")
        extra = [gw.data_ptr()]
    _check(getattr(L, grd + "_f32")(*args, *[i.data_ptr() for i in imgs], gf.data_ptr(), grad.data_ptr(), *extra,
                                      ws.data_ptr(), ws.numel(), None))
    out.append(np_(grad))
    if M:
        out.append(np_(gw))
    return out


def run_candidates(family, loss, st, prm, cand, sigma):
    """the candidates entry: (rc, f (B,J) or (B,M,J)).  cand: (B,J,K) rows, (B,M,J,K) for the segmentation, or (B,J,...)
    node grids; prm gives the depth grid's motion rows"""
    L = _L()
    B = st.B
    M = st.t["w"].shape[1] if family == "segmentation" else None
    J = cand.shape[2] if M else cand.shape[1]
    c = _dev(np.ascontiguousarray(cand, np.float32 if family in ("grid_flow", "depth_grid") else np.float64))
    gp = Params(family, rows=prm.rows, grids=np.asarray(cand)[:, 0] if family in ("grid_flow", "depth_grid") else None)
    name = _names(family, loss)[2]
    ws = torch.empty(_query(name, B, gp, M, J), dtype=torch.uint8, device="cuda")
    f = torch.full((B, M, J) if M else (B, J), float("nan"), dtype=torch.float64, device="cuda")
    cx, cy = centre(family)
    keep = []
    if family == "grid_flow":
        model = [c.data_ptr(), J, cand.shape[-2], cand.shape[-1]]
    elif family == "depth_grid":
        r = _dev(prm.rows)
        keep.append(r)
        model = [r.data_ptr(), cx, cy, c.data_ptr(), J, cand.shape[-2], cand.shape[-1]]
    else:
        model = [WARP[family], c.data_ptr(), J, cand.shape[-1], cx, cy]
    sc = [sigma, 0, 0.0] if loss == "contrast" else [sigma]
    rc = getattr(L, name + "_f32")(*_front(family, loss, st), *model, H, W, *sc, f.data_ptr(), ws.data_ptr(), ws.numel(),
                                    None)
    return rc, f


# ---- host images and f64 references ----------------------------------------------------------------------------------
def host_images(family, loss, s, vel):
    """the exact variant's f64 images and f: vel (B,2) ((B,M,2) for the segmentation) are the linvel velocities"""
    flow = family == "grid_flow"
    if family == "segmentation":
        M = vel.shape[1]
        iwe = np.stack([S.linvel_iwe(s, vel[:, m], weight=s["w"][:, m]) for m in range(M)], axis=1)
        return np.stack([S.variance_f(iwe[:, m]) for m in range(M)], axis=1), [iwe]
    if loss == "contrast":
        iwe = S.linvel_iwe(s, vel, flow)
        return S.variance_f(iwe), [iwe]
    Si, Ci = S.linvel_ts_images(s, vel, flow)
    f, T = S.timestamp_f(Si, Ci)
    return f, [T, Ci]


def reference(family, loss, sub, prm, sigma, g):
    """f64 f and gradient of the windows of `sub` and the bound's (M, c, E) (segmentation: also the weight gradient's),
    as MB.check takes them; cast: whether the kernel rounds the gradient from f64 to f32"""
    x, y, d, tau, p, off = (sub[k] for k in ("x", "y", "d", "tau", "p", "off"))
    rho = sub["r"]
    c = centre(family)
    gt = torch.from_numpy(np.asarray(g, np.float64))
    if family in ("grid_flow", "depth_grid"):
        n64 = torch.tensor(prm.grids.astype(np.float64), requires_grad=True)
        if family == "grid_flow":
            out = GR.reference(x, y, d, p, off, n64, H, W, sigma, "variance") if loss == "contrast" else \
                GTR.reference(x, y, d, tau, p, off, n64, H, W, sigma)
        else:
            mot = prm.rows[:, :6]
            intr = (S.FOCAL, S.FOCAL) + c
            out = DR.contrast(x, y, d, p, off, n64, mot, intr, sigma, "variance", img_size=(H, W)) if loss == "contrast" \
                else DTR.reference(x, y, d, tau, p, off, n64, mot, intr, sigma, img_size=(H, W))
        (out[0] * gt).sum().backward()
        imgs = [a.detach().numpy() for a in out[1:]]
        im = imgs[0] if loss == "contrast" else tuple(imgs)
        tau_ = None if loss == "contrast" else tau
        if family == "grid_flow":
            bnd = MB.grid_flow_bound(loss, x, y, d, p, off, prm.grids, H, W, sigma, g, im, tau=tau_)
        else:
            bnd = MB.depth_grid_bound(loss, x, y, d, p, off, prm.grids, prm.rows[:, :6], intr, sigma, g, im, (H, W),
                                      tau=tau_)
        return out[0].detach().numpy(), n64.grad.numpy(), bnd
    p64 = torch.tensor(np.asarray(prm.rows, np.float64), requires_grad=True)
    if family == "segmentation":
        w64 = torch.tensor(sub["w"].astype(np.float64), requires_grad=True)
        fr, iwe = P.segmentation("affine", x, y, d, p, w64, off, p64, sigma, "variance", 3.0, (H, W), c)
        (fr * gt).sum().backward()
        bnd = MB.segmentation_bound("affine", x, y, d, p, sub["w"], off, prm.rows, sigma, g, iwe.detach().numpy(), c, (H, W))
        return fr.detach().numpy(), (p64.grad.numpy(), w64.grad.numpy()), bnd
    if family in ("affine", "homography"):
        out = P.contrast(family, x, y, d, p, off, p64, sigma, "variance", 3.0, (H, W), c) if loss == "contrast" else \
            P.timestamp(family, x, y, d, tau, p, off, p64, sigma, (H, W), c)
    elif family == "camera_rotation":
        out = CR.contrast(x, y, d, p, off, p64, sigma, "variance", c, img_size=(H, W)) if loss == "contrast" else \
            CR.timestamp(x, y, d, tau, p, off, p64, sigma, c, img_size=(H, W))
    else:
        out = CM.contrast(x, y, d, p, rho, off, p64, sigma, "variance", c, img_size=(H, W)) if loss == "contrast" else \
            CM.timestamp(x, y, d, tau, p, rho, off, p64, sigma, c, img_size=(H, W))
    (out[0] * gt).sum().backward()
    r = rho if family == "camera_motion" else None
    imgs = [a.detach().numpy() for a in out[1:3]]
    if loss == "contrast":
        bnd = MB.param_contrast_bound(family, x, y, d, p, off, prm.rows, sigma, "variance", 3.0, g, imgs[0], c, (H, W), r)
    else:
        bnd = MB.param_timestamp_bound(family, x, y, d, tau, p, off, prm.rows, sigma, g, imgs[0], imgs[1], c, (H, W), r)
    return out[0].detach().numpy(), p64.grad.numpy(), bnd


def check_gradients(family, loss, f, grads, ref, what):
    """f to 1e-5 and every gradient component within its bound"""
    fr, gr, bnd = ref
    np.testing.assert_allclose(f, fr, rtol=1e-5, atol=1e-12, err_msg=what)
    if family == "segmentation":
        M, c, E, Mw, cw, Ew = bnd
        MB.check(grads[0], gr[0], M, c, E, what + " parameters")
        MB.check(grads[1], gr[1], Mw, cw, Ew, what + " weights", cast=True)
    else:
        MB.check(grads, gr, *bnd, what, cast=family in ("grid_flow", "depth_grid"))


def _drop(loss):
    return 0.0 if loss == "contrast" else np.nan


def _rtol(b, giant):
    return 1e-5 if b == giant else 1e-6


CASES = [(fam, loss) for fam in ("affine", "homography", "camera_rotation", "camera_motion", "grid_flow", "depth_grid")
         for loss in ("contrast", "timestamp")] + [("segmentation", M) for M in (2, 3, 4)]


def _case(family, loss):
    """(loss, M, cap) of a CASES entry: the segmentation's 'loss' is its M"""
    if family == "segmentation":
        return "contrast", loss, MOTION_CAP // loss
    return loss, None, MOTION_CAP if loss == "contrast" else TS_CAP


def _grad_of(out, M):
    return (out[-2], out[-1]) if M else out[-1]


def _take_grad(grads, M, idx, sub_off, full_off):
    """the gradient rows of the windows idx (the segmentation's weight gradient: their events' rows)"""
    if not M:
        return grads[idx]
    ev = np.concatenate([np.arange(full_off[b], full_off[b + 1]) for b in idx])
    return grads[0][idx], grads[1][ev]


# ---- 1. the entries at their caps ------------------------------------------------------------------------------------
@pytest.mark.parametrize("variant", ["exact", "random"])
@pytest.mark.parametrize("family,loss", CASES)
def test_entry_at_its_cap(family, loss, variant):
    loss, M, cap = _case(family, loss)
    exact = variant == "exact"
    if exact and family not in S.EXACT_FAMILIES:
        pytest.skip("the camera rotation has no exact embedding of the linvel warp")
    giant = GIANT_AT.get(cap, cap // 2)
    seed = 1000 + 10 * CASES.index((family, loss if M is None else M)) + exact
    s = make_stream(exact, cap, giant, seed, M)
    sigma = 0.0 if exact else 1.0
    if exact:
        prm, vel = exact_params(family, cap, seed, seed + 1, M)
    else:
        prm = random_params(family, cap, seed + 1, M)
    idx = S.sampled_windows(s["sizes"], giant, M or (1 if loss == "contrast" else 2), seed=seed)
    checked = idx[idx != giant]
    if not exact:
        S.drop_unsafe(s, family, checked, prm.of, _drop(loss))
    nonempty = np.flatnonzero(s["sizes"][checked] > 1)
    zero = int(checked[nonempty[0]])
    g = incoming((cap,) if M is None else (cap, M), seed + 2, zero_in=zero)
    st = Stream(s)
    out = run(family, loss, st, prm, sigma, g)
    f, grads = out[0], _grad_of(out, M)
    assert np.isfinite(f).all()
    empty = s["sizes"] == 0
    gmain = grads[0] if M else grads
    assert (f[empty] == 0).all() and (gmain[empty] == 0).all() and (gmain[zero] == 0).all()
    what = "%s %s %s" % (family, loss if M is None else "M=%d" % M, variant)
    if exact:
        fh, imgs = host_images(family, loss, s, vel)
        for a, b in zip(out[1:1 + len(imgs)], imgs):
            assert np.array_equal(a, b.astype(np.float32)), what
        if loss == "contrast":
            assert np.array_equal(f, fh), what
        else:
            np.testing.assert_allclose(f, fh, rtol=1e-13, atol=0, err_msg=what)
    # window order: the same windows reversed give the same f
    r = S.reversed_stream(s)
    fr = run(family, loss, Stream(r), prm.reversed(), sigma)[0][::-1]
    if exact:
        np.testing.assert_allclose(fr, f, rtol=0 if loss == "contrast" else 1e-13, atol=0, err_msg=what)
    else:
        rest = np.arange(cap) != giant
        np.testing.assert_allclose(fr[rest], f[rest], rtol=1e-6, atol=0, err_msg=what)
        np.testing.assert_allclose(fr[giant], f[giant], rtol=1e-5, atol=0, err_msg=what)
    # the sampled windows alone
    for b in idx:
        one = run(family, loss, st.window(b), prm.take([b]), sigma)
        if exact:
            for a, c in zip(one[1:], out[1:]):
                assert np.array_equal(a[0], c[b]), (what, b)
            assert np.allclose(one[0][0], f[b], rtol=0 if loss == "contrast" else 1e-13, atol=0), (what, b)
        else:
            assert np.all(np.abs(one[0][0] - f[b]) <= _rtol(b, giant) * np.abs(f[b])), (what, b, one[0][0], f[b])
    # the f64 reference and the gradients' bounds on the sampled windows but the giant
    sub = st.select(checked)
    ref = reference(family, loss, sub, prm.take(checked), sigma, g[checked])
    check_gradients(family, loss, f[checked], _take_grad(grads, M, checked, sub["off"], s["off"]), ref, what)
    # cap + 1 windows are refused before any launch: f stays NaN
    big = Stream(st.select(np.concatenate((np.arange(cap), [1]))))
    rc, f2 = run(family, loss, big, prm.take(np.concatenate((np.arange(cap), [1]))), sigma)
    assert rc == E_ARG and torch.isnan(f2).all(), what


# ---- 2. the giant window first, in the middle and last -------------------------------------------------------------
@pytest.mark.parametrize("family,loss", CASES)
def test_giant_window_in_a_batch_equals_it_alone(family, loss):
    """4095 windows (1365 with M models): the giant window at 0, B // 2 and B - 1 runs on one CTA of the batch and on
    hundreds alone; its images (exact variant: bit for bit), f and gradient agree, and the gradient meets its bound
    both ways.  The node gradients meet in f64 atomics in a different order in the two layouts."""
    loss, M, _ = _case(family, loss)
    exact = family in S.EXACT_FAMILIES
    B = 4095 // (M or 1)
    seed = 2000 + 10 * CASES.index((family, loss if M is None else M))
    sigma = 0.0 if exact else 1.0
    ref = first = None
    for giant in (0, B // 2, B - 1):
        s = make_stream(exact, B, giant, seed, M)
        prm = exact_params(family, B, seed, seed + 1, M)[0] if exact else random_params(family, B, seed + 1, M)
        g = incoming((B,) if M is None else (B, M), seed + 2)
        sl = slice(s["off"][giant], s["off"][giant + 1])
        if first is None:
            first = prm.take([giant]), g[giant].copy(), {k: s[k][sl].copy() for k in EVENT_KEYS if k in s}
        for k, v in first[2].items():
            s[k][sl] = v
        # the giant window keeps its parameters and incoming gradient wherever it sits
        for a, v in ((prm.rows, first[0].rows), (prm.grids, first[0].grids)):
            if a is not None:
                a[giant] = v[0]
        g[giant] = first[1]
        if not exact:
            S.drop_unsafe(s, family, [giant], prm.of, _drop(loss))
        st = Stream(s)
        out = run(family, loss, st, prm, sigma, g)
        one = run(family, loss, st.window(giant), prm.take([giant]), sigma, g[giant:giant + 1])
        nimg = 1 if loss == "contrast" else 2
        for a, c in zip(one[1:1 + nimg], out[1:1 + nimg]):
            if exact:
                assert np.array_equal(a[0], c[giant]), giant
            else:
                np.testing.assert_allclose(a[0], c[giant], rtol=1e-5, atol=1e-5 * np.abs(c[giant]).max())
        tol = 0 if exact and loss == "contrast" else 1e-13 if exact else 1e-5
        assert np.all(np.abs(one[0][0] - out[0][giant]) <= tol * np.abs(out[0][giant])), giant
        sub = st.select([giant])
        if ref is None:                      # the giant window's events and parameters are the same at every position
            ref = reference(family, loss, sub, prm.take([giant]), sigma, g[giant:giant + 1])
        what = "%s %s giant at %d" % (family, loss if M is None else M, giant)
        gb = _take_grad(_grad_of(out, M), M, [giant], sub["off"], s["off"])
        check_gradients(family, loss, out[0][giant:giant + 1], gb, ref, what + " batched")
        check_gradients(family, loss, one[0], _grad_of(one, M), ref, what + " alone")
        if family in ("grid_flow", "depth_grid"):
            # Both layouts form the same f32 term per warp of 32 consecutive events (warps start at first + 32 k), so
            # they differ only in the order of the f64 sums (per CTA, then across CTAs) and in the final f32 cast: far
            # tighter than the rounding bound, whose k_I the giant's busiest pixel makes loose
            Mn = ref[2][0]
            alone = _grad_of(one, M).astype(np.float64)
            err = np.abs(gb.astype(np.float64) - alone)
            assert (err <= 1e-10 * Mn + 2.0 ** -23 * np.abs(alone)).all(), (what, err.max(), np.abs(alone).max())


# ---- 3. the candidates passes ----------------------------------------------------------------------------------------
def _jmax(family, M):
    return 32 // M if M else 32


def _exact_candidates(family, stream_seed, B, J, seed, M=None):
    """(cand, vel): J exact-embedding candidates per window (and model)"""
    vel = S.exact_velocity_set((B, J) if M is None else (B, M, J), seed)
    if family in ("affine", "homography", "segmentation"):
        return S.exact_rows(family, vel), vel
    if family == "grid_flow":
        return np.stack([S.exact_rows(family, vel[:, j]) for j in range(J)], axis=1), vel
    rho = S.window_rhos(B, stream_seed)
    return np.stack([S.exact_rows(family, vel[:, j], rho) for j in range(J)], axis=1), vel


CAND_CASES = [(fam, loss) for fam in ("affine", "homography", "camera_motion", "grid_flow") for loss in ("contrast", "timestamp")] \
    + [("segmentation", M) for M in (2, 3, 4)]


@pytest.mark.parametrize("family,loss", CAND_CASES)
def test_candidates_entry_at_its_cap(family, loss):
    """(cap, 1) and (cap // J, J) with J at the pass maximum on the exact variant: every f[b, j] equals the forward entry
    at candidate j and the host's exact value; one window more is refused.  The windows are the skewed small ones without
    the giant (the giant-window tests cover it), so that the host images of every candidate stay cheap."""
    loss, M, cap = _case(family, loss)
    seed = 3000 + 10 * CAND_CASES.index((family, loss if M is None else M))
    for J in (1, _jmax(family, M)):
        B = cap // J
        s = make_stream(True, B, None, seed + J, M)
        st = Stream(s)
        cand, vel = _exact_candidates(family, seed + J, B, J, seed + J + 1, M)
        rc, f = run_candidates(family, loss, st, Params(family), cand, 0.0)
        _check(rc)
        f = np_(f)
        for j in range(J):
            cj = cand[:, :, j] if M else cand[:, j]
            prm = Params(family, grids=np.ascontiguousarray(cj)) if family == "grid_flow" else Params(family, rows=cj)
            fw = run(family, loss, st, prm, 0.0)[0]
            vj = vel[:, :, j] if M else vel[:, j]
            fh = host_images(family, loss, s, vj)[0]
            got = f[:, :, j] if M else f[:, j]
            tol = 0 if loss == "contrast" else 1e-13
            np.testing.assert_allclose(got, fw, rtol=tol, atol=0, err_msg="%s J=%d j=%d forward" % (family, J, j))
            np.testing.assert_allclose(got, fh, rtol=tol, atol=0, err_msg="%s J=%d j=%d host" % (family, J, j))
        more = np.concatenate((np.arange(B), [0]))
        rc, f2 = run_candidates(family, loss, Stream(st.select(more)), Params(family), cand[more], 0.0)
        assert rc == E_ARG and torch.isnan(f2).all()


@pytest.mark.parametrize("loss", ["contrast", "timestamp"])
def test_depth_grid_candidates_entry_at_its_cap(loss):
    """the depth grid's candidates at (cap, 1) and (cap // 32, 32): each window has its own camera-motion rows, each
    candidate a uniform grid of one of the exact rhos; f[b, j] equals the forward at that grid and the host's exact
    value of the linvel velocity the rows and that rho give (rows built for rho 1 and nodes of rho 1 or 2:
    tests/test_batch_limits_models_cpu.py proves this embedding exact)"""
    cap = MOTION_CAP if loss == "contrast" else TS_CAP
    for J in (1, 32):
        B = cap // J
        s = make_stream(True, B, None, 3500 + J)
        st = Stream(s)
        rng = np.random.default_rng(3600 + J)
        # rows of rho 1: v = -vel / FOCAL; candidate rho r moves the events by r times that velocity
        vel = S.exact_velocity_set((B,), 3700 + J)
        rows = S.exact_rows("camera_motion", vel, np.ones(B))
        rhos = rng.choice(S.DEPTH_CANDIDATE_RHOS, (B, J))
        cand = np.broadcast_to(rhos[:, :, None, None], (B, J, H, W)).astype(np.float32)
        rc, f = run_candidates("depth_grid", loss, st, Params("depth_grid", rows=rows), cand, 0.0)
        _check(rc)
        f = np_(f)
        for j in range(J):
            fw = run("depth_grid", loss, st, Params("depth_grid", rows=rows, grids=np.ascontiguousarray(cand[:, j])), 0.0)[0]
            fh = host_images("depth_grid", loss, s, vel * rhos[:, j, None])[0]
            tol = 0 if loss == "contrast" else 1e-13
            np.testing.assert_allclose(f[:, j], fw, rtol=tol, atol=0, err_msg="J=%d j=%d forward" % (J, j))
            np.testing.assert_allclose(f[:, j], fh, rtol=tol, atol=0, err_msg="J=%d j=%d host" % (J, j))
        more = np.concatenate((np.arange(B), [0]))
        rc, f2 = run_candidates("depth_grid", loss, Stream(st.select(more)), Params("depth_grid", rows=rows[more]),
                                cand[more], 0.0)
        assert rc == E_ARG and torch.isnan(f2).all()


@pytest.mark.parametrize("loss", ["contrast", "timestamp"])
def test_camera_rotation_candidates_entry_at_its_cap(loss):
    """the random variant: (cap, 1) and (cap // 32, 32) equal the per-candidate forward entry to 1e-6"""
    cap = MOTION_CAP if loss == "contrast" else TS_CAP
    for J in (1, 32):
        B = cap // J
        s = make_stream(False, B, None, 3800 + J)
        st = Stream(s)
        cand = np.stack([S.random_rows("camera_rotation", B, 3900 + J + j) for j in range(J)], axis=1)
        rc, f = run_candidates("camera_rotation", loss, st, Params("camera_rotation"), cand, 1.0)
        _check(rc)
        f = np_(f)
        for j in range(J):
            fw = run("camera_rotation", loss, st, Params("camera_rotation", rows=cand[:, j].copy()), 1.0)[0]
            bad = np.abs(f[:, j] - fw) > 1e-6 * np.abs(fw)
            assert not bad.any(), (J, j, np.flatnonzero(bad)[:5])


# ---- the torch candidates functions across window chunks and candidate passes ---------------------------------------
TORCH_B = {"contrast": 4095, "timestamp": 2047, 2: 4095, 3: 4369, 4: 4095}
SPREAD = {"affine": [4, 4, 0.5, 0.5, 0.5, 0.5], "homography": [4, 4, 0.5, 0.5, 0.5, 0.5, 0.05, 0.05],
          "camera_rotation": [0.5, 0.5, 0.5, 0, 0], "camera_motion": [0.5, 0.5, 0.5, 0.4, 0.4, 0.4, 0, 0],
          "segmentation": [4, 4, 0.5, 0.5, 0.5, 0.5]}


def _warpfunc(family):
    from event_utils_b200.contrast_max import warps
    if family in ("camera_rotation", "camera_motion", "depth_grid"):
        return (warps.camera_rotation_warp if family == "camera_rotation" else warps.camera_motion_warp)(S.INTR)
    return {"affine": warps.affine_warp, "homography": warps.homography_warp,
            "segmentation": warps.affine_warp}[family](center=S.CENTRE)


def torch_loss(family, loss, st, prm, sigma, kind="objective", t0=0.0):
    """the torch loss (kind "objective") or candidates function ("candidates", prm.rows / prm.grids (B,J,...)) at t0 = 0:
    numpy f.  The timestamp functions normalise the stamps themselves."""
    import event_utils_b200.contrast_max as C
    t = st.t
    ev = (t["x"], t["y"], t["d"], t["p"])
    ends = t["off"][1:]
    kw = dict(t0=t0, blur_sigma=sigma, batch_end_indices=ends)
    if loss == "contrast":
        kw["objective"] = "variance"
    if family == "grid_flow":
        fn = getattr(C, "grid_flow_%s_%s_torch" % ("contrast" if loss == "contrast" else "timestamp", kind))
        return np_(fn(*ev, _dev(prm.grids), (H, W), **kw))
    if family == "depth_grid":
        fn = getattr(C, "depth_grid_%s_%s_torch" % ("contrast" if loss == "contrast" else "timestamp", kind))
        return np_(fn(*ev, _dev(prm.grids), _dev(prm.rows[:, :6]), _warpfunc(family), (H, W), **kw))
    K = {"camera_rotation": 3, "camera_motion": 6}.get(family)
    rows = _dev(np.ascontiguousarray(prm.rows[..., :K]))
    if family == "segmentation":
        fn = C.motion_segmentation_candidates_torch if kind == "candidates" else C.motion_segmentation_objective_torch
        args = (rows, t["w"]) if kind == "candidates" else (t["w"], rows)
        return np_(fn(*ev, *args, _warpfunc(family), img_size=(H, W), **kw))
    kw["img_size"] = (H, W)
    if family == "camera_motion":
        kw["inv_depth"] = t["r"]
    name = "motion_%s_%s_torch" % ("contrast" if loss == "contrast" else "timestamp", kind)
    return np_(getattr(C, name)(*ev, rows, _warpfunc(family), **kw))


def distinct_candidates(family, B, J, seed, M=None):
    """J candidates per window (and model) sharing no component (candidate_checks.distinct_sets around the random
    variant's parameters)"""
    rng = np.random.default_rng(seed)
    base = random_params(family, B * (M or 1), seed + 1)
    if family in ("grid_flow", "depth_grid"):
        # node k of candidate j: base_k (0.8 + 0.4 j / J), distinct in f32 for every non-zero node
        g = base.grids.reshape(B, 1, -1).astype(np.float64)
        c = (g * (0.8 + 0.4 * np.arange(J) / J)[None, :, None]).reshape((B, J) + base.grids.shape[1:]).astype(np.float32)
        return Params(family, rows=base.rows, grids=c)
    c = CC.distinct_sets(base.rows, J, rng, SPREAD[family])
    if family.startswith("camera"):
        c[..., -2:] = S.FOCAL                         # the torch functions take the focal lengths from the warp
    if M:
        c = c.reshape(B, M, J, -1)
    return Params(family, rows=c)


@pytest.mark.parametrize("family,loss", CASES)
def test_candidates_function_across_window_chunks_and_passes(family, loss):
    """J = 70 distinct candidates at the B of tests/test_batch_limits_models_cpu.CANDIDATE_CASES: three window chunks
    (the last of one window) and at least three candidate passes.  Every f[b, j] equals the torch loss at candidate j
    (to 1e-6), and on the sampled windows the f64 reference"""
    loss, M, _ = _case(family, loss)
    B = TORCH_B[M or loss]
    J = 70
    seed = 4000 + 10 * CASES.index((family, loss if M is None else M))
    s = make_stream(False, B, None, seed, M)
    cand = distinct_candidates(family, B, J, seed + 1, M)
    CC.assert_distinct(cand.grids.reshape(B, J, -1) if cand.grids is not None else
                       cand.rows[..., :-2] if family.startswith("camera") else cand.rows)
    idx = S.sampled_windows(s["sizes"], B // 2, 1, seed=seed, count=16)

    def cand_j(j):
        if cand.grids is not None:
            return Params(family, rows=cand.rows, grids=np.ascontiguousarray(cand.grids[:, j]))
        return Params(family, rows=np.ascontiguousarray(cand.rows[:, :, j] if M else cand.rows[:, j]))
    S.drop_unsafe(s, family, idx, lambda b: [q for j in range(J) for q in cand_j(j).of(b)], _drop(loss))
    st = Stream(s)
    sigma = 1.0
    f = torch_loss(family, loss, st, cand, sigma, "candidates")
    sub = st.select(idx)
    if loss == "timestamp":
        sub["tau"] = P.tau_f32(sub["d"], sub["off"])      # the stamps the torch functions form, from t = d and t0 = 0
    for j in range(J):
        fj = f[:, :, j] if M else f[:, j]
        fw = torch_loss(family, loss, st, cand_j(j), sigma)
        np.testing.assert_allclose(fj, fw, rtol=1e-6, atol=1e-12, err_msg="%s %s j=%d" % (family, loss, j))
        if j in (0, 31, 32, 69):
            pj = cand_j(j).take(idx)
            g = np.ones((len(idx),) if M is None else (len(idx), M))
            fr = reference(family, loss, sub, pj, sigma, g)[0]
            np.testing.assert_allclose(fj[idx], fr, rtol=1e-5, atol=1e-12, err_msg="%s %s j=%d f64" % (family, loss, j))


@pytest.mark.parametrize("loss", ["contrast", "timestamp"])
def test_grid_flow_nan_candidate_flags_only_itself(loss):
    """a full 32-candidate pass in which candidate 0 of one window and candidate 31 of another (bits 0 and 31 of the
    per-candidate nonfinite mask) are grids of NaN nodes, which every event of their windows reads: those two f are NaN,
    every other equals the pass without them"""
    B, J = 64, 32
    s = make_stream(False, B, None, 5000)
    st = Stream(s)
    cand = S.random_rows("grid_flow", B * J, 5001).reshape(B, J, 2, *S.RANDOM_GRID)
    _, f0 = run_candidates("grid_flow", loss, st, Params("grid_flow"), cand, 1.0)
    busy = np.flatnonzero(s["sizes"] >= 2)
    cells = ((int(busy[0]), 0), (int(busy[1]), 31))
    bad = cand.copy()
    for b, j in cells:
        bad[b, j] = np.nan
    _, f1 = run_candidates("grid_flow", loss, st, Params("grid_flow"), bad, 1.0)
    f0, f1 = np_(f0), np_(f1)
    assert np.isfinite(f0).all()
    nan = np.zeros((B, J), bool)
    for b, j in cells:
        nan[b, j] = True
    assert np.isnan(f1[nan]).all(), f1[nan]
    assert np.array_equal(f1[~nan], f0[~nan])


@pytest.mark.parametrize("loss", ["contrast", "timestamp"])
def test_depth_grid_nan_node_is_no_event(loss):
    """a NaN node drops the events that read it: a grid of NaN nodes gives the no-event value, not NaN, and leaves the
    other candidates and windows alone"""
    B, J = 64, 32
    s = make_stream(False, B, None, 5100)
    st = Stream(s)
    prm = random_params("depth_grid", B, 5101)
    cand = np.broadcast_to(prm.grids[:, None], (B, J) + prm.grids.shape[1:]).copy()
    cand *= np.linspace(0.5, 1.5, J, dtype=np.float32)[None, :, None, None]
    _, f0 = run_candidates("depth_grid", loss, st, prm, cand, 1.0)
    bad = cand.copy()
    bad[3, 31] = np.nan
    _, f1 = run_candidates("depth_grid", loss, st, prm, bad, 1.0)
    f0, f1 = np_(f0), np_(f1)
    assert f1[3, 31] == CC.no_event_value("variance" if loss == "contrast" else None, H, W)
    keep = np.ones((B, J), bool)
    keep[3, 31] = False
    assert np.array_equal(f1[keep], f0[keep])


# ---- 4. the fits past the entry caps ---------------------------------------------------------------------------------
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


def _ceil(a, b):
    return -(-a // b)


def _fit(family, loss, st, M, max_iter):
    """fn() running one short fit from a fixed start on every window, with every input built on the GPU beforehand"""
    import event_utils_b200.contrast_max as C
    t = st.t
    ev = (t["x"], t["y"], t["d"], t["p"])
    B = st.B
    # t0 None: each window's last stamp, read on the device (a host t0 would be copied with a synchronisation)
    kw = dict(batch_end_indices=t["off"][1:], t0=None, blur_sigma=1.0, max_iter=max_iter)
    if family == "grid_flow":
        x0 = torch.full((B, 2, 2, 2), 0.0, dtype=torch.float64, device="cuda")
        x0[:, 0] = -4.0
        fn = C.grid_flow_fit_torch if loss == "contrast" else C.grid_flow_timestamp_fit_torch
        scale = torch.ones((), dtype=torch.float64, device="cuda")
        return lambda: fn(*ev, (H, W), grid_shapes=((2, 2),), x0=x0, param_scale=scale, **kw)
    if family == "depth_grid":
        # every window its own camera motion, so that a chunk reading another chunk's rows (_lead) shows
        st.motion = S.random_rows("depth_grid", B, 6500)[0]
        mot = _dev(st.motion[:, :6])
        rng_ = torch.tensor([0.1, 2.0], dtype=torch.float64, device="cuda").expand(B, 2).contiguous()
        x0 = torch.full((B, 2, 2), 0.5, dtype=torch.float64, device="cuda")
        fn = C.depth_grid_fit_torch if loss == "contrast" else C.depth_grid_timestamp_fit_torch
        return lambda: fn(*ev, mot, _warpfunc(family), (H, W), rng_, grid_shapes=((2, 2),), x0=x0, **kw)
    if family == "segmentation":
        x0 = torch.zeros((B, M, 6), dtype=torch.float64, device="cuda")
        x0[:, :, 0] = torch.linspace(-20, 20, M, dtype=torch.float64, device="cuda")
        kw.pop("max_iter")
        return lambda: C.motion_segmentation_fit_torch(*ev, _warpfunc(family), x0, img_size=(H, W), em_iters=1, max_iter=max_iter,
                                               **kw)
    K = {"affine": 6, "homography": 8, "camera_rotation": 3, "camera_motion": 6}[family]
    x0 = torch.zeros((B, K), dtype=torch.float64, device="cuda")
    x0[:, 0] = 0.5
    extra = {"inv_depth": t["r"]} if family == "camera_motion" else {}
    fn = C.motion_contrast_fit_torch if loss == "contrast" else C.motion_timestamp_fit_torch
    if loss == "contrast":
        kw["objective"] = "variance"
    else:
        box = torch.tensor([[-30.0, 30.0]], dtype=torch.float64, device="cuda").expand(K, 2).contiguous()
        kw["bounds"] = box
    scale = torch.full((K,), 0.5, dtype=torch.float64, device="cuda")
    return lambda: fn(*ev, _warpfunc(family), img_size=(H, W), x0=x0, param_scale=scale, **extra, **kw)


def _fit_f_at(family, loss, whole, fit, M, cap):
    """the loss at the fit's result, in calls of at most `cap` windows: (got, want)"""
    s = whole.s
    B = whole.B
    got, want = [], []
    for b0 in range(0, B, cap):
        idx = np.arange(b0, min(B, b0 + cap))
        sub = whole.select(idx)
        if family == "segmentation":
            ev = np.concatenate([np.arange(s["off"][b], s["off"][b + 1]) for b in idx])
            sub["w"] = np_(fit.weights)[ev]
            prm = Params(family, rows=np_(fit.params)[idx])
            got.append(np_(fit.f)[idx])
        elif family == "grid_flow":
            prm = Params(family, grids=np_(fit.flow)[idx].astype(np.float32))
            got.append(np_(fit.contrast if loss == "contrast" else fit.loss)[idx])
        elif family == "depth_grid":
            prm = Params(family, rows=whole.motion[idx], grids=np_(fit.inv_depth)[idx].astype(np.float32))
            got.append(np_(fit.contrast if loss == "contrast" else fit.loss)[idx])
        else:
            prm = Params(family, rows=np_(fit.params)[idx])
            got.append(np_(fit.f)[idx])
        want.append(torch_loss(family, loss, Stream(sub), prm, 1.0, t0=None))
    return np.concatenate(got), np.concatenate(want)


FIT_CASES = [(fam, loss) for fam in ("affine", "homography", "camera_rotation", "camera_motion", "grid_flow", "depth_grid")
             for loss in ("contrast", "timestamp")] + [("segmentation", M) for M in (2, 3, 4)]


@pytest.mark.parametrize("family,loss", FIT_CASES)
def test_short_fit_past_the_entry_cap(family, loss):
    """cap + 1 windows (65536 contrast, 32768 timestamp, 65535 // M + 1 segmentation), max_iter 2 and one grid level:
    no host synchronisation, and every window's f is the loss at the returned parameters.  The launches follow the
    chunk counts: a forward/gradient class of cap windows per call and a line-search class of cap // (M jc) windows per
    call, each class's launches measured at one window and at one window past the line search's chunk"""
    loss, M, cap = _case(family, loss)
    cap_f = cap
    jc = min(8, 32 // (M or 1))
    cap_c = (MOTION_CAP if loss == "contrast" else TS_CAP) // ((M or 1) * jc)
    max_iter = 2
    counts = {}
    for B in (1, cap_c + 1, cap_f + 1):
        s = make_stream(False, B, None, 6000 + B, M)
        st = Stream(s)
        run_fit = _fit(family, loss, st, M, max_iter)
        run_fit()                                                 # warm-up: scratch buffers
        fit, counts[B] = _launches(run_fit)
    n1, n3, n2 = counts[1], counts[cap_c + 1], counts[cap_f + 1]
    per_c, per_f = n3 - n1, 2 * n1 - n3
    assert per_c > 0 and per_f > 0, counts
    B = cap_f + 1
    assert n2 == per_f * _ceil(B, cap_f) + per_c * _ceil(B, cap_c), (counts, per_f, per_c)
    got, want = _fit_f_at(family, loss, st, fit, M, cap)
    assert np.isfinite(got).all()
    np.testing.assert_allclose(got, want, rtol=1e-6, atol=1e-9)
