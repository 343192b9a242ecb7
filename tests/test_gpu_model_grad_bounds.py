"""Every gradient component of the newer families, window by window, against its f64 reference within the rounding
bound of tests/model_grad_bounds.py: the planar models, the camera rotation and the camera motion (all K columns of
the C entries and the first 3 or 6 of the torch losses), the segmentation's parameter and weight gradients, and the
grid-flow and depth-grid node gradients of both losses, on skewed batches and on streams built to stress the
per-node-cell warp reduction.  Each window has its own incoming gradient g_b of mixed sign and magnitude, and one
non-empty window has g_b = 0."""
import zlib

import numpy as np
import pytest
import torch

import camera_motion_reference as CM
import camera_rotation_reference as CR
import depth_grid_reference as DR
import depth_grid_timestamp_reference as DTR
import grid_flow_reference as GR
import grid_flow_timestamp_reference as GTR
import model_grad_bounds as B
import planar_motion_reference as P

pytestmark = pytest.mark.gpu

H, W = 60, 80
CENTRE = (40.0, 30.0)
INTR = (70.3, 64.9, 43.7, 27.2)
ROWS = {"affine": [(20.0, -10.0, 3.0, -2.0, 1.5, -4.0), (-30.0, 15.0, -2.0, 4.0, -3.0, 1.0)],
        "homography": [(20.0, -10.0, 3.0, -2.0, 1.5, -4.0, 0.05, -0.03), (-30.0, 15.0, -2.0, 4.0, -3.0, 1.0, -0.04, 0.06)],
        "camera_rotation": [(2.0, -3.0, 4.0) + INTR[:2], (-2.0, 1.5, -8.0) + INTR[:2]],
        "camera_motion": [(2.0, -3.0, 4.0, 1.0, -0.8, 1.5) + INTR[:2], (-1.5, 1.5, -8.0, -1.5, 0.5, -1.0) + INTR[:2]]}


def _note(what, r):
    """the largest err / bound of one check, printed for the record (pytest -s)"""
    print("err/bound %s %.3e" % (what, r))


def _cuda(*arrays):
    return [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in arrays]


def incoming(rng, B_, zero):
    """g_b of mixed sign and magnitude (f32 values: the C entries take g as f32), zero in window `zero`"""
    g = (rng.standard_normal(B_) * 10.0 ** rng.uniform(-2, 2, B_)).astype(np.float32).astype(np.float64)
    g[zero] = 0.0
    return g


def skewed_sizes(rng):
    """72 windows: one empty, one of a single event, 69 of 33..47 events and one about 64 times the mean"""
    s = list(rng.integers(33, 48, 72))
    s[3], s[10] = 0, 1
    s[40] = 22001
    return s


def _centre(family):
    return INTR[2:] if family.startswith("camera") else CENTRE


def _warp_of(family, rng, x, y, d, rho, row):
    prm = np.asarray(row, np.float64)
    if family in ("affine", "homography"):
        return P.warp_f32(family, x, y, d, prm, CENTRE)
    if family == "camera_rotation":
        return CR.warp(x, y, d, prm[:3], (prm[3], prm[4]) + INTR[2:])
    return CM.warp(x, y, d, rho, prm[:3], prm[3:6], (prm[6], prm[7]) + INTR[2:])


def safe_windows(family, seed, sizes, rows):
    """windows of random events, keeping those whose warp lies 1e-3 px from every integer (or is not kept), so f32 and
    f64 take the same taps; a window keeps its requested length where it can"""
    rng = np.random.default_rng(seed)
    out = [[] for _ in range(6)]
    for b, n in enumerate(sizes):
        got = 0
        while got < n:
            m = 2 * (n - got) + 8
            x = (rng.random(m) * (W - 1)).astype(np.float32)
            y = (rng.random(m) * (H - 1)).astype(np.float32)
            d = (-rng.integers(0, 410, m) / 4096.0).astype(np.float32)
            r = rng.uniform(0.125, 1.0, m).astype(np.float32)
            xw, yw = _warp_of(family, rng, x, y, d, r, rows[b])
            with np.errstate(invalid="ignore"):
                ok = np.isfinite(xw) & np.isfinite(yw) & (np.abs(xw - np.round(xw)) >= 1e-3) & (np.abs(yw - np.round(yw)) >= 1e-3)
            k = np.flatnonzero(ok)[:n - got]
            for o, a in zip(out, (x, y, d, r)):
                o.append(a[k])
            got += k.size
        out[4].append((rng.integers(0, 2, n) * 2 - 1).astype(np.float32))
    x, y, d, r, p = (np.concatenate(o) if o else np.zeros(0, np.float32) for o in out[:5])
    order = [np.argsort(d[lo:hi], kind="stable") + lo for lo, hi in zip(np.cumsum([0] + sizes[:-1]), np.cumsum(sizes))]
    idx = np.concatenate(order).astype(np.int64)
    off = np.concatenate(([0], np.cumsum(sizes))).astype(np.int64)
    return x[idx], y[idx], d[idx], p, r[idx], off


def c_entry(family, loss, events, off, rows, scalars, g):
    """the C forward and gradient entries: f, the images and grad_params (B, K) at grad_f = g"""
    from event_utils_b200 import _lib
    L = _lib.lib()
    Bn = len(off) - 1
    stem = {"contrast": "evk_cmax_motion_objective", "timestamp": "evk_motion_timestamp_objective"}[loss]
    if family == "camera_motion":
        stem = {"contrast": "evk_cmax_motion_depth_objective", "timestamp": "evk_motion_timestamp_depth_objective"}[loss]
    code = {"affine": _lib.WARP_AFFINE, "homography": _lib.WARP_HOMOGRAPHY, "camera_rotation": _lib.WARP_CAMERA_ROTATION,
            "camera_motion": _lib.WARP_CAMERA_MOTION}[family]
    prm = torch.tensor(np.asarray(rows, np.float64), device="cuda")
    outs = [(Bn,), (Bn, H + 1, W + 1)] if loss == "contrast" else [(Bn,), (Bn, 2, H + 1, W + 1), (Bn, 2, H + 1, W + 1)]
    res = [torch.empty(s, dtype=torch.float64 if i == 0 else torch.float32, device="cuda") for i, s in enumerate(outs)]
    ws = torch.empty(getattr(L, stem + "_workspace_bytes")(Bn, H, W), dtype=torch.uint8, device="cuda")
    O = torch.from_numpy(off).cuda()
    c = _centre(family)
    lead = [a.data_ptr() for a in events] + [O.data_ptr(), Bn, events[0].shape[0], code, prm.data_ptr(), prm.shape[-1],
                                             c[0], c[1], H, W]
    _lib.check(getattr(L, stem + "_f32")(*lead, *scalars, *[r.data_ptr() for r in res], ws.data_ptr(), ws.numel(), None))
    gf = torch.from_numpy(np.asarray(g, np.float32)).cuda()
    out = torch.empty(prm.shape, dtype=torch.float64, device="cuda")
    _lib.check(getattr(L, stem + "_grad_f32")(*lead, *scalars, *[r.data_ptr() for r in res[1:]], gf.data_ptr(),
                                               out.data_ptr(), ws.data_ptr(), ws.numel(), None))
    torch.cuda.synchronize()
    return out.cpu().numpy()


def reference(family, loss, x, y, d, tau, p, rho, off, rows, sigma, name, g):
    p64 = torch.tensor(np.asarray(rows, np.float64), requires_grad=True)
    c = _centre(family)
    if family in ("affine", "homography"):
        out = (P.contrast(family, x, y, d, p, off, p64, sigma, name, 3.0, (H, W), c) if loss == "contrast" else
               P.timestamp(family, x, y, d, tau, p, off, p64, sigma, (H, W), c))
    elif family == "camera_rotation":
        out = (CR.contrast(x, y, d, p, off, p64, sigma, name, c, img_size=(H, W)) if loss == "contrast" else
               CR.timestamp(x, y, d, tau, p, off, p64, sigma, c, img_size=(H, W)))
    else:
        out = (CM.contrast(x, y, d, p, rho, off, p64, sigma, name, c, img_size=(H, W)) if loss == "contrast" else
               CM.timestamp(x, y, d, tau, p, rho, off, p64, sigma, c, img_size=(H, W)))
    (out[0] * torch.from_numpy(g)).sum().backward()
    return p64.grad.numpy(), [a.detach().numpy() for a in out[1:]]


def torch_grad(family, loss, x, y, d, p, rho, off, rows, sigma, name, g):
    from event_utils_b200.contrast_max import motion_contrast_objective_torch, motion_timestamp_objective_torch
    from event_utils_b200.contrast_max import warps
    K = {"camera_rotation": 3, "camera_motion": 6}.get(family)
    prm = torch.tensor(np.asarray(rows, np.float64)[:, :K], device="cuda", requires_grad=True)
    if family.startswith("camera"):
        wf = warps.camera_rotation_warp(INTR) if family == "camera_rotation" else warps.camera_motion_warp(INTR)
    else:
        wf = {"affine": warps.affine_warp, "homography": warps.homography_warp}[family](center=CENTRE)
    kw = {"inv_depth": torch.from_numpy(rho).cuda()} if family == "camera_motion" else {}
    ends = torch.from_numpy(off[1:]).cuda()
    if loss == "contrast":
        f = motion_contrast_objective_torch(*_cuda(x, y, d, p), prm, wf, t0=0.0, objective=name, blur_sigma=sigma,
                                            img_size=(H, W), batch_end_indices=ends, **kw)
    else:
        f = motion_timestamp_objective_torch(*_cuda(x, y, d, p), prm, wf, t0=0.0, blur_sigma=sigma, img_size=(H, W),
                                             batch_end_indices=ends, **kw)
    (f * torch.from_numpy(g).cuda()).sum().backward()
    return prm.grad.cpu().numpy()


FAMILIES = ["affine", "homography", "camera_rotation", "camera_motion"]
CASES = [("contrast", "variance", 0.0), ("contrast", "variance", 1.0), ("contrast", "soe", 0.0), ("contrast", "soe", 1.0),
         ("timestamp", None, 0.0), ("timestamp", None, 1.0)]


@pytest.mark.parametrize("loss,name,sigma", CASES)
@pytest.mark.parametrize("family", FAMILIES)
def test_parametric_gradients_on_a_skewed_batch(family, loss, name, sigma):
    rng = np.random.default_rng(zlib.crc32(repr((family, loss, name, sigma)).encode()))
    sizes = skewed_sizes(rng)
    rows = np.array([ROWS[family][b % 2] for b in range(len(sizes))])
    x, y, d, p, rho, off = safe_windows(family, int(rng.integers(1 << 30)), sizes, rows)
    tau = P.tau_f32(d, off)
    g = incoming(rng, len(sizes), zero=20)
    r = rho if family == "camera_motion" else None
    ev = (x, y, d, p) if loss == "contrast" else (x, y, d, tau, p)
    ev = ev + ((rho,) if family == "camera_motion" else ())
    scalars = (sigma, {"variance": 0, "soe": 2}[name], 0.0) if loss == "contrast" else (sigma,)
    got = c_entry(family, loss, _cuda(*ev), off, rows, scalars, g)
    ref, imgs = reference(family, loss, x, y, d, tau, p, rho, off, rows, sigma, name, g)
    if loss == "contrast":
        M, c, E = B.param_contrast_bound(family, x, y, d, p, off, rows, sigma, name, 3.0, g, imgs[0], _centre(family), (H, W), r)
    else:
        M, c, E = B.param_timestamp_bound(family, x, y, d, tau, p, off, rows, sigma, g, *imgs, _centre(family), (H, W), r)
    what = "%s %s %s sigma %g" % (family, loss, name, sigma)
    _note(family + " C", B.check(got, ref, M, c, E, "C entry " + what))
    assert (got[20] == 0).all() and (got[3] == 0).all()
    K = got.shape[1] - 2 if family.startswith("camera") else got.shape[1]
    tg = torch_grad(family, loss, x, y, d, p, rho, off, rows, sigma, name, g)
    _note(family + " torch", B.check(tg, ref[:, :K], M[:, :K], c[:, :K], E[:, :K], "torch " + what))
    # the big window alone runs on many CTAs instead of few
    lo, hi = off[40], off[41]
    sl = slice(lo, hi)
    one = [a[sl] for a in ev]
    alone = c_entry(family, loss, _cuda(*one), np.array([0, hi - lo], np.int64), rows[40:41], scalars, g[40:41])
    _note(family + " C", B.check(alone[0], ref[40], M[40], c[40], E[40], "alone " + what))


@pytest.mark.parametrize("family", ["affine", "homography", "camera_rotation"])
def test_segmentation_parameter_and_weight_gradients(family):
    from event_utils_b200.contrast_max import motion_segmentation_objective_torch
    from event_utils_b200.contrast_max import warps
    rng = np.random.default_rng(7)
    rows2 = np.array(ROWS[family])
    sizes = [3001, 0, 1, 2500, 47]
    Mo = 2
    rows = np.stack([rows2[[b % 2, (b + 1) % 2]] for b in range(len(sizes))])
    # keep events safe under both models of their window
    x, y, d, p, _, off = safe_windows(family, 9, sizes, rows[:, 0])
    xw, yw = zip(*[_warp_of(family, rng, x[off[b]:off[b + 1]], y[off[b]:off[b + 1]], d[off[b]:off[b + 1]], None, rows[b, 1])
                   for b in range(len(sizes))])
    xw, yw = np.concatenate(xw), np.concatenate(yw)
    with np.errstate(invalid="ignore"):
        ok = ~(np.isfinite(xw) & np.isfinite(yw)) | ((np.abs(xw - np.round(xw)) >= 1e-3) & (np.abs(yw - np.round(yw)) >= 1e-3))
    assert ok.mean() > 0.9
    p = np.where(ok, p, 0.0).astype(np.float32)       # an unsafe event: zero polarity, no term in either model
    w = rng.random((x.size, Mo)).astype(np.float32)
    g = incoming(rng, len(sizes) * Mo, zero=0).reshape(len(sizes), Mo)
    K = 3 if family == "camera_rotation" else rows.shape[-1]
    wf = warps.camera_rotation_warp(INTR) if family == "camera_rotation" else \
        {"affine": warps.affine_warp, "homography": warps.homography_warp}[family](center=CENTRE)
    prm = torch.tensor(rows[..., :K], device="cuda", requires_grad=True)
    wt = torch.from_numpy(w).cuda().requires_grad_(True)
    f = motion_segmentation_objective_torch(*_cuda(x, y, d, p), wt, prm, wf, t0=0.0, blur_sigma=1.0, img_size=(H, W),
                                            batch_end_indices=torch.from_numpy(off[1:]).cuda())
    (f * torch.from_numpy(g).cuda()).sum().backward()
    p64 = torch.tensor(rows, dtype=torch.float64, requires_grad=True)
    w64 = torch.tensor(w, dtype=torch.float64, requires_grad=True)
    c = _centre(family)
    if family == "camera_rotation":
        fr, iwe = CR.segmentation(x, y, d, p, w64, off, p64, 1.0, "variance", c, img_size=(H, W))
    else:
        fr, iwe = P.segmentation(family, x, y, d, p, w64, off, p64, 1.0, "variance", 3.0, (H, W), c)
    (fr * torch.from_numpy(g)).sum().backward()
    M, cc, E, Mw, cw, Ew = B.segmentation_bound(family, x, y, d, p, w, off, rows, 1.0, g, iwe.detach().numpy(), c, (H, W))
    _note(family + " seg params", B.check(prm.grad.cpu().numpy(), p64.grad.numpy()[..., :K], M[..., :K], cc[..., :K], E[..., :K],
                                          "seg params " + family))
    _note(family + " seg weights", B.check(wt.grad.cpu().numpy(), w64.grad.numpy(), Mw, cw, Ew, "seg weights " + family,
                                           cast=True))
    assert (prm.grad[0, 0] == 0).all()


# ---- the node passes ----------------------------------------------------------------------------------------------

def node_cell_stream(rng, gh, gw, h, w, n):
    """One window's events in four parts: (a) sorted by node cell, so whole warps share a key; (b) two cells
    alternating lane by lane; (c) a run of one cell, every fifth event moved to x in (w-1, w) beyond the last node column
    (another key; two of its taps lie inside the grid) and every third event marked to add no term; (d) the outer ring
    of nodes.  Returns x, y and the mask of the marked events."""
    rx, ry = (w - 1) / (gw - 1), (h - 1) / (gh - 1)
    q = n // 4
    xa, ya = rng.random(q) * (w - 1), rng.random(q) * (h - 1)
    key = np.floor(ya / ry) * gw + np.floor(xa / rx)
    o = np.argsort(key, kind="stable")
    xa, ya = xa[o], ya[o]
    cx0, cy0 = (rng.integers(0, gw - 1, 2) + 0.5) * rx, (rng.integers(0, gh - 1, 2) + 0.5) * ry
    alt = np.arange(q) % 2
    xb = cx0[alt] + (rng.random(q) - 0.5) * 0.9 * rx
    yb = cy0[alt] + (rng.random(q) - 0.5) * 0.9 * ry
    xc = np.full(q, cx0[0]) + (rng.random(q) - 0.5) * 0.9 * rx
    yc = np.full(q, cy0[0]) + (rng.random(q) - 0.5) * 0.9 * ry
    xc[::5] = w - 1 + 0.05 + 0.9 * rng.random(xc[::5].size)
    m = n - 3 * q
    side = rng.integers(0, 4, m)
    t = rng.random(m)
    xd = np.where(side == 0, t * rx * 0.9, np.where(side == 1, w - 1 - t * rx * 0.9, rng.random(m) * (w - 1)))
    yd = np.where(side == 2, t * ry * 0.9, np.where(side == 3, h - 1 - t * ry * 0.9, rng.random(m) * (h - 1)))
    mark = np.zeros(n, bool)
    mark[2 * q + 1:3 * q:3] = True
    return np.concatenate((xa, xb, xc, xd)).astype(np.float32), np.concatenate((ya, yb, yc, yd)).astype(np.float32), mark


def node_windows(seed, sizes, gh, gw, h, w, drop):
    """node_cell_stream's windows back to back.  The marked events get the polarity `drop`, which adds no term: 0 for
    the contrast loss (a zero splat weight), NaN for the timestamp losses (in neither image).  The timestamp losses also
    get NaN polarities at every 13th event.  Lanes without a term also come from the events the warp sends off the
    canvas or (depth grid) behind the camera or through a negative node, and from the padded lanes past the end of
    every window, none of whose lengths is a multiple of 32."""
    rng = np.random.default_rng(seed)
    empty = (np.zeros(0, np.float32),) * 2 + (np.zeros(0, bool),)
    xs, ys, ms = zip(*[node_cell_stream(rng, gh, gw, h, w, n) if n else empty for n in sizes])
    x, y, mark = np.concatenate(xs), np.concatenate(ys), np.concatenate(ms)
    n = x.size
    d = (-rng.integers(0, 410, n) / 4096.0).astype(np.float32)
    p = (rng.integers(0, 2, n) * 2 - 1).astype(np.float32)
    if np.isnan(drop):
        p[7::13] = np.nan
    p[mark] = drop
    return x, y, d, p, np.concatenate(([0], np.cumsum(sizes))).astype(np.int64)


GRIDS = [(2, 2, H, W), (3, 4, H, W), (64, 64, 64, 64)]
NODE_CASES = [("contrast", "variance", 0.0), ("contrast", "soe", 1.0), ("timestamp", None, 0.0), ("timestamp", None, 1.0)]


def _unreached_zero(got, M):
    assert (got[M == 0] == 0).all(), "a node no event reaches has a gradient"


@pytest.mark.parametrize("loss,name,sigma", NODE_CASES)
@pytest.mark.parametrize("grid", GRIDS)
def test_grid_flow_node_gradient(grid, loss, name, sigma):
    from event_utils_b200.contrast_max import grid_flow_contrast_objective_torch, grid_flow_timestamp_objective_torch
    gh, gw, h, w = grid
    rng = np.random.default_rng(gh * 100 + gw)
    sizes = [6001, 0, 1, 4007, 129]
    x, y, d, p, off = node_windows(gh + gw, sizes, gh, gw, h, w, 0.0 if loss == "contrast" else np.nan)
    grids = (rng.standard_normal((len(sizes), 2, gh, gw)) * 20).astype(np.float32)
    grids[:, 0, :, -1] = -40.0        # the last node column sends events near the right edge off the canvas
    g = incoming(rng, len(sizes), zero=4)
    gt = torch.from_numpy(grids).cuda().requires_grad_(True)
    ends = torch.from_numpy(off[1:]).cuda()
    g64 = torch.from_numpy(grids.astype(np.float64)).requires_grad_(True)
    if loss == "contrast":
        f = grid_flow_contrast_objective_torch(*_cuda(x, y, d, p), gt, (h, w), t0=0.0, objective=name, blur_sigma=sigma,
                                               batch_end_indices=ends)
        fr, iwe = GR.reference(x, y, d, p, off, g64, h, w, sigma, name)
        imgs, tau = iwe.detach().numpy(), None
    else:
        # t0 = 0 and ts = d: the loss's tau is tau_f32(d)
        f = grid_flow_timestamp_objective_torch(*_cuda(x, y, d, p), gt, (h, w), t0=0.0, blur_sigma=sigma,
                                                batch_end_indices=ends)
        tau = P.tau_f32(d, off)
        fr, T, C = GTR.reference(x, y, d, tau, p, off, g64, h, w, sigma)
        imgs = (T.detach().numpy(), C.detach().numpy())
    (f * torch.from_numpy(g).cuda()).sum().backward()
    (fr * torch.from_numpy(g)).sum().backward()
    got, ref = gt.grad.cpu().numpy(), g64.grad.numpy()
    M, c, E = B.grid_flow_bound(loss, x, y, d, p, off, grids, h, w, sigma, g, imgs, name or "variance", tau=tau)
    _note("grid flow " + loss, B.check(got, ref, M, c, E, "grid flow %s %s %s %g" % (grid, loss, name, sigma), cast=True))
    _unreached_zero(got, M)
    assert (got[4] == 0).all() and (got[1] == 0).all()


# window 3 (4007 events) moves forward fast enough to put about a third of its events behind the camera
MOTION = [(2.0, -3.0, 4.0, 1.0, -0.8, 1.5), (-1.5, 1.5, -2.0, -1.5, 0.5, -1.0), (1.0, 0.5, -1.0, 0.8, -0.3, 2.0),
          (0.5, 1.0, -0.5, 0.4, 0.6, 30.0), (-0.5, 2.0, 1.0, -0.6, 0.9, 1.0)]


def _depth_safe(x, y, d, p, off, grids, intr, h, w, drop):
    """the polarity `drop` (0 for the contrast loss, NaN for the timestamp loss: no term either way) for the events whose
    warp lies within 1e-3 px of an integer, where f32 and f64 may take different taps"""
    p = p.copy()
    for b in range(len(off) - 1):
        sl = slice(off[b], off[b + 1])
        r = DR.event_rho_f32(x[sl], y[sl], grids[b], h, w)
        xw, yw = CM.warp(x[sl], y[sl], d[sl], r, MOTION[b][:3], MOTION[b][3:], intr)
        with np.errstate(invalid="ignore"):
            bad = np.isfinite(xw) & ((np.abs(xw - np.round(xw)) < 1e-3) | (np.abs(yw - np.round(yw)) < 1e-3))
        p[sl][bad] = drop
    return p


@pytest.mark.parametrize("loss,name,sigma", NODE_CASES)
@pytest.mark.parametrize("grid", GRIDS)
def test_depth_grid_node_gradient(grid, loss, name, sigma):
    from event_utils_b200.contrast_max import depth_grid_contrast_objective_torch, depth_grid_timestamp_objective_torch
    from event_utils_b200.contrast_max import warps
    gh, gw, h, w = grid
    intr = (70.3, 64.9, 0.55 * w, 0.45 * h)
    rng = np.random.default_rng(gh * 10 + gw)
    sizes = [6001, 0, 1, 4007, 129]
    x, y, d, p, off = node_windows(gh * gw, sizes, gh, gw, h, w, 0.0 if loss == "contrast" else np.nan)
    grids = rng.uniform(0.125, 1.0, (len(sizes), gh, gw)).astype(np.float32)
    grids[0, 0, 1] = -0.3                                # a negative node: the events that read it are dropped
    p = _depth_safe(x, y, d, p, off, grids, intr, h, w, 0.0 if loss == "contrast" else np.nan)
    sl = slice(off[3], off[4])
    xw, _ = CM.warp(x[sl], y[sl], d[sl], DR.event_rho_f32(x[sl], y[sl], grids[3], h, w), MOTION[3][:3], MOTION[3][3:], intr)
    assert np.isnan(xw).mean() > 0.1                     # lanes behind the camera inside the runs of window 3
    g = incoming(rng, len(sizes), zero=4)
    gt = torch.tensor(grids.astype(np.float64), device="cuda", requires_grad=True)
    mot = torch.tensor(np.asarray(MOTION), device="cuda")
    ends = torch.from_numpy(off[1:]).cuda()
    wf = warps.camera_motion_warp(intr)
    g64 = torch.from_numpy(grids.astype(np.float64)).requires_grad_(True)
    if loss == "contrast":
        f = depth_grid_contrast_objective_torch(*_cuda(x, y, d, p), gt, mot, wf, (h, w), t0=0.0, objective=name,
                                                blur_sigma=sigma, batch_end_indices=ends)
        fr, iwe = DR.contrast(x, y, d, p, off, g64, MOTION, intr, sigma, name, img_size=(h, w))
        imgs, tau = iwe.detach().numpy(), None
    else:
        f = depth_grid_timestamp_objective_torch(*_cuda(x, y, d, p), gt, mot, wf, (h, w), t0=0.0, blur_sigma=sigma,
                                                 batch_end_indices=ends)
        tau = P.tau_f32(d, off)
        fr, T, C = DTR.reference(x, y, d, tau, p, off, g64, MOTION, intr, sigma, img_size=(h, w))
        imgs = (T.detach().numpy(), C.detach().numpy())
    (f * torch.from_numpy(g).cuda()).sum().backward()
    (fr * torch.from_numpy(g)).sum().backward()
    got, ref = gt.grad.cpu().numpy(), g64.grad.numpy()
    M, c, E = B.depth_grid_bound(loss, x, y, d, p, off, grids, MOTION, intr, sigma, g, imgs, (h, w), name or "variance",
                              tau=tau)
    _note("depth grid " + loss, B.check(got, ref, M, c, E, "depth grid %s %s %s %g" % (grid, loss, name, sigma), cast=True))
    _unreached_zero(got, M)
    assert (got[4] == 0).all() and (got[1] == 0).all()
    if loss == "contrast" and sigma == 0.0:
        assert np.count_nonzero(M[2]) <= 4          # the one-event window reaches one node cell
