"""f64 torch references of the batched contrast, timestamp and segmentation losses under the planar motion models
(affine_warp, homography_warp) -- TEST INFRASTRUCTURE ONLY.

Per window: the keep decision and the floor of x', y' from an op-by-op f32 restatement of the kernel's warp (model_taps
in csrc/evk_cmax.cu; an event past the homography's horizon, w <= 0 or w not finite, comes out as NaN and is not kept),
then the warp in f64, differentiable in the parameters.  The splat, blur and objectives are those of
tests/flow_objective_reference.py, the timestamp images those of tests/motion_timestamp_reference.py, and the loops
restate tests/motion_objective_reference.py, motion_timestamp_reference.py and motion_segmentation_reference.py with
these warps.  Autograd through them gives the exact derivative the backward kernels implement."""
import numpy as np
import torch

from flow_objective_reference import blur_matrix, objective_of, splat
from flow_timestamp_reference import tau_f32  # noqa: F401  (re-exported for the tests)
from motion_objective_reference import contributes

f32 = np.float32
DIMS = {"affine": 6, "homography": 8}
CENTRE = (120.0, 90.0)


def warp_f32(kind, x, y, d, prm, centre=CENTRE):
    """The kernel's f32 warp, op by op: x', y' as float32 arrays, NaN past the horizon (prm cast to f32 like the
    kernel's (R)M.m[k])."""
    x, y, d = (np.asarray(a, f32) for a in (x, y, d))
    m = [f32(v) for v in prm]
    cx, cy = f32(centre[0]), f32(centre[1])
    with np.errstate(all="ignore"):
        u, v = (x - cx).astype(f32), (y - cy).astype(f32)
        sx = ((m[0] + m[2] * u) + m[3] * v).astype(f32)
        sy = ((m[1] + m[5] * v) + m[4] * u).astype(f32)
        mx, my = (d * sx).astype(f32), (d * sy).astype(f32)
        xw, yw = (x - mx).astype(f32), (y - my).astype(f32)
        if kind == "affine":
            return xw, yw
        nx, ny = (u - mx).astype(f32), (v - my).astype(f32)
        q = (d * ((m[6] * u).astype(f32) + (m[7] * v).astype(f32))).astype(f32)
        w = (f32(1) - q).astype(f32)
        xw = (xw + ((nx * q).astype(f32) / w).astype(f32)).astype(f32)
        yw = (yw + ((ny * q).astype(f32) / w).astype(f32)).astype(f32)
        past = ~((w > 0) & np.isfinite(w))
        xw[past] = np.nan
        yw[past] = np.nan
        return xw, yw


def warp_f64(kind, x, y, d, prm, centre=CENTRE):
    """The same warp in f64 torch, differentiable in prm (a (K,) f64 tensor)."""
    u, v = x - centre[0], y - centre[1]
    sx = (prm[0] + prm[2] * u) + prm[3] * v
    sy = (prm[1] + prm[5] * v) + prm[4] * u
    if kind == "affine":
        return x - d * sx, y - d * sy
    w = 1 - d * (prm[6] * u + prm[7] * v)
    return centre[0] + (u - d * sx) / w, centre[1] + (v - d * sy) / w


def jacobian(kind, x, y, d, prm, centre=CENTRE):
    """(2, K, n) f64 rows dx'/dp_k, dy'/dp_k (the closed forms of contrast_max/warps.py)"""
    x, y, d = (np.asarray(a, np.float64) for a in (x, y, d))
    z = np.zeros_like(d)
    u, v = x - centre[0], y - centre[1]
    du, dv = d * u, d * v
    rx, ry = [-d, z, -du, -dv, z, z], [z, -d, z, z, -du, -dv]
    if kind == "affine":
        return np.array([rx, ry])
    p = [float(a) for a in prm]
    sx, sy = (p[0] + p[2] * u) + p[3] * v, (p[1] + p[5] * v) + p[4] * u
    nx, ny = u - d * sx, v - d * sy
    w = 1 - d * (p[6] * u + p[7] * v)
    return np.array([[r / w for r in rx] + [nx * du / w ** 2, nx * dv / w ** 2],
                     [r / w for r in ry] + [ny * du / w ** 2, ny * dv / w ** 2]])


def _window(lo, hi, *arrays):
    sl = slice(lo, max(lo, hi))
    return [a[sl] for a in arrays]


def _kept(kind, xb, yb, db, prm, H, W, centre):
    """the f32 warp x', y' of the window's events and the mask of those that contribute"""
    xw32, yw32 = warp_f32(kind, xb, yb, db, prm.detach().numpy(), centre)
    return xw32, yw32, contributes(xw32, yw32, H, W)


def _footprint(kind, xb, yb, db, k, xw32, yw32, prm, centre):
    t64 = [torch.from_numpy(a[k].astype(np.float64)) for a in (xb, yb, db)]
    xw, yw = warp_f64(kind, *t64, prm, centre)
    px = torch.from_numpy(np.floor(xw32[k]).astype(np.int64))
    py = torch.from_numpy(np.floor(yw32[k]).astype(np.int64))
    return px, py, xw - px.double(), yw - py.double()


def contrast(kind, x, y, d, p, offsets, params, sigma, name, param=3.0, img_size=(180, 240), centre=CENTRE):
    """f (B,) f64 torch (differentiable in `params`, a (B,K) f64 tensor) and the IWEs (B,H+1,W+1) of the motion contrast
    loss.  x, y, d, p: f32 numpy arrays (d = t - t0 of each event's window); offsets: B+1 ints."""
    H, W = img_size
    Hc, Wc = H + 1, W + 1
    My, Mx = (torch.from_numpy(blur_matrix(n, sigma)) for n in (Hc, Wc))
    fs, iwes = [], []
    n = x.shape[0]
    for b in range(params.shape[0]):
        xb, yb, db, pb = _window(max(int(offsets[b]), 0), min(int(offsets[b + 1]), n), x, y, d, p)
        xw32, yw32, keep = _kept(kind, xb, yb, db, params[b], H, W, centre)
        k = np.flatnonzero(keep)
        if k.size:
            px, py, dx, dy = _footprint(kind, xb, yb, db, k, xw32, yw32, params[b], centre)
            img = splat(px, py, dx, dy, torch.from_numpy(pb[k].astype(np.float64)), Hc, Wc)
        else:
            img = torch.zeros((Hc, Wc), dtype=torch.float64) + 0 * params[b].sum()
        fs.append(objective_of(My @ img @ Mx.T, name, param))
        iwes.append(img)
    return torch.stack(fs), torch.stack(iwes)


def timestamp(kind, x, y, d, tau, p, offsets, params, sigma, img_size=(180, 240), centre=CENTRE):
    """f (B,) f64 torch (differentiable in `params`), T and C (B,2,H+1,W+1) of the motion timestamp loss"""
    H, W = img_size
    Hc, Wc = H + 1, W + 1
    My, Mx = (torch.from_numpy(blur_matrix(n, sigma)) for n in (Hc, Wc))
    fs, Ts, Cs = [], [], []
    n = x.shape[0]
    for b in range(params.shape[0]):
        xb, yb, db, ub, pb = _window(max(int(offsets[b]), 0), min(int(offsets[b + 1]), n), x, y, d, tau, p)
        xw32, yw32, keep = _kept(kind, xb, yb, db, params[b], H, W, centre)
        imgs, cnts = [], []
        for sel in (pb > 0, pb <= 0):
            k = np.flatnonzero(keep & sel)
            if k.size:
                px, py, dx, dy = _footprint(kind, xb, yb, db, k, xw32, yw32, params[b], centre)
                S = splat(px, py, dx, dy, torch.from_numpy(ub[k].astype(np.float64)), Hc, Wc)
                C = 1 + splat(px, py, dx, dy, torch.ones(k.size, dtype=torch.float64), Hc, Wc)
            else:
                S = torch.zeros((Hc, Wc), dtype=torch.float64) + 0 * params[b].sum()
                C = torch.ones((Hc, Wc), dtype=torch.float64)
            imgs.append(S / C)
            cnts.append(C)
        T = torch.stack(imgs)
        G = My @ T @ Mx.T
        fs.append((G * G).sum())
        Ts.append(T)
        Cs.append(torch.stack(cnts))
    return torch.stack(fs), torch.stack(Ts), torch.stack(Cs)


def segmentation(kind, x, y, d, p, w, offsets, params, sigma, name, param=3.0, img_size=(180, 240), centre=CENTRE):
    """f (B,M) f64 torch, differentiable in params ((B,M,K) f64) and w ((N,M) f64), and the images (B,M,H+1,W+1)"""
    H, W = img_size
    Hc, Wc = H + 1, W + 1
    My, Mx = (torch.from_numpy(blur_matrix(n, sigma)) for n in (Hc, Wc))
    B, M, _ = params.shape
    n = x.shape[0]
    fs, imgs = [], []
    for b in range(B):
        lo = max(int(offsets[b]), 0)
        xb, yb, db, pb = _window(lo, min(int(offsets[b + 1]), n), x, y, d, p)
        for m in range(M):
            xw32, yw32, keep = _kept(kind, xb, yb, db, params[b, m], H, W, centre)
            k = np.flatnonzero(keep)
            if k.size:
                px, py, dx, dy = _footprint(kind, xb, yb, db, k, xw32, yw32, params[b, m], centre)
                wk = torch.from_numpy(pb[k].astype(np.float64)) * w[lo + torch.from_numpy(k), m]
                img = splat(px, py, dx, dy, wk, Hc, Wc)
            else:
                img = torch.zeros((Hc, Wc), dtype=torch.float64) + 0 * params[b, m].sum() + 0 * w[:, m].sum()
            fs.append(objective_of(My @ img @ Mx.T, name, param))
            imgs.append(img)
    return torch.stack(fs).reshape(B, M), torch.stack(imgs).reshape(B, M, Hc, Wc)


def assign(kind, x, y, d, offsets, params, iwe, sigma, eps, img_size=(180, 240), centre=CENTRE):
    """(N,M) f64 memberships of the E-step (motion_segmentation_reference.assign with these warps)"""
    H, W = img_size
    Hc, Wc = H + 1, W + 1
    My, Mx = blur_matrix(Hc, sigma), blur_matrix(Wc, sigma)
    B, M, _ = np.shape(params)
    n = x.shape[0]
    out = np.full((n, M), 1.0 / M)
    for b in range(B):
        lo, hi = max(int(offsets[b]), 0), min(int(offsets[b + 1]), n)
        if hi <= lo:
            continue
        c = np.zeros((hi - lo, M))
        for m in range(M):
            G = My @ np.asarray(iwe[b, m], np.float64) @ Mx.T
            xw, yw = warp_f32(kind, x[lo:hi], y[lo:hi], d[lo:hi], np.asarray(params[b, m]), centre)
            k = np.flatnonzero(contributes(xw, yw, H, W))
            px, py = np.floor(xw[k]).astype(np.int64), np.floor(yw[k]).astype(np.int64)
            dx, dy = xw[k].astype(np.float64) - px, yw[k].astype(np.float64) - py
            v = ((1 - dx) * (1 - dy) * G[py, px] + dx * (1 - dy) * G[py, px + 1] + (1 - dx) * dy * G[py + 1, px] +
                 dx * dy * G[py + 1, px + 1])
            c[k, m] = np.where(v < 0, 0.0, v)
        den = c.sum(1, keepdims=True) + M * eps
        with np.errstate(invalid="ignore", divide="ignore"):
            out[lo:hi] = np.where(den == 0, 1.0 / M, (c + eps) / den)
    return out


def planar_scene(kind, truth, rng, n_pts=300, per_pt=150, duration=0.05, centre=CENTRE, radius=60.0, t_end=None):
    """A static cloud of points moving with the planar motion `truth` during `duration`: the event positions are chosen
    so that the f64 warp of `kind` at `truth` (t0 = the last stamp, or t_end) maps every event of a point back onto the
    point.  f64 arrays x, y, t, p."""
    ang, rad = rng.uniform(0, 2 * np.pi, n_pts), radius * np.sqrt(rng.uniform(0.05, 1, n_pts))
    r0x, r0y = np.repeat(rad * np.cos(ang), per_pt), np.repeat(rad * np.sin(ang), per_pt)
    p = np.repeat(rng.integers(0, 2, n_pts) * 2.0 - 1.0, per_pt)
    order = rng.permutation(r0x.size)
    r0x, r0y, p = r0x[order], r0y[order], p[order]
    t = np.sort(rng.uniform(0, duration, r0x.size))
    d = t - (t[-1] if t_end is None else t_end)
    hx, hy, a11, a12, a21, a22 = truth[:6]
    g1, g2 = (truth[6], truth[7]) if kind == "homography" else (0.0, 0.0)
    # (I - d A + d r g^T) u = r + d h for u = (x - cx, y - cy), r the point relative to the centre
    m00, m01 = 1 - d * a11 + d * r0x * g1, -d * a12 + d * r0x * g2
    m10, m11 = -d * a21 + d * r0y * g1, 1 - d * a22 + d * r0y * g2
    bx, by = r0x + d * hx, r0y + d * hy
    det = m00 * m11 - m01 * m10
    u, v = (m11 * bx - m01 * by) / det, (m00 * by - m10 * bx) / det
    return centre[0] + u, centre[1] + v, t, p
