"""f64 references of the batched contrast, timestamp and segmentation losses under the camera-rotation model
(camera_rotation_warp, EVK_WARP_CAMERA_ROTATION) -- TEST INFRASTRUCTURE ONLY.

The warp rotates each event's bearing with R = exp([d w]x) from scipy's Rotation.from_rotvec, independently of the
kernel's Rodrigues formula; its 5-column Jacobian (w, fx, fy) is the matrix form dP/dw = -d [P]x J_l(d w) with the
textbook SO(3) left Jacobian, and dP/df through the bearing.  The kernel's sine cannot be restated bit for bit, so the
keep decision and the floor of x', y' come from this f64 warp: the GPU tests place their events at least 1e-3 px from
every integer, where f32 rounding cannot move a tap.  A loss row is (wx, wy, wz, fx, fy), the row of the C entries, and
every position is the f64 warp with the Jacobian as its derivative, so autograd through the losses gives the exact
derivative, the focal lengths included.  The splat, blur and objectives are those of tests/flow_objective_reference.py
and the loops restate tests/planar_motion_reference.py."""
import numpy as np
import torch
from scipy.spatial.transform import Rotation

from flow_objective_reference import blur_matrix, objective_of, splat
from flow_timestamp_reference import tau_f32  # noqa: F401  (re-exported for the tests)
from motion_objective_reference import contributes


def skew(v):
    """(n,3) -> (n,3,3) cross-product matrices [v]x"""
    v = np.atleast_2d(v)
    z = np.zeros(v.shape[0])
    return np.stack((np.stack((z, -v[:, 2], v[:, 1]), -1), np.stack((v[:, 2], z, -v[:, 0]), -1),
                     np.stack((-v[:, 1], v[:, 0], z), -1)), 1)


def _bearings(x, y, fx, fy, cx, cy):
    x, y = np.asarray(x, np.float64), np.asarray(y, np.float64)
    return np.stack(((x - cx) / fx, (y - cy) / fy, np.ones_like(x)), -1)


def _rotated(x, y, d, omega, fx, fy, cx, cy):
    b = _bearings(x, y, fx, fy, cx, cy)
    R = Rotation.from_rotvec(np.outer(np.asarray(d, np.float64), np.asarray(omega, np.float64))).as_matrix()
    return b, R, np.einsum("nij,nj->ni", R, b)


def warp(x, y, d, omega, intr):
    """f64 x', y' of events (x, y) at d = t - t0 under the angular velocity omega and intr = (fx, fy, cx, cy); NaN for
    an event rotated behind the camera (Pz <= 0)"""
    fx, fy, cx, cy = intr
    _, _, P = _rotated(x, y, d, omega, fx, fy, cx, cy)
    with np.errstate(all="ignore"):
        xw, yw = cx + fx * P[:, 0] / P[:, 2], cy + fy * P[:, 1] / P[:, 2]
    behind = ~(P[:, 2] > 0)
    xw[behind] = np.nan
    yw[behind] = np.nan
    return xw, yw


def left_jacobian(theta):
    """(n,3) rotation vectors -> (n,3,3) J_l = I + (1 - cos phi) / phi^2 [theta]x + (phi - sin phi) / phi^3 [theta]x^2"""
    phi = np.linalg.norm(theta, axis=1)
    small = phi < 1e-3
    ps = np.where(small, 1.0, phi)
    b = np.where(small, 0.5 - phi ** 2 / 24, (1 - np.cos(ps)) / ps ** 2)
    c = np.where(small, 1.0 / 6 - phi ** 2 / 120, (ps - np.sin(ps)) / ps ** 3)
    K = skew(theta)
    return np.eye(3) + b[:, None, None] * K + c[:, None, None] * (K @ K)


def jacobian(x, y, d, omega, intr):
    """(2, 5, n) f64 rows dx'/d(wx, wy, wz, fx, fy) and dy'/d(...)"""
    fx, fy, cx, cy = intr
    d = np.asarray(d, np.float64)
    b, R, P = _rotated(x, y, d, omega, fx, fy, cx, cy)
    n = b.shape[0]
    dP = np.empty((n, 3, 5))
    dP[:, :, :3] = -d[:, None, None] * (skew(P) @ left_jacobian(np.outer(d, omega)))
    dP[:, :, 3] = R[:, :, 0] * (-b[:, 0] / fx)[:, None]          # b_x = (x - cx) / fx
    dP[:, :, 4] = R[:, :, 1] * (-b[:, 1] / fy)[:, None]
    Px, Py, Pz = P.T
    gx = np.stack((fx / Pz, np.zeros(n), -fx * Px / Pz ** 2), -1)
    gy = np.stack((np.zeros(n), fy / Pz, -fy * Py / Pz ** 2), -1)
    jx, jy = np.einsum("ni,nik->kn", gx, dP), np.einsum("ni,nik->kn", gy, dP)
    jx[3] += Px / Pz
    jy[4] += Py / Pz
    return np.array([jx, jy])


def embedding_matrix(intr):
    """E (8,3): the homography_warp parameters about (cx, cy) that hold the rotation w to first order in d, h = E w.
    The generator of homography_warp is -K'[w]x K'^-1 with K' = diag(fx, fy, 1) on (x - cx, y - cy, 1):
    (hx, hy, a11, a12, a21, a22, g1, g2) = (-fx wy, fy wx, 0, fx/fy wz, -fy/fx wz, 0, wy/fx, -wx/fy)"""
    fx, fy = intr[0], intr[1]
    E = np.zeros((8, 3))
    E[0, 1], E[1, 0] = -fx, fy
    E[3, 2], E[4, 2] = fx / fy, -fy / fx
    E[6, 1], E[7, 0] = 1.0 / fx, -1.0 / fy
    return E


def embedding(omega, intr):
    return embedding_matrix(intr) @ np.asarray(omega, np.float64)


def _window(lo, hi, *arrays):
    sl = slice(lo, max(lo, hi))
    return [a[sl] for a in arrays]


def _kept(xb, yb, db, prm, H, W, centre):
    p = prm.detach().numpy()
    xw, yw = warp(xb, yb, db, p[:3], (p[3], p[4]) + tuple(centre))
    return xw, yw, contributes(xw, yw, H, W)


def _footprint(xb, yb, db, k, xw, yw, prm, centre):
    """floors of the f64 warp and the bilinear fractions, differentiable in prm through the analytic Jacobian"""
    p = prm.detach().numpy()
    J = torch.from_numpy(jacobian(xb[k], yb[k], db[k], p[:3], (p[3], p[4]) + tuple(centre)))
    delta = prm - prm.detach()
    px, py = np.floor(xw[k]), np.floor(yw[k])
    dx = torch.from_numpy(xw[k] - px) + J[0].T @ delta
    dy = torch.from_numpy(yw[k] - py) + J[1].T @ delta
    return torch.from_numpy(px.astype(np.int64)), torch.from_numpy(py.astype(np.int64)), dx, dy


def contrast(x, y, d, p, offsets, params, sigma, name, centre, param=3.0, img_size=(180, 240)):
    """f (B,) f64 torch (differentiable in `params`, a (B,5) f64 tensor of rows (wx, wy, wz, fx, fy)) and the IWEs
    (B,H+1,W+1) of the motion contrast loss.  x, y, d, p: f32 numpy arrays; offsets: B+1 ints; centre = (cx, cy)."""
    H, W = img_size
    Hc, Wc = H + 1, W + 1
    My, Mx = (torch.from_numpy(blur_matrix(n, sigma)) for n in (Hc, Wc))
    fs, iwes = [], []
    n = x.shape[0]
    for b in range(params.shape[0]):
        xb, yb, db, pb = _window(max(int(offsets[b]), 0), min(int(offsets[b + 1]), n), x, y, d, p)
        xw, yw, keep = _kept(xb, yb, db, params[b], H, W, centre)
        k = np.flatnonzero(keep)
        if k.size:
            px, py, dx, dy = _footprint(xb, yb, db, k, xw, yw, params[b], centre)
            img = splat(px, py, dx, dy, torch.from_numpy(pb[k].astype(np.float64)), Hc, Wc)
        else:
            img = torch.zeros((Hc, Wc), dtype=torch.float64) + 0 * params[b].sum()
        fs.append(objective_of(My @ img @ Mx.T, name, param))
        iwes.append(img)
    return torch.stack(fs), torch.stack(iwes)


def timestamp(x, y, d, tau, p, offsets, params, sigma, centre, img_size=(180, 240)):
    """f (B,) f64 torch (differentiable in `params`, (B,5)), T and C (B,2,H+1,W+1) of the motion timestamp loss"""
    H, W = img_size
    Hc, Wc = H + 1, W + 1
    My, Mx = (torch.from_numpy(blur_matrix(n, sigma)) for n in (Hc, Wc))
    fs, Ts, Cs = [], [], []
    n = x.shape[0]
    for b in range(params.shape[0]):
        xb, yb, db, ub, pb = _window(max(int(offsets[b]), 0), min(int(offsets[b + 1]), n), x, y, d, tau, p)
        xw, yw, keep = _kept(xb, yb, db, params[b], H, W, centre)
        imgs, cnts = [], []
        for sel in (pb > 0, pb <= 0):
            k = np.flatnonzero(keep & sel)
            if k.size:
                px, py, dx, dy = _footprint(xb, yb, db, k, xw, yw, params[b], centre)
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


def segmentation(x, y, d, p, w, offsets, params, sigma, name, centre, param=3.0, img_size=(180, 240)):
    """f (B,M) f64 torch, differentiable in params ((B,M,5) f64) and w ((N,M) f64), and the images (B,M,H+1,W+1)"""
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
            xw, yw, keep = _kept(xb, yb, db, params[b, m], H, W, centre)
            k = np.flatnonzero(keep)
            if k.size:
                px, py, dx, dy = _footprint(xb, yb, db, k, xw, yw, params[b, m], centre)
                wk = torch.from_numpy(pb[k].astype(np.float64)) * w[lo + torch.from_numpy(k), m]
                img = splat(px, py, dx, dy, wk, Hc, Wc)
            else:
                img = torch.zeros((Hc, Wc), dtype=torch.float64) + 0 * params[b, m].sum() + 0 * w[:, m].sum()
            fs.append(objective_of(My @ img @ Mx.T, name, param))
            imgs.append(img)
    return torch.stack(fs).reshape(B, M), torch.stack(imgs).reshape(B, M, Hc, Wc)


def assign(x, y, d, offsets, params, iwe, sigma, eps, centre, img_size=(180, 240)):
    """(N,M) f64 memberships of the E-step (motion_segmentation_reference.assign with this warp); params (B,M,5)"""
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
            prm = np.asarray(params[b, m], np.float64)
            xw, yw = warp(x[lo:hi], y[lo:hi], d[lo:hi], prm[:3], (prm[3], prm[4]) + tuple(centre))
            k = np.flatnonzero(contributes(xw, yw, H, W))
            px, py = np.floor(xw[k]).astype(np.int64), np.floor(yw[k]).astype(np.int64)
            dx, dy = xw[k] - px, yw[k] - py
            v = ((1 - dx) * (1 - dy) * G[py, px] + dx * (1 - dy) * G[py, px + 1] + (1 - dx) * dy * G[py + 1, px] +
                 dx * dy * G[py + 1, px + 1])
            c[k, m] = np.where(v < 0, 0.0, v)
        den = c.sum(1, keepdims=True) + M * eps
        with np.errstate(invalid="ignore", divide="ignore"):
            out[lo:hi] = np.where(den == 0, 1.0 / M, (c + eps) / den)
    return out


def rotation_scene(omega, intr, rng, img_size=(180, 240), n_pts=300, per_pt=150, duration=0.05, t_end=None, margin=10.0):
    """Static points on the viewing sphere seen by a camera rotating at omega during `duration`: every event of a point
    lies at exp(-[omega]x d) of the point's bearing (d = t - t0, t0 the last stamp or t_end), so the f64 warp at omega
    maps it back onto the point.  The points are drawn inside the canvas (margin px from its edges) at t0; events that
    fall off the canvas are dropped.  f64 arrays x, y, t, p."""
    H, W = img_size
    fx, fy, cx, cy = intr
    px, py = rng.uniform(margin, W - margin, n_pts), rng.uniform(margin, H - margin, n_pts)
    b0 = _bearings(px, py, fx, fy, cx, cy)
    pol = rng.integers(0, 2, n_pts) * 2.0 - 1.0
    idx = rng.permutation(np.repeat(np.arange(n_pts), per_pt))
    t = np.sort(rng.uniform(0, duration, idx.size))
    d = t - (t[-1] if t_end is None else t_end)
    P = np.einsum("nij,nj->ni", Rotation.from_rotvec(-np.outer(d, omega)).as_matrix(), b0[idx])
    with np.errstate(all="ignore"):
        x, y = cx + fx * P[:, 0] / P[:, 2], cy + fy * P[:, 1] / P[:, 2]
    on = (P[:, 2] > 0) & (x > 0) & (x < W - 1) & (y > 0) & (y < H - 1)
    return x[on], y[on], t[on], pol[idx][on]
