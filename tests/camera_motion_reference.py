"""f64 references of the batched contrast and timestamp losses under the camera-motion model (camera_motion_warp,
EVK_WARP_CAMERA_MOTION), and a scene of textured points at several depths seen by a moving camera -- TEST
INFRASTRUCTURE ONLY.

The warp rotates each event's bearing with R = exp([d w]x) from scipy's Rotation.from_rotvec and adds the translation
(rho d) v, independently of the kernel's Rodrigues formula; its 8-column Jacobian (w, v, fx, fy) is the matrix form
dP/dw = -d [R b]x J_l(d w) with the SO(3) left Jacobian of camera_rotation_reference, dP/dv = rho d I and dP/df through
the bearing.  As there, the keep decision and the floor of x', y' come from this f64 warp (the GPU tests place their
events at least 1e-3 px from every integer), and every position is the f64 warp with the Jacobian as its derivative, so
autograd through the losses gives the exact derivative of a row (wx, wy, wz, vx, vy, vz, fx, fy), the row of the C
entries.  The splat, blur, objectives and stamps are those of tests/flow_objective_reference.py and
tests/flow_timestamp_reference.py; the bearings, cross-product matrices, left Jacobian and windows those of
tests/camera_rotation_reference.py."""
import numpy as np
import torch
from scipy.spatial.transform import Rotation

from camera_rotation_reference import _bearings, _window, left_jacobian, skew
from flow_objective_reference import blur_matrix, objective_of, splat
from flow_timestamp_reference import tau_f32  # noqa: F401  (re-exported for the tests)
from motion_objective_reference import contributes


def _moved(x, y, d, rho, omega, v, fx, fy, cx, cy):
    """bearings b, rotations R, the rotated bearings U = R b and P = U + (rho d) v"""
    b = _bearings(x, y, fx, fy, cx, cy)
    d = np.asarray(d, np.float64)
    R = Rotation.from_rotvec(np.outer(d, np.asarray(omega, np.float64))).as_matrix()
    U = np.einsum("nij,nj->ni", R, b)
    with np.errstate(invalid="ignore"):          # an infinite rho times d = 0 or v = 0
        s = np.asarray(rho, np.float64) * d
        return b, R, U, U + s[:, None] * np.asarray(v, np.float64)[None, :]


def warp(x, y, d, rho, omega, v, intr):
    """f64 x', y' of events (x, y) with inverse depth rho at d = t - t0 under the angular velocity omega, the linear
    velocity v and intr = (fx, fy, cx, cy); NaN for an event that is not kept (Pz <= 0, or rho negative or not finite)"""
    fx, fy, cx, cy = intr
    _, _, _, P = _moved(x, y, d, rho, omega, v, fx, fy, cx, cy)
    with np.errstate(all="ignore"):
        xw, yw = cx + fx * P[:, 0] / P[:, 2], cy + fy * P[:, 1] / P[:, 2]
        out = ~(P[:, 2] > 0) | ~(np.asarray(rho, np.float64) >= 0) | ~np.isfinite(rho)
    xw[out] = np.nan
    yw[out] = np.nan
    return xw, yw


def jacobian(x, y, d, rho, omega, v, intr):
    """(2, 8, n) f64 rows dx'/d(wx, wy, wz, vx, vy, vz, fx, fy) and dy'/d(...)"""
    fx, fy, cx, cy = intr
    d = np.asarray(d, np.float64)
    b, R, U, P = _moved(x, y, d, rho, omega, v, fx, fy, cx, cy)
    n = b.shape[0]
    dP = np.zeros((n, 3, 8))
    dP[:, :, :3] = -d[:, None, None] * (skew(U) @ left_jacobian(np.outer(d, omega)))
    dP[:, :, 3:6] = (np.asarray(rho, np.float64) * d)[:, None, None] * np.eye(3)
    dP[:, :, 6] = R[:, :, 0] * (-b[:, 0] / fx)[:, None]
    dP[:, :, 7] = R[:, :, 1] * (-b[:, 1] / fy)[:, None]
    Px, Py, Pz = P.T
    gx = np.stack((fx / Pz, np.zeros(n), -fx * Px / Pz ** 2), -1)
    gy = np.stack((np.zeros(n), fy / Pz, -fy * Py / Pz ** 2), -1)
    jx, jy = np.einsum("ni,nik->kn", gx, dP), np.einsum("ni,nik->kn", gy, dP)
    jx[6] += Px / Pz
    jy[7] += Py / Pz
    return np.array([jx, jy])


def _split(row, centre):
    p = np.asarray(row, np.float64)
    return p[:3], p[3:6], (p[6], p[7]) + tuple(centre)


def _footprint(xb, yb, db, rb, k, xw, yw, prm, centre):
    """floors of the f64 warp and the bilinear fractions, differentiable in prm through the analytic Jacobian"""
    om, v, intr = _split(prm.detach().numpy(), centre)
    J = torch.from_numpy(jacobian(xb[k], yb[k], db[k], rb[k], om, v, intr))
    delta = prm - prm.detach()
    px, py = np.floor(xw[k]), np.floor(yw[k])
    dx = torch.from_numpy(xw[k] - px) + J[0].T @ delta
    dy = torch.from_numpy(yw[k] - py) + J[1].T @ delta
    return torch.from_numpy(px.astype(np.int64)), torch.from_numpy(py.astype(np.int64)), dx, dy


def _windows(x, y, d, rho, offsets, params, centre, H, W, *extra):
    """per window b: its events, the kept ones under params[b] and a footprint function of a subset of them"""
    n = x.shape[0]
    for b in range(params.shape[0]):
        lo, hi = max(int(offsets[b]), 0), min(int(offsets[b + 1]), n)
        xb, yb, db, rb, *eb = _window(lo, hi, x, y, d, rho, *extra)
        om, v, intr = _split(params[b].detach().numpy(), centre)
        xw, yw = warp(xb, yb, db, rb, om, v, intr)
        keep = contributes(xw, yw, H, W)
        yield b, eb, keep, lambda k: _footprint(xb, yb, db, rb, k, xw, yw, params[b], centre)


def contrast(x, y, d, p, rho, offsets, params, sigma, name, centre, param=3.0, img_size=(180, 240)):
    """f (B,) f64 torch (differentiable in `params`, a (B,8) f64 tensor of rows (wx, wy, wz, vx, vy, vz, fx, fy)) and
    the IWEs (B,H+1,W+1) of the motion contrast loss.  x, y, d, p, rho: f32 numpy arrays; offsets: B+1 ints; centre =
    (cx, cy)."""
    H, W = img_size
    Hc, Wc = H + 1, W + 1
    My, Mx = (torch.from_numpy(blur_matrix(n, sigma)) for n in (Hc, Wc))
    fs, iwes = [], []
    for b, (pb,), keep, footprint in _windows(x, y, d, rho, offsets, params, centre, H, W, p):
        k = np.flatnonzero(keep)
        if k.size:
            img = splat(*footprint(k), torch.from_numpy(pb[k].astype(np.float64)), Hc, Wc)
        else:
            img = torch.zeros((Hc, Wc), dtype=torch.float64) + 0 * params[b].sum()
        fs.append(objective_of(My @ img @ Mx.T, name, param))
        iwes.append(img)
    return torch.stack(fs), torch.stack(iwes)


def timestamp(x, y, d, tau, p, rho, offsets, params, sigma, centre, img_size=(180, 240)):
    """f (B,) f64 torch (differentiable in `params`, (B,8)), T and C (B,2,H+1,W+1) of the motion timestamp loss"""
    H, W = img_size
    Hc, Wc = H + 1, W + 1
    My, Mx = (torch.from_numpy(blur_matrix(n, sigma)) for n in (Hc, Wc))
    fs, Ts, Cs = [], [], []
    for b, (ub, pb), keep, footprint in _windows(x, y, d, rho, offsets, params, centre, H, W, tau, p):
        imgs, cnts = [], []
        for sel in (pb > 0, pb <= 0):
            k = np.flatnonzero(keep & sel)
            if k.size:
                px, py, dx, dy = footprint(k)
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


def motion_scene(omega, v, intr, rng, img_size=(180, 240), n_pts=300, per_pt=150, depths=(1.0, 8.0), duration=0.05,
                 t_end=None, margin=10.0):
    """Static textured points at depths drawn uniformly in `depths` (Z at t0), seen by a camera whose pose at time t in
    its frame at t0 is (exp(d [omega]x), d v), d = t - t0 (t0 the last stamp or t_end).  Point X0 appears at
    X_t = exp(d [omega]x)^T (X0 - d v) in the camera at t, so its events lie at the projection of X_t with the inverse
    depth 1 / Z_t, and the f64 warp at (omega, v) maps every event back onto the point's pixel at t0.  The points are
    drawn inside the canvas (margin px from its edges) at t0; events that fall off the canvas or behind the camera are
    dropped.  f64 arrays x, y, t, p and the events' inverse depth rho."""
    H, W = img_size
    fx, fy, cx, cy = intr
    px, py = rng.uniform(margin, W - margin, n_pts), rng.uniform(margin, H - margin, n_pts)
    X0 = _bearings(px, py, fx, fy, cx, cy) * rng.uniform(depths[0], depths[1], n_pts)[:, None]
    pol = rng.integers(0, 2, n_pts) * 2.0 - 1.0
    idx = rng.permutation(np.repeat(np.arange(n_pts), per_pt))
    t = np.sort(rng.uniform(0, duration, idx.size))
    d = t - (t[-1] if t_end is None else t_end)
    Rt = Rotation.from_rotvec(-np.outer(d, omega)).as_matrix()          # exp(d [omega]x)^T
    Xt = np.einsum("nij,nj->ni", Rt, X0[idx] - d[:, None] * np.asarray(v, np.float64)[None, :])
    with np.errstate(all="ignore"):
        x, y = cx + fx * Xt[:, 0] / Xt[:, 2], cy + fy * Xt[:, 1] / Xt[:, 2]
        rho = 1.0 / Xt[:, 2]
    on = (Xt[:, 2] > 0) & (x > 0) & (x < W - 1) & (y > 0) & (y < H - 1)
    return x[on], y[on], t[on], pol[idx][on], rho[on]
