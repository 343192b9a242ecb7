"""f64 torch reference of the batched depth-grid contrast objective (contrast_max/depth_grid.py), and scenes of textured
points on known inverse-depth surfaces seen by a moving camera -- TEST INFRASTRUCTURE ONLY.

Per sample: the inverse depth of each event interpolated from the node grid with the kernel's f32 node cell and
weights (grid_flow_reference.node_taps), in f64 and differentiable in the nodes; the warp of camera_motion_reference at
the f32 rho the kernel computes (node_flow's order of terms), which decides the keep rules and the floors; and the
derivative of x', y' in rho, dP/drho = d v through the projection, as the tangent of the footprint.  The splat, blur
and objectives are those of tests/flow_objective_reference.py."""
import numpy as np
import torch
from scipy.spatial.transform import Rotation

import camera_motion_reference as CM
from camera_rotation_reference import _bearings
from flow_objective_reference import blur_matrix, objective_of, splat
from grid_flow_reference import node_taps
from motion_objective_reference import contributes

f32 = np.float32


def event_rho_f32(x, y, grid, H, W):
    """rho of every event in the kernel's f32 order of terms (node_depth)"""
    g = np.asarray(grid, f32)
    rows, cols, w, inside = node_taps(x, y, g.shape[0], g.shape[1], H, W)
    r = np.zeros(len(rows), f32)
    for k in range(4):
        q = np.where(inside[:, k], g[rows[:, k], cols[:, k]], f32(0))
        with np.errstate(all="ignore"):
            r = (r + q * w[:, k]).astype(f32)
    return r


def rho_jacobian(x, y, d, rho, omega, v, intr):
    """(2, n) f64 dx'/drho, dy'/drho: dP/drho = d v through the projection"""
    fx, fy, cx, cy = intr
    d = np.asarray(d, np.float64)
    _, _, _, P = CM._moved(x, y, d, rho, omega, v, fx, fy, cx, cy)
    dP = d[:, None] * np.asarray(v, np.float64)[None, :]
    Px, Py, Pz = P.T
    return np.array([fx * (dP[:, 0] * Pz - Px * dP[:, 2]) / Pz ** 2, fy * (dP[:, 1] * Pz - Py * dP[:, 2]) / Pz ** 2])


def contrast(x, y, d, p, offsets, grid, motion, intr, sigma, name, param=3.0, img_size=(180, 240)):
    """f (B,) f64 torch (differentiable in `grid`, a (B,gh,gw) f64 tensor) and the IWEs (B,H+1,W+1).  x, y, d, p: f32
    numpy arrays; offsets: B+1 ints; motion: (B,6) (wx, wy, wz, vx, vy, vz); intr = (fx, fy, cx, cy)."""
    H, W = img_size
    Hc, Wc = H + 1, W + 1
    B, gh, gw = grid.shape
    My, Mx = (torch.from_numpy(blur_matrix(n, sigma)) for n in (Hc, Wc))
    motion = np.asarray(motion, np.float64).reshape(B, 6)
    fs, iwes = [], []
    n = x.shape[0]
    for b in range(B):
        lo, hi = max(int(offsets[b]), 0), min(int(offsets[b + 1]), n)
        sl = slice(lo, max(lo, hi))
        xb, yb, db, pb = x[sl], y[sl], d[sl], p[sl]
        om, v = motion[b, :3], motion[b, 3:]
        r32 = event_rho_f32(xb, yb, grid[b].detach().numpy(), H, W)
        xw, yw = CM.warp(xb, yb, db, r32, om, v, intr)
        k = np.flatnonzero(contributes(xw, yw, H, W))
        if k.size:
            rows, cols, w, _ = node_taps(xb[k], yb[k], gh, gw, H, W)
            rho = (grid[b][torch.from_numpy(rows), torch.from_numpy(cols)] * torch.from_numpy(w.astype(np.float64))).sum(1)
            delta = rho - rho.detach()
            J = torch.from_numpy(rho_jacobian(xb[k], yb[k], db[k], r32[k], om, v, intr))
            px, py = np.floor(xw[k]), np.floor(yw[k])
            dx = torch.from_numpy(xw[k] - px) + J[0] * delta
            dy = torch.from_numpy(yw[k] - py) + J[1] * delta
            img = splat(torch.from_numpy(px.astype(np.int64)), torch.from_numpy(py.astype(np.int64)), dx, dy,
                        torch.from_numpy(pb[k].astype(np.float64)), Hc, Wc)
        else:
            img = torch.zeros((Hc, Wc), dtype=torch.float64) + 0 * grid[b].sum()
        fs.append(objective_of(My @ img @ Mx.T, name, param))
        iwes.append(img)
    return torch.stack(fs), torch.stack(iwes)


def slanted_plane(a, bx, by):
    """the inverse depth a + bx (x - cx) / fx + by (y - cy) / fy of the plane n . X = 1 with n = (bx, by, a): affine in
    the pixel coordinates, so exactly representable on any node grid"""
    return lambda px, py, intr: a + bx * (px - intr[2]) / intr[0] + by * (py - intr[3]) / intr[1]


def two_planes(left, right, x_step):
    """a step at column x_step between two fronto-parallel planes of inverse depth left and right"""
    return lambda px, py, intr: np.where(px < x_step, left, right)


def depth_scene(surface, omega, v, intr, rng, img_size=(180, 240), n_pts=600, per_pt=60, duration=0.05, margin=8.0):
    """Static textured points at the pixels (px, py) at t0 with the inverse depth surface(px, py, intr), seen by a camera
    whose pose at time t in its frame at t0 is (exp(d [omega]x), d v), d = t - t0 (t0 the last stamp), as
    camera_motion_reference.motion_scene.  Returns f64 x, y, t, p of the events that stay on the sensor and in front of
    the camera, and the points' pixels and true inverse depth (px, py, rho0)."""
    H, W = img_size
    fx, fy, cx, cy = intr
    px, py = rng.uniform(margin, W - margin, n_pts), rng.uniform(margin, H - margin, n_pts)
    rho0 = surface(px, py, intr)
    X0 = _bearings(px, py, fx, fy, cx, cy) / rho0[:, None]
    pol = rng.integers(0, 2, n_pts) * 2.0 - 1.0
    idx = rng.permutation(np.repeat(np.arange(n_pts), per_pt))
    t = np.sort(rng.uniform(0, duration, idx.size))
    d = t - t[-1]
    Rt = Rotation.from_rotvec(-np.outer(d, omega)).as_matrix()
    Xt = np.einsum("nij,nj->ni", Rt, X0[idx] - d[:, None] * np.asarray(v, np.float64)[None, :])
    with np.errstate(all="ignore"):
        x, y = cx + fx * Xt[:, 0] / Xt[:, 2], cy + fy * Xt[:, 1] / Xt[:, 2]
    on = (Xt[:, 2] > 0) & (x > 0) & (x < W - 1) & (y > 0) & (y < H - 1)
    return x[on], y[on], t[on], pol[idx][on], (px, py, rho0)


def grid_at(grid, px, py, H, W):
    """f64 bilinear interpolation (align_corners) of one (gh, gw) grid at the pixels (px, py)"""
    g = np.asarray(grid, np.float64)
    gh, gw = g.shape
    ix, iy = np.asarray(px) * (gw - 1) / (W - 1), np.asarray(py) * (gh - 1) / (H - 1)
    x0, y0 = np.clip(np.floor(ix).astype(int), 0, gw - 2), np.clip(np.floor(iy).astype(int), 0, gh - 2)
    fx, fy = ix - x0, iy - y0
    return ((1 - fx) * (1 - fy) * g[y0, x0] + fx * (1 - fy) * g[y0, x0 + 1] + (1 - fx) * fy * g[y0 + 1, x0]
            + fx * fy * g[y0 + 1, x0 + 1])
