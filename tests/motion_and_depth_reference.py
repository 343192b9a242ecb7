"""f64 torch reference of the joint motion-and-depth contrast loss (contrast_max/motion_and_depth.py): the depth-grid
reference of depth_grid_reference.contrast with the warp differentiable in the camera motion (w, v) as well as in the
nodes.  As in the other references the footprint is the f64 warp's, and its tangent carries the gradient: the
fractions of every kept event move by dx'/drho delta_rho + dx'/d(w, v) . delta_motion (camera_motion_reference.jacobian),
which is the exact derivative of the bilinear splat wherever no event crosses a pixel or the bounds mask."""
import numpy as np
import torch

import camera_motion_reference as CM
from depth_grid_reference import event_rho_f32, rho_jacobian
from flow_objective_reference import blur_matrix, objective_of, splat
from grid_flow_reference import node_taps
from motion_objective_reference import contributes


def contrast(x, y, d, p, offsets, grid, motion, intr, sigma, name, param=3.0, img_size=(180, 240), exact=False):
    """f (B,) f64 torch, differentiable in `grid` ((B,gh,gw) f64 tensor) and in `motion` ((B,6) f64 tensor).  x, y, d,
    p: f32 numpy arrays; offsets: B+1 ints; intr = (fx, fy, cx, cy).  Each event's rho is the kernel's f32
    interpolation (event_rho_f32), or with `exact` the f64 one, which central differences need."""
    H, W = img_size
    Hc, Wc = H + 1, W + 1
    B, gh, gw = grid.shape
    My, Mx = (torch.from_numpy(blur_matrix(n, sigma)) for n in (Hc, Wc))
    mot = motion.detach().numpy().reshape(B, 6)
    fs = []
    n = x.shape[0]
    for b in range(B):
        lo, hi = max(int(offsets[b]), 0), min(int(offsets[b + 1]), n)
        sl = slice(lo, max(lo, hi))
        xb, yb, db, pb = x[sl], y[sl], d[sl], p[sl]
        om, v = mot[b, :3], mot[b, 3:]
        gb = grid[b].detach().numpy()
        if exact:
            rows, cols, w, _ = node_taps(xb, yb, gh, gw, H, W)
            r = (gb[rows, cols] * w.astype(np.float64)).sum(1)
        else:
            r = event_rho_f32(xb, yb, gb, H, W).astype(np.float64)
        xw, yw = CM.warp(xb, yb, db, r, om, v, intr)
        k = np.flatnonzero(contributes(xw, yw, H, W))
        if k.size:
            rows, cols, w, _ = node_taps(xb[k], yb[k], gh, gw, H, W)
            rho = (grid[b][torch.from_numpy(rows), torch.from_numpy(cols)] * torch.from_numpy(w.astype(np.float64))).sum(1)
            delta = rho - rho.detach()
            dm = motion[b] - motion[b].detach()
            J = torch.from_numpy(rho_jacobian(xb[k], yb[k], db[k], r[k], om, v, intr))
            Jm = torch.from_numpy(CM.jacobian(xb[k], yb[k], db[k], r[k], om, v, intr)[:, :6])     # (2, 6, n)
            px, py = np.floor(xw[k]), np.floor(yw[k])
            dx = torch.from_numpy(xw[k] - px) + J[0] * delta + (Jm[0] * dm[:, None]).sum(0)
            dy = torch.from_numpy(yw[k] - py) + J[1] * delta + (Jm[1] * dm[:, None]).sum(0)
            img = splat(torch.from_numpy(px.astype(np.int64)), torch.from_numpy(py.astype(np.int64)), dx, dy,
                        torch.from_numpy(pb[k].astype(np.float64)), Hc, Wc)
        else:
            img = torch.zeros((Hc, Wc), dtype=torch.float64) + 0 * grid[b].sum() + 0 * motion[b].sum()
        fs.append(objective_of(My @ img @ Mx.T, name, param))
    return torch.stack(fs)
