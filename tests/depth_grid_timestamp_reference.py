"""f64 torch reference of the batched depth-grid average-timestamp loss (contrast_max/depth_grid_timestamp.py) -- TEST
INFRASTRUCTURE ONLY.

Per sample: the inverse depth of each event interpolated from the node grid with the kernel's f32 node cell and weights
(depth_grid_reference.event_rho_f32, grid_flow_reference.node_taps), in f64 and differentiable in the nodes; the warp of
camera_motion_reference at that f32 rho, which decides the keep rules and the floors; the derivative of x', y' in rho
(depth_grid_reference.rho_jacobian) as the tangent of the footprint; then per polarity the bilinear sums S = sum tau k
and C = 1 + sum k on the (H+1, W+1) canvas, T = S / C, the blur and f = sum G_+^2 + sum G_-^2 of
tests/flow_timestamp_reference.py."""
import numpy as np
import torch

import camera_motion_reference as CM
from depth_grid_reference import event_rho_f32, rho_jacobian
from flow_objective_reference import blur_matrix, splat
from grid_flow_reference import node_taps
from motion_objective_reference import contributes


def reference(x, y, d, tau, p, offsets, grid, motion, intr, sigma, img_size=(180, 240)):
    """f (B,) f64 torch (differentiable in `grid`, a (B,gh,gw) f64 tensor), T and C (B,2,H+1,W+1), polarity 0 positive.
    x, y, d, tau, p: f32 numpy arrays as the kernel receives them (d = t - t0 of each event's sample); offsets: B+1
    ints; motion: (B,6) (wx, wy, wz, vx, vy, vz); intr = (fx, fy, cx, cy)."""
    H, W = img_size
    Hc, Wc = H + 1, W + 1
    B, gh, gw = grid.shape
    My, Mx = (torch.from_numpy(blur_matrix(n, sigma)) for n in (Hc, Wc))
    motion = np.asarray(motion, np.float64).reshape(B, 6)
    fs, Ts, Cs = [], [], []
    n = x.shape[0]
    for b in range(B):
        lo, hi = max(int(offsets[b]), 0), min(int(offsets[b + 1]), n)
        sl = slice(lo, max(lo, hi))
        xb, yb, db, ub, pb = x[sl], y[sl], d[sl], tau[sl], p[sl]
        om, v = motion[b, :3], motion[b, 3:]
        r32 = event_rho_f32(xb, yb, grid[b].detach().numpy(), H, W)
        xw, yw = CM.warp(xb, yb, db, r32, om, v, intr)
        keep = contributes(xw, yw, H, W)
        imgs, cnts = [], []
        for sel in (pb > 0, pb <= 0):
            k = np.flatnonzero(keep & sel)
            if k.size:
                rows, cols, w, _ = node_taps(xb[k], yb[k], gh, gw, H, W)
                wt = torch.from_numpy(w.astype(np.float64))
                rho = (grid[b][torch.from_numpy(rows), torch.from_numpy(cols)] * wt).sum(1)
                delta = rho - rho.detach()
                J = torch.from_numpy(rho_jacobian(xb[k], yb[k], db[k], r32[k], om, v, intr))
                px, py = np.floor(xw[k]), np.floor(yw[k])
                dx = torch.from_numpy(xw[k] - px) + J[0] * delta
                dy = torch.from_numpy(yw[k] - py) + J[1] * delta
                px, py = torch.from_numpy(px.astype(np.int64)), torch.from_numpy(py.astype(np.int64))
                S = splat(px, py, dx, dy, torch.from_numpy(ub[k].astype(np.float64)), Hc, Wc)
                C = 1 + splat(px, py, dx, dy, torch.ones(k.size, dtype=torch.float64), Hc, Wc)
            else:
                S = torch.zeros((Hc, Wc), dtype=torch.float64) + 0 * grid[b].sum()
                C = torch.ones((Hc, Wc), dtype=torch.float64)
            imgs.append(S / C)
            cnts.append(C)
        T = torch.stack(imgs)
        G = My @ T @ Mx.T
        fs.append((G * G).sum())
        Ts.append(T)
        Cs.append(torch.stack(cnts))
    return torch.stack(fs), torch.stack(Ts), torch.stack(Cs)
