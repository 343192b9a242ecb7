"""f64 torch reference of the batched grid-flow average-timestamp loss (contrast_max/grid_flow_timestamp.py) -- TEST
INFRASTRUCTURE ONLY.

Per sample: the flow at each event interpolated bilinearly from the node grid in f64 (differentiable in the nodes), with
the node cell and weights and the keep and floor decisions taken from the kernel's f32 arithmetic
(tests/grid_flow_reference.py), then the per-polarity timestamp images, blur and loss of
tests/flow_timestamp_reference.py."""
import numpy as np
import torch

import flow_objective_reference as FR
import grid_flow_reference as GR

f32 = np.float32


def reference(x, y, d, tau, p, offsets, grid, H, W, sigma):
    """f (B,) f64 torch (differentiable in `grid`, a (B,2,gh,gw) f64 tensor), T and C (B,2,H+1,W+1), polarity 0
    positive.  x, y, d, tau, p: f32 numpy arrays as the kernel receives them (d = t - t0 of each event's sample);
    offsets: B+1 ints."""
    B, _, gh, gw = grid.shape
    Hc, Wc = H + 1, W + 1
    My, Mx = (torch.from_numpy(FR.blur_matrix(n, sigma)) for n in (Hc, Wc))
    fs, Ts, Cs = [], [], []
    n = x.shape[0]
    for b in range(B):
        lo, hi = max(int(offsets[b]), 0), min(int(offsets[b + 1]), n)
        sl = slice(lo, max(lo, hi))
        xb, yb, db, ub, pb = x[sl], y[sl], d[sl], tau[sl], p[sl]
        u32, v32 = GR.event_flow_f32(xb, yb, grid[b].detach().numpy(), H, W)
        with np.errstate(all="ignore"):
            xw32, yw32 = (xb + u32 * db).astype(f32), (yb + v32 * db).astype(f32)
        keep, finite = FR.keep_mask(xw32, yw32, H, W)
        imgs, cnts = [], []
        for sel in (pb > 0, pb <= 0):
            k = np.flatnonzero(keep & sel)
            if k.size:
                rows, cols, w, _ = GR.node_taps(xb[k], yb[k], gh, gw, H, W)
                wt = torch.from_numpy(w.astype(np.float64))
                r, c = torch.from_numpy(rows), torch.from_numpy(cols)
                dk = torch.from_numpy(db[k].astype(np.float64))
                xw = torch.from_numpy(xb[k].astype(np.float64)) + (grid[b, 0][r, c] * wt).sum(1) * dk
                yw = torch.from_numpy(yb[k].astype(np.float64)) + (grid[b, 1][r, c] * wt).sum(1) * dk
                px = torch.from_numpy(np.floor(xw32[k]).astype(np.int64))
                py = torch.from_numpy(np.floor(yw32[k]).astype(np.int64))
                dx, dy = xw - px.double(), yw - py.double()
                S = FR.splat(px, py, dx, dy, torch.from_numpy(ub[k].astype(np.float64)), Hc, Wc)
                C = 1 + FR.splat(px, py, dx, dy, torch.ones(k.size, dtype=torch.float64), Hc, Wc)
            else:
                S = torch.zeros((Hc, Wc), dtype=torch.float64) + 0 * grid[b].sum()
                C = torch.ones((Hc, Wc), dtype=torch.float64)
            T = S / C
            if not finite.all():
                T, C = T + float("nan"), C + float("nan")
            imgs.append(T)
            cnts.append(C)
        T = torch.stack(imgs)
        G = My @ T @ Mx.T
        fs.append((G * G).sum())
        Ts.append(T)
        Cs.append(torch.stack(cnts))
    return torch.stack(fs), torch.stack(Ts), torch.stack(Cs)
