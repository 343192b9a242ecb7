"""f64 torch reference of the batched grid-flow contrast objective (contrast_max/grid_flow.py) -- TEST INFRASTRUCTURE ONLY.

Per sample: the flow at each event interpolated bilinearly from the node grid in f64 (differentiable in the nodes),
with the node cell and weights and the keep and floor decisions taken from the kernel's f32 arithmetic (node_sample and
flow_obj_keep in csrc/evk_cmax.cu), then the splat, blur and objectives of tests/flow_objective_reference.py."""
import numpy as np
import torch

import flow_objective_reference as FR

f32 = np.float32


def node_taps(x, y, gh, gw, H, W):
    """The kernel's f32 node cell of every event: the (N,4) node rows, columns, f32 weights (nw, ne, sw, se) and the
    inside mask of each tap"""
    x, y = np.asarray(x, f32), np.asarray(y, f32)
    rx, ry = f32(gw - 1) / f32(W - 1), f32(gh - 1) / f32(H - 1)
    with np.errstate(all="ignore"):
        ix, iy = x * rx, y * ry
        ok = (np.abs(ix) < f32(1e9)) & (np.abs(iy) < f32(1e9))
        ix, iy = np.where(ok, ix, f32(0)), np.where(ok, iy, f32(0))
        fx, fy = np.floor(ix).astype(f32), np.floor(iy).astype(f32)
        x0, y0 = fx.astype(np.int64), fy.astype(np.int64)
        xs, ys = fx + f32(1), fy + f32(1)
        w = np.stack(((xs - ix) * (ys - iy), (ix - fx) * (ys - iy), (xs - ix) * (iy - fy), (ix - fx) * (iy - fy)), 1).astype(f32)
    cols = np.stack((x0, x0 + 1, x0, x0 + 1), 1)
    rows = np.stack((y0, y0, y0 + 1, y0 + 1), 1)
    inside = ok[:, None] & (cols >= 0) & (cols < gw) & (rows >= 0) & (rows < gh)
    return np.clip(rows, 0, gh - 1), np.clip(cols, 0, gw - 1), np.where(inside, w, f32(0)), inside


def event_flow_f32(x, y, grid, H, W):
    """u, v of every event in the kernel's f32 order of terms (node_flow)"""
    g = np.asarray(grid, f32)
    rows, cols, w, inside = node_taps(x, y, g.shape[1], g.shape[2], H, W)
    u, v = np.zeros(len(rows), f32), np.zeros(len(rows), f32)
    for k in range(4):
        qu = np.where(inside[:, k], g[0][rows[:, k], cols[:, k]], f32(0))
        qv = np.where(inside[:, k], g[1][rows[:, k], cols[:, k]], f32(0))
        with np.errstate(all="ignore"):
            u = (u + qu * w[:, k]).astype(f32)
            v = (v + qv * w[:, k]).astype(f32)
    return u, v


def reference(x, y, d, p, offsets, grid, H, W, sigma, name, param=3.0):
    """f (B,) f64 torch (differentiable in `grid`, a (B,2,gh,gw) f64 tensor) and the IWEs (B,H+1,W+1).  x, y, d, p: f32
    numpy arrays (d = t - t0 of each event's sample, as the kernel receives it); offsets: B+1 ints."""
    B, _, gh, gw = grid.shape
    Hc, Wc = H + 1, W + 1
    My, Mx = (torch.from_numpy(FR.blur_matrix(n, sigma)) for n in (Hc, Wc))
    fs, iwes = [], []
    n = x.shape[0]
    for b in range(B):
        lo, hi = max(int(offsets[b]), 0), min(int(offsets[b + 1]), n)
        sl = slice(lo, max(lo, hi))
        xb, yb, db, pb = x[sl], y[sl], d[sl], p[sl]
        u32, v32 = event_flow_f32(xb, yb, grid[b].detach().numpy(), H, W)
        with np.errstate(all="ignore"):
            xw32, yw32 = (xb + u32 * db).astype(f32), (yb + v32 * db).astype(f32)
        keep, finite = FR.keep_mask(xw32, yw32, H, W)
        k = np.flatnonzero(keep)
        if k.size:
            rows, cols, w, _ = node_taps(xb[k], yb[k], gh, gw, H, W)
            wt = torch.from_numpy(w.astype(np.float64))
            r, c = torch.from_numpy(rows), torch.from_numpy(cols)
            u = (grid[b, 0][r, c] * wt).sum(1)
            v = (grid[b, 1][r, c] * wt).sum(1)
            dk = torch.from_numpy(db[k].astype(np.float64))
            xw = torch.from_numpy(xb[k].astype(np.float64)) + u * dk
            yw = torch.from_numpy(yb[k].astype(np.float64)) + v * dk
            px = torch.from_numpy(np.floor(xw32[k]).astype(np.int64))
            py = torch.from_numpy(np.floor(yw32[k]).astype(np.int64))
            img = FR.splat(px, py, xw - px.double(), yw - py.double(), torch.from_numpy(pb[k].astype(np.float64)), Hc, Wc)
        else:
            img = torch.zeros((Hc, Wc), dtype=torch.float64) + 0 * grid[b].sum()
        if not finite.all():
            img = img + float("nan")
        G = My @ img @ Mx.T
        fs.append(FR.objective_of(G, name, param))
        iwes.append(img)
    return torch.stack(fs), torch.stack(iwes)
