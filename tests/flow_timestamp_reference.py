"""f64 torch reference of the batched dense-flow average-timestamp loss (contrast_max/flow_timestamp_objective.py) --
TEST INFRASTRUCTURE ONLY.

Per sample: the warp of tests/autograd_ports.warp_events_flow_torch in f64 (differentiable in the flow), the keep
decision 0 <= x' < W, 0 <= y' < H and the floor of x', y' taken from the kernel's f32 warp (flow_objective_reference),
per polarity the bilinear sums S = sum tau k and C = 1 + sum k on the (H+1, W+1) canvas, T = S / C, the blur as two
dense f64 matrices and f = sum G_+^2 + sum G_-^2.  Autograd through it gives the exact derivative the backward kernel
implements."""
import numpy as np
import torch

from autograd_ports import warp_events_flow_torch
from flow_objective_reference import blur_matrix, keep_mask, splat, warp_f32

f32 = np.float32


def tau_f32(t, offsets, reverse=False):
    """evk_tsimg.cu's normalised stamp per sample, op by op in f32: denom = (t_last - t_first) + 1e-6f, then
    (t - t_first) / denom or (-t + t_last) / denom."""
    t = np.asarray(t, f32)
    out = np.empty_like(t)
    for b in range(len(offsets) - 1):
        lo, hi = int(offsets[b]), int(offsets[b + 1])
        if hi <= lo:
            continue
        tf, tl = t[lo], t[hi - 1]
        den = f32(f32(tl - tf) + f32(1e-6))
        num = (-t[lo:hi] + tl) if reverse else (t[lo:hi] - tf)
        out[lo:hi] = (num.astype(f32) / den).astype(f32)
    return out


def reference(x, y, d, tau, p, offsets, flow, sigma):
    """f (B,) f64 torch (differentiable in `flow`, a (B,2,H,W) f64 tensor), T and C (B,2,H+1,W+1), polarity 0 positive.
    x, y, d, tau, p: f32 numpy arrays as the kernel receives them (d = t - t0 of each event's sample); offsets: B+1 ints."""
    B, _, H, W = flow.shape
    Hc, Wc = H + 1, W + 1
    My, Mx = (torch.from_numpy(blur_matrix(n, sigma)) for n in (Hc, Wc))
    fs, Ts, Cs = [], [], []
    n = x.shape[0]
    for b in range(B):
        lo, hi = max(int(offsets[b]), 0), min(int(offsets[b + 1]), n)
        sl = slice(lo, max(lo, hi))
        xb, yb, db, ub, pb = x[sl], y[sl], d[sl], tau[sl], p[sl]
        xw32, yw32 = warp_f32(xb, yb, db, flow[b].detach().numpy())
        keep, finite = keep_mask(xw32, yw32, H, W)
        imgs, cnts = [], []
        for sel in (pb > 0, pb <= 0):
            k = np.flatnonzero(keep & sel)
            if k.size:
                xw, yw = warp_events_flow_torch(torch.from_numpy(xb[k].astype(np.float64)),
                                                torch.from_numpy(yb[k].astype(np.float64)),
                                                torch.from_numpy(db[k].astype(np.float64)), None, flow[b].unsqueeze(0),
                                                t0=torch.zeros((), dtype=torch.float64))
                xw, yw = xw.reshape(-1), yw.reshape(-1)
                px = torch.from_numpy(np.floor(xw32[k]).astype(np.int64))
                py = torch.from_numpy(np.floor(yw32[k]).astype(np.int64))
                dx, dy = xw - px.double(), yw - py.double()
                S = splat(px, py, dx, dy, torch.from_numpy(ub[k].astype(np.float64)), Hc, Wc)
                C = 1 + splat(px, py, dx, dy, torch.ones(k.size, dtype=torch.float64), Hc, Wc)
            else:
                S = torch.zeros((Hc, Wc), dtype=torch.float64) + 0 * flow[b].sum()
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


def grad_magnitude(x, y, d, tau, p, offsets, flow, sigma, g, T, C):
    """Per flow cell, the sum over the events that reach it of |d| w_tap sum_4 |dk/dx'| (|tau| Am + Tm Am), the
    magnitudes of the terms the backward adds there, with Am = blur(2 |g_b| 2 blur(T)) / C (twice |G|, to cover the
    error of G), Tm = T: the scale of a per-cell error bound.  Also the number of terms per cell plus the largest number
    of events anchored at one canvas pixel (the summation lengths the bound's gamma() needs)."""
    B, _, H, W = flow.shape
    Hc, Wc = H + 1, W + 1
    My, Mx = blur_matrix(Hc, sigma), blur_matrix(Wc, sigma)
    out = np.zeros((B, 2, H, W))
    cnt = np.zeros((B, 2, H, W))
    kI = 0
    n = x.shape[0]
    for b in range(B):
        lo, hi = max(int(offsets[b]), 0), min(int(offsets[b + 1]), n)
        if hi <= lo:
            continue
        xb, yb, db, ub, pb = x[lo:hi], y[lo:hi], d[lo:hi], tau[lo:hi], p[lo:hi]
        xw, yw = warp_f32(xb, yb, db, flow[b].detach().numpy())
        keep, _ = keep_mask(xw, yw, H, W)
        for s, sel in enumerate((pb > 0, pb <= 0)):
            Ts = np.abs(np.asarray(T[b, s], np.float64))
            Gm = My @ Ts @ Mx.T
            Am = (My @ (4 * abs(float(g[b])) * Gm) @ Mx.T) / np.asarray(C[b, s], np.float64)
            k = np.flatnonzero(keep & sel)
            if not k.size:
                continue
            px, py = np.floor(xw[k]).astype(np.int64), np.floor(yw[k]).astype(np.int64)
            kI = max(kI, 4 * int(np.bincount(py * Wc + px).max()))
            uk = np.abs(ub[k]).astype(np.float64)
            s_ = np.zeros(k.size)
            for oy, ox in ((0, 0), (0, 1), (1, 0), (1, 1)):
                s_ += Am[py + oy, px + ox] * (uk + Ts[py + oy, px + ox])
            s_ *= np.abs(db[k])
            ix, iy = xb[k].astype(np.float64), yb[k].astype(np.float64)
            fx, fy = np.floor(ix), np.floor(iy)
            for ddy, ddx in ((0, 0), (0, 1), (1, 0), (1, 1)):
                wx = (ix - fx) if ddx else (fx + 1 - ix)
                wy = (iy - fy) if ddy else (fy + 1 - iy)
                xx, yy = fx.astype(np.int64) + ddx, fy.astype(np.int64) + ddy
                ins = (xx >= 0) & (xx < W) & (yy >= 0) & (yy < H)
                for c in range(2):
                    np.add.at(out[b, c], (yy[ins], xx[ins]), (s_ * wx * wy)[ins])
                    np.add.at(cnt[b, c], (yy[ins], xx[ins]), 1.0)
    return out, cnt + kI


def edge_scene(seed=9, n=200000, H=120, W=160, u_true=(32.0, -21.0)):
    """Events of 24 line segments moving with the uniform flow u_true over 0.2 time units, sharp at the last stamp when
    warped by u_true (t0 = the last stamp); f64 arrays x, y, t, p."""
    rng = np.random.default_rng(seed)
    seg = rng.random((24, 4)) * [W - 40, H - 40, W - 40, H - 40] + 20
    s = rng.integers(0, 24, n)
    a = rng.random(n)
    x0 = seg[s, 0] + a * (seg[s, 2] - seg[s, 0])
    y0 = seg[s, 1] + a * (seg[s, 3] - seg[s, 1])
    t = np.sort(rng.random(n)) * 0.2
    dt = t - t[-1]
    x = x0 - u_true[0] * dt
    y = y0 - u_true[1] * dt
    p = np.where(rng.random(n) < 0.8, 1.0, -1.0)
    return x, y, t, p
