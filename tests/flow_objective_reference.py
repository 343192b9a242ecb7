"""f64 torch reference of the batched dense-flow contrast objective (contrast_max/flow_objective.py) -- TEST
INFRASTRUCTURE ONLY.

Per sample: the warp of tests/autograd_ports.warp_events_flow_torch in f64 (differentiable in the flow), the keep
decision 0 <= x' < W, 0 <= y' < H and the floor of x', y' taken from the kernel's f32 warp (as tests/grad_reference.py
takes discrete decisions from the forward's f32 arithmetic), a bilinear splat of p on the (H+1, W+1) canvas, the blur as
two dense f64 matrices (scipy's gaussian_filter1d, mode reflect, truncate 4, applied to identity columns) and the
objective.  Autograd through it gives the exact derivative the backward kernel implements."""
import numpy as np
import scipy.ndimage
import torch

from autograd_ports import warp_events_flow_torch

f32 = np.float32


def warp_f32(x, y, d, flow):
    """The kernel's f32 warp (flow_sample in csrc/evk_cmax.cu), op by op: x', y' as float32 arrays."""
    x, y, d = (np.asarray(a, f32) for a in (x, y, d))
    flow = np.asarray(flow, f32)
    H, W = flow.shape[1], flow.shape[2]
    wm1, hm1 = f32(W - 1), f32(H - 1)
    with np.errstate(all="ignore"):
        ix = ((x / wm1 * f32(2) - f32(1)) + f32(1)) / f32(2) * wm1
        iy = ((y / hm1 * f32(2) - f32(1)) + f32(1)) / f32(2) * hm1
        ok = (np.abs(ix) < f32(1e9)) & (np.abs(iy) < f32(1e9))
        fx, fy = np.floor(np.where(ok, ix, 0)).astype(f32), np.floor(np.where(ok, iy, 0)).astype(f32)
        x0, y0 = fx.astype(np.int64), fy.astype(np.int64)
        wx1, wx0, wy1, wy0 = (fx + f32(1)) - ix, ix - fx, (fy + f32(1)) - iy, iy - fy
        u, v = np.zeros_like(x), np.zeros_like(x)
        for dy_, dx_, w in ((0, 0, wx1 * wy1), (0, 1, wx0 * wy1), (1, 0, wx1 * wy0), (1, 1, wx0 * wy0)):
            yy, xx = y0 + dy_, x0 + dx_
            inside = ok & (yy >= 0) & (yy < H) & (xx >= 0) & (xx < W)
            fu = np.where(inside, flow[0][np.clip(yy, 0, H - 1), np.clip(xx, 0, W - 1)], f32(0))
            fv = np.where(inside, flow[1][np.clip(yy, 0, H - 1), np.clip(xx, 0, W - 1)], f32(0))
            u = np.where(ok, u + fu * w, u).astype(f32)
            v = np.where(ok, v + fv * w, v).astype(f32)
        return (x + u * d).astype(f32), (y + v * d).astype(f32)


def keep_mask(xw, yw, H, W):
    """The keep rule on the f32 warped positions; non-finite positions are reported separately."""
    finite = np.isfinite(xw) & np.isfinite(yw)
    with np.errstate(invalid="ignore"):
        keep = finite & (xw >= 0) & (xw < f32(W)) & (yw >= 0) & (yw < f32(H))
    return keep, finite


def blur_matrix(n, sigma):
    """M with M @ a == scipy.ndimage.gaussian_filter1d(a, sigma, axis=0) (mode reflect, truncate 4), in f64."""
    if sigma <= 0:
        return np.eye(n)
    return scipy.ndimage.gaussian_filter1d(np.eye(n), sigma, axis=0, mode="reflect", truncate=4.0)


def splat(px, py, dx, dy, w, Hc, Wc):
    img = torch.zeros((Hc, Wc), dtype=torch.float64)
    img = img.index_put((py, px), w * (1 - dx) * (1 - dy), accumulate=True)
    img = img.index_put((py, px + 1), w * dx * (1 - dy), accumulate=True)
    img = img.index_put((py + 1, px), w * (1 - dx) * dy, accumulate=True)
    return img.index_put((py + 1, px + 1), w * dx * dy, accumulate=True)


def objective_of(G, name, param):
    P = G.numel()
    if name == "variance":
        return -((G - G.mean()) ** 2).mean()
    if name == "sos":
        return -(G * G).sum() / P
    if name == "soe":
        return -torch.exp(G).sum() / P
    if name == "sosa":
        return -torch.exp(-param * G).sum()
    raise ValueError(name)


def reference(x, y, d, p, offsets, flow, sigma, name, param=3.0):
    """f (B,) f64 torch (differentiable in `flow`, a (B,2,H,W) f64 tensor), the IWEs (B,H+1,W+1) and the images of
    the |p| splats (the per-pixel magnitudes of the IWE sums).  x, y, d, p: f32 numpy arrays
    (d = t - t0 of each event's sample, as the kernel receives it); offsets: B+1 ints."""
    B, _, H, W = flow.shape
    Hc, Wc = H + 1, W + 1
    My, Mx = (torch.from_numpy(blur_matrix(n, sigma)) for n in (Hc, Wc))
    fs, iwes, mags = [], [], []
    n = x.shape[0]
    for b in range(B):
        lo, hi = max(int(offsets[b]), 0), min(int(offsets[b + 1]), n)
        sl = slice(lo, max(lo, hi))
        xb, yb, db, pb = x[sl], y[sl], d[sl], p[sl]
        xw32, yw32 = warp_f32(xb, yb, db, flow[b].detach().numpy())
        keep, finite = keep_mask(xw32, yw32, H, W)
        k = np.flatnonzero(keep)
        if k.size:
            xw, yw = warp_events_flow_torch(torch.from_numpy(xb[k].astype(np.float64)), torch.from_numpy(yb[k].astype(np.float64)),
                                            torch.from_numpy(db[k].astype(np.float64)), None, flow[b].unsqueeze(0),
                                            t0=torch.zeros((), dtype=torch.float64))
            xw, yw = xw.reshape(-1), yw.reshape(-1)
            px = torch.from_numpy(np.floor(xw32[k]).astype(np.int64))
            py = torch.from_numpy(np.floor(yw32[k]).astype(np.int64))
            dx, dy = xw - px.double(), yw - py.double()
            pk = torch.from_numpy(pb[k].astype(np.float64))
            img = splat(px, py, dx, dy, pk, Hc, Wc)
            mag = splat(px, py, dx.detach(), dy.detach(), pk.abs(), Hc, Wc)
        else:
            img = torch.zeros((Hc, Wc), dtype=torch.float64) + 0 * flow[b].sum()
            mag = torch.zeros((Hc, Wc), dtype=torch.float64)
        if not finite.all():
            img = img + float("nan")
        G = My @ img @ Mx.T
        fs.append(objective_of(G, name, param))
        iwes.append(img)
        mags.append(mag)
    return torch.stack(fs), torch.stack(iwes), torch.stack(mags)


def grad_magnitude(x, y, d, p, offsets, flow, sigma, name, param, g, iwe, mag):
    """Per flow cell, the sum over the events that reach it of |d| w_tap |p| sum_4 Wmag (the magnitudes of the terms the
    backward adds there), with Wmag = blur(|g_b| Cmag) and Cmag the magnitude of df/dG including the error of G
    (blur of the |p| image): the scale of a per-cell error bound.  Also the number of terms per cell plus the largest
    number of events anchored at one IWE pixel (the summation lengths the bound's gamma() needs)."""
    B, _, H, W = flow.shape
    Hc, Wc = H + 1, W + 1
    My, Mx = blur_matrix(Hc, sigma), blur_matrix(Wc, sigma)
    P = Hc * Wc
    out = np.zeros((B, 2, H, W))
    cnt = np.zeros((B, 2, H, W))
    kI = 0
    n = x.shape[0]
    for b in range(B):
        lo, hi = max(int(offsets[b]), 0), min(int(offsets[b + 1]), n)
        G = My @ np.asarray(iwe[b], np.float64) @ Mx.T
        Ga = My @ np.asarray(mag[b], np.float64) @ Mx.T
        if name in ("variance", "sos"):
            C = 2 * (np.abs(G) + Ga) / P
        elif name == "soe":
            C = np.exp(G) * (1 + Ga) / P
        else:
            C = abs(param) * np.exp(-param * G) * (1 + abs(param) * Ga)
        Wm = My @ (abs(float(g[b])) * C) @ Mx.T
        if hi <= lo:
            continue
        xb, yb, db, pb = x[lo:hi], y[lo:hi], d[lo:hi], p[lo:hi]
        xw, yw = warp_f32(xb, yb, db, flow[b].detach().numpy())
        keep, _ = keep_mask(xw, yw, H, W)
        k = np.flatnonzero(keep)
        px, py = np.floor(xw[k]).astype(np.int64), np.floor(yw[k]).astype(np.int64)
        kI = max(kI, 4 * int(np.bincount(py * Wc + px, minlength=1).max(initial=0)))
        s = (Wm[py, px] + Wm[py, px + 1] + Wm[py + 1, px] + Wm[py + 1, px + 1]) * np.abs(pb[k]) * np.abs(db[k])
        ix, iy = xb[k].astype(np.float64), yb[k].astype(np.float64)
        fx, fy = np.floor(ix), np.floor(iy)
        for ddy, ddx in ((0, 0), (0, 1), (1, 0), (1, 1)):
            wx = (ix - fx) if ddx else (fx + 1 - ix)
            wy = (iy - fy) if ddy else (fy + 1 - iy)
            xx, yy = fx.astype(np.int64) + ddx, fy.astype(np.int64) + ddy
            ins = (xx >= 0) & (xx < W) & (yy >= 0) & (yy < H)
            for c in range(2):
                np.add.at(out[b, c], (yy[ins], xx[ins]), (s * wx * wy)[ins])
                np.add.at(cnt[b, c], (yy[ins], xx[ins]), 1.0)
    return out, cnt + kI
