"""f64 torch reference of the batched parametric average-timestamp loss (contrast_max/motion_timestamp_objective.py) --
TEST INFRASTRUCTURE ONLY.

Per sample: the contribute decision (finite, 0 < x' < W, 0 < y' < H) and the floor of x', y' taken from the f32
restatement of the kernel's warp (motion_objective_reference.warp_f32 / contributes), then the warp in f64
(motion_objective_reference.warp_f64, differentiable in the parameters), per polarity the bilinear sums S = sum tau k and
C = 1 + sum k on the (H+1, W+1) canvas (flow_objective_reference.splat), T = S / C, the blur as two dense f64 matrices
and f = sum G_+^2 + sum G_-^2.  Autograd through it gives the exact derivative the backward kernel implements."""
import numpy as np
import torch

from flow_objective_reference import blur_matrix, splat
from flow_timestamp_reference import tau_f32  # noqa: F401  (the stamps the kernel receives; re-exported for the tests)
from motion_objective_reference import DIMS, contributes, jacobian, warp_f32, warp_f64  # noqa: F401

CENTRE = (120.0, 90.0)


def reference(kind, x, y, d, tau, p, offsets, params, sigma, img_size=(180, 240), centre=CENTRE):
    """f (B,) f64 torch (differentiable in `params`, a (B,K) f64 tensor), T and C (B,2,H+1,W+1), polarity 0 positive.
    x, y, d, tau, p: f32 numpy arrays as the kernel receives them (d = t - t0 of each event's sample); offsets: B+1
    ints."""
    H, W = img_size
    Hc, Wc = H + 1, W + 1
    My, Mx = (torch.from_numpy(blur_matrix(n, sigma)) for n in (Hc, Wc))
    fs, Ts, Cs = [], [], []
    n = x.shape[0]
    for b in range(params.shape[0]):
        lo, hi = max(int(offsets[b]), 0), min(int(offsets[b + 1]), n)
        sl = slice(lo, max(lo, hi))
        xb, yb, db, ub, pb = x[sl], y[sl], d[sl], tau[sl], p[sl]
        xw32, yw32 = warp_f32(kind, xb, yb, db, params[b].detach().numpy(), centre)
        keep = contributes(xw32, yw32, H, W)
        imgs, cnts = [], []
        for sel in (pb > 0, pb <= 0):
            k = np.flatnonzero(keep & sel)
            if k.size:
                t64 = [torch.from_numpy(a[k].astype(np.float64)) for a in (xb, yb, db)]
                xw, yw = warp_f64(kind, *t64, params[b], centre)
                px = torch.from_numpy(np.floor(xw32[k]).astype(np.int64))
                py = torch.from_numpy(np.floor(yw32[k]).astype(np.int64))
                dx, dy = xw - px.double(), yw - py.double()
                S = splat(px, py, dx, dy, torch.from_numpy(ub[k].astype(np.float64)), Hc, Wc)
                C = 1 + splat(px, py, dx, dy, torch.ones(k.size, dtype=torch.float64), Hc, Wc)
            else:
                # in the graph, with a zero gradient even for NaN parameters (whose events all contribute nothing)
                S = torch.zeros((Hc, Wc), dtype=torch.float64) + 0 * torch.nan_to_num(params[b]).sum()
                C = torch.ones((Hc, Wc), dtype=torch.float64)
            imgs.append(S / C)
            cnts.append(C)
        T = torch.stack(imgs)
        G = My @ T @ Mx.T
        fs.append((G * G).sum())
        Ts.append(T)
        Cs.append(torch.stack(cnts))
    return torch.stack(fs), torch.stack(Ts), torch.stack(Cs)


def grad_magnitude(kind, x, y, d, tau, p, offsets, params, sigma, g, T, C, img_size=(180, 240), centre=CENTRE):
    """Per sample and component, the sum over the contributing events of (|dx'/dp_k| + |dy'/dp_k|) sum_4 Am (|tau| + Tm),
    the magnitudes of the terms the backward adds, with Am = blur(2 |g_b| 2 blur(|T|)) / C (twice |G|, to cover the
    error of G) and Tm = |T|: the scale of a per-component error bound.  Also the number of contributing events per
    sample plus the largest number of events anchored at one canvas pixel (the summation lengths the bound's gamma()
    needs)."""
    H, W = img_size
    Hc, Wc = H + 1, W + 1
    My, Mx = blur_matrix(Hc, sigma), blur_matrix(Wc, sigma)
    B, K = params.shape
    out, cnt = np.zeros((B, K)), np.zeros((B, K))
    n = x.shape[0]
    for b in range(B):
        lo, hi = max(int(offsets[b]), 0), min(int(offsets[b + 1]), n)
        if hi <= lo:
            continue
        prm = params[b].detach().numpy()
        xb, yb, db, ub, pb = x[lo:hi], y[lo:hi], d[lo:hi], tau[lo:hi], p[lo:hi]
        xw, yw = warp_f32(kind, xb, yb, db, prm, centre)
        keep = contributes(xw, yw, H, W)
        kI, total = 0, 0
        for s, sel in enumerate((pb > 0, pb <= 0)):
            Ts = np.abs(np.asarray(T[b, s], np.float64))
            Gm = My @ Ts @ Mx.T
            Am = (My @ (4 * abs(float(g[b])) * Gm) @ Mx.T) / np.asarray(C[b, s], np.float64)
            k = np.flatnonzero(keep & sel)
            if not k.size:
                continue
            px, py = np.floor(xw[k]).astype(np.int64), np.floor(yw[k]).astype(np.int64)
            kI = max(kI, 4 * int(np.bincount(py * Wc + px).max()))
            total += k.size
            uk = np.abs(ub[k]).astype(np.float64)
            s_ = np.zeros(k.size)
            for oy, ox in ((0, 0), (0, 1), (1, 0), (1, 1)):
                s_ += Am[py + oy, px + ox] * (uk + Ts[py + oy, px + ox])
            J = np.abs(jacobian(kind, xb[k], yb[k], db[k], prm, centre)).sum(axis=0).T      # (n, K)
            out[b] += (s_[:, None] * J).sum(axis=0)
        cnt[b] = total + kI
    return out, cnt


def rotating_scene(seed=5, n_pts=300, per_pt=100, centre=(120.0, 90.0), omega=6.0, duration=0.05, radius=60.0):
    """Points of a static scene seen by a camera rotating at omega about centre (image plane) during `duration`: the
    events of each point trace an arc that pure_rotation_warp (cx, cy, omega) with t0 = the last stamp undoes.  f64
    arrays x, y, t, p."""
    rng = np.random.default_rng(seed)
    ang, rad = rng.uniform(0, 2 * np.pi, n_pts), radius * np.sqrt(rng.uniform(0.05, 1, n_pts))
    x0, y0 = np.repeat(centre[0] + rad * np.cos(ang), per_pt), np.repeat(centre[1] + rad * np.sin(ang), per_pt)
    p = np.repeat(rng.integers(0, 2, n_pts) * 2.0 - 1.0, per_pt)
    order = rng.permutation(x0.size)
    x0, y0, p = x0[order], y0[order], p[order]
    t = np.sort(rng.uniform(0, duration, x0.size))
    a = omega * (t - t[-1])
    u, v = x0 - centre[0], y0 - centre[1]
    x, y = centre[0] + np.cos(a) * u - np.sin(a) * v, centre[1] + np.sin(a) * u + np.cos(a) * v
    return x, y, t, p
