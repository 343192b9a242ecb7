"""f64 torch reference of the weighted multi-model contrast and of the assignment of contrast_max/motion_segmentation.py --
TEST INFRASTRUCTURE ONLY.

Per window b and model m: the keep decisions and floors of tests/motion_objective_reference.py under params[b, m]
(the kernel's f32 warp, op by op), the warp in f64 (differentiable in the parameters), a bilinear splat of p * w[:, m]
(differentiable in the weights) on the (H+1, W+1) canvas, the blur as two dense f64 matrices and the objective.
Autograd through it gives the exact derivatives the backward kernel implements."""
import numpy as np
import torch

import motion_objective_reference as R
from flow_objective_reference import blur_matrix, objective_of, splat


def reference(kind, x, y, d, p, w, offsets, params, sigma, name, param=3.0, img_size=(180, 240), centre=(120.0, 90.0)):
    """f (B,M) f64 torch, differentiable in params ((B,M,K) f64 tensor) and w ((N,M) f64 tensor), and the images
    (B,M,H+1,W+1).  x, y, d, p: f32 numpy arrays (d = t - t0 of each event's window); offsets: B+1 ints."""
    H, W = img_size
    Hc, Wc = H + 1, W + 1
    My, Mx = (torch.from_numpy(blur_matrix(n, sigma)) for n in (Hc, Wc))
    B, M, _ = params.shape
    n = x.shape[0]
    fs, imgs = [], []
    for b in range(B):
        lo, hi = max(int(offsets[b]), 0), min(int(offsets[b + 1]), n)
        lo, hi = lo, max(lo, hi)
        xb, yb, db, pb = x[lo:hi], y[lo:hi], d[lo:hi], p[lo:hi]
        for m in range(M):
            xw32, yw32 = R.warp_f32(kind, xb, yb, db, params[b, m].detach().numpy(), centre)
            k = np.flatnonzero(R.contributes(xw32, yw32, H, W))
            if k.size:
                t64 = [torch.from_numpy(a[k].astype(np.float64)) for a in (xb, yb, db)]
                xw, yw = R.warp_f64(kind, *t64, params[b, m], centre)
                px = torch.from_numpy(np.floor(xw32[k]).astype(np.int64))
                py = torch.from_numpy(np.floor(yw32[k]).astype(np.int64))
                wk = torch.from_numpy(pb[k].astype(np.float64)) * w[lo + torch.from_numpy(k), m]
                img = splat(px, py, xw - px.double(), yw - py.double(), wk, Hc, Wc)
            else:
                img = torch.zeros((Hc, Wc), dtype=torch.float64) + 0 * params[b, m].sum() + 0 * w[:, m].sum()
            fs.append(objective_of(My @ img @ Mx.T, name, param))
            imgs.append(img)
    return torch.stack(fs).reshape(B, M), torch.stack(imgs).reshape(B, M, Hc, Wc)


def assign(kind, x, y, d, offsets, params, iwe, sigma, eps, img_size=(180, 240), centre=(120.0, 90.0)):
    """(N,M) f64 memberships: c = max(0, sum_taps k G) with the bilinear fractions k of the f32 warp and the blurred
    images G of iwe (B,M,H+1,W+1), normalised with eps; rows outside every window 1/M"""
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
            xw, yw = R.warp_f32(kind, x[lo:hi], y[lo:hi], d[lo:hi], np.asarray(params[b, m]), centre)
            k = np.flatnonzero(R.contributes(xw, yw, H, W))
            px, py = np.floor(xw[k]).astype(np.int64), np.floor(yw[k]).astype(np.int64)
            dx, dy = xw[k].astype(np.float64) - px, yw[k].astype(np.float64) - py
            v = ((1 - dx) * (1 - dy) * G[py, px] + dx * (1 - dy) * G[py, px + 1] + (1 - dx) * dy * G[py + 1, px] +
                 dx * dy * G[py + 1, px + 1])
            c[k, m] = np.where(v < 0, 0.0, v)
        den = c.sum(1, keepdims=True) + M * eps
        with np.errstate(invalid="ignore", divide="ignore"):
            out[lo:hi] = np.where(den == 0, 1.0 / M, (c + eps) / den)
    return out
