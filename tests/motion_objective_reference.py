"""f64 torch reference of the batched parametric contrast objective (contrast_max/motion_objective.py) -- TEST
INFRASTRUCTURE ONLY.

Per sample: the keep decision (0 < x' < W, 0 < y' < H: the bounds mask 0 < x' <= W, then the clip of the splat, which
gives an event at x' = W zero weight) and the floor of x', y' taken from an f32 restatement of the kernel's warp
(model_taps in csrc/evk_cmax.cu, op by op, as tests/flow_objective_reference.py takes its decisions), then the warp in
f64 (differentiable in the parameters), a bilinear splat of p on the (H+1, W+1) canvas, the blur as two dense f64
matrices and the objective -- the splat, blur and objectives of tests/flow_objective_reference.py.  Autograd through it
gives the exact derivative the backward kernel implements."""
import numpy as np
import torch

from flow_objective_reference import blur_matrix, objective_of, splat

f32 = np.float32
DIMS = {"linvel": 2, "rotation": 3, "xyztheta": 4}


def warp_f32(kind, x, y, d, prm, centre=(120.0, 90.0)):
    """The kernel's f32 warp, op by op: x', y' as float32 arrays (prm: the model's parameters, cast to f32 like the
    kernel's (R)M.m[k])."""
    x, y, d = (np.asarray(a, f32) for a in (x, y, d))
    m = [f32(v) for v in prm]
    with np.errstate(all="ignore"):
        if kind == "linvel":
            return (x - d * m[0]).astype(f32), (y - d * m[1]).astype(f32)
        if kind == "rotation":
            cx, cy, om = m
            a = (om * d).astype(f32)
            s, c = np.sin(a).astype(f32), np.cos(a).astype(f32)      # sincosf: within an ulp of these
            u, v = (x - cx).astype(f32), (y - cy).astype(f32)
            return (cx + (c * u + s * v)).astype(f32), (cy + (c * v - s * u)).astype(f32)
        hx, hy, hz, th = m
        cx, cy = f32(centre[0]), f32(centre[1])
        u, v = (x - cx).astype(f32), (y - cy).astype(f32)
        return (x - d * ((hx + hz * u) - th * v)).astype(f32), (y - d * ((hy + hz * v) + th * u)).astype(f32)


def warp_f64(kind, x, y, d, prm, centre=(120.0, 90.0)):
    """The same warp in f64 torch, differentiable in prm (a (K,) f64 tensor)."""
    if kind == "linvel":
        return x - d * prm[0], y - d * prm[1]
    if kind == "rotation":
        cx, cy, om = prm[0], prm[1], prm[2]
        a = om * d
        c, s = torch.cos(a), torch.sin(a)
        u, v = x - cx, y - cy
        return cx + (c * u + s * v), cy + (c * v - s * u)
    hx, hy, hz, th = prm[0], prm[1], prm[2], prm[3]
    u, v = x - centre[0], y - centre[1]
    return x - d * ((hx + hz * u) - th * v), y - d * ((hy + hz * v) + th * u)


def contributes(xw, yw, H, W):
    """The events whose splat is not zero: finite, 0 < x' < W and 0 < y' < H in f32."""
    with np.errstate(invalid="ignore"):
        return np.isfinite(xw) & np.isfinite(yw) & (xw > 0) & (xw < f32(W)) & (yw > 0) & (yw < f32(H))


def reference(kind, x, y, d, p, offsets, params, sigma, name, param=3.0, img_size=(180, 240), centre=(120.0, 90.0)):
    """f (B,) f64 torch (differentiable in `params`, a (B,K) f64 tensor), the IWEs (B,H+1,W+1) and the images of the
    |p| splats.  x, y, d, p: f32 numpy arrays (d = t - t0 of each event's sample, as the kernel receives it);
    offsets: B+1 ints."""
    H, W = img_size
    Hc, Wc = H + 1, W + 1
    My, Mx = (torch.from_numpy(blur_matrix(n, sigma)) for n in (Hc, Wc))
    fs, iwes, mags = [], [], []
    n = x.shape[0]
    for b in range(params.shape[0]):
        lo, hi = max(int(offsets[b]), 0), min(int(offsets[b + 1]), n)
        sl = slice(lo, max(lo, hi))
        xb, yb, db, pb = x[sl], y[sl], d[sl], p[sl]
        xw32, yw32 = warp_f32(kind, xb, yb, db, params[b].detach().numpy(), centre)
        k = np.flatnonzero(contributes(xw32, yw32, H, W))
        if k.size:
            t64 = [torch.from_numpy(a[k].astype(np.float64)) for a in (xb, yb, db)]
            xw, yw = warp_f64(kind, *t64, params[b], centre)
            px = torch.from_numpy(np.floor(xw32[k]).astype(np.int64))
            py = torch.from_numpy(np.floor(yw32[k]).astype(np.int64))
            dx, dy = xw - px.double(), yw - py.double()
            pk = torch.from_numpy(pb[k].astype(np.float64))
            img = splat(px, py, dx, dy, pk, Hc, Wc)
            mag = splat(px, py, dx.detach(), dy.detach(), pk.abs(), Hc, Wc)
        else:
            img = torch.zeros((Hc, Wc), dtype=torch.float64) + 0 * params[b].sum()
            mag = torch.zeros((Hc, Wc), dtype=torch.float64)
        G = My @ img @ Mx.T
        fs.append(objective_of(G, name, param))
        iwes.append(img)
        mags.append(mag)
    return torch.stack(fs), torch.stack(iwes), torch.stack(mags)


def grad_magnitude(kind, x, y, d, p, offsets, params, sigma, name, param, g, iwe, mag, img_size=(180, 240),
                   centre=(120.0, 90.0)):
    """Per sample and component, the sum over the kept events of |p| (|jx_k| + |jy_k|) sum_4 Wmag (the magnitudes of the
    terms the backward adds), with Wmag = blur(|g_b| Cmag) and Cmag the magnitude of df/dG including the error of G: the
    scale of a per-component error bound.  Also the number of kept events per sample plus the largest number of events
    anchored at one IWE pixel (the summation lengths the bound's gamma() needs)."""
    H, W = img_size
    Hc, Wc = H + 1, W + 1
    My, Mx = blur_matrix(Hc, sigma), blur_matrix(Wc, sigma)
    P = Hc * Wc
    B, K = params.shape
    out, cnt = np.zeros((B, K)), np.zeros((B, K))
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
        prm = params[b].detach().numpy()
        xb, yb, db, pb = x[lo:hi], y[lo:hi], d[lo:hi], p[lo:hi]
        xw, yw = warp_f32(kind, xb, yb, db, prm, centre)
        k = np.flatnonzero(contributes(xw, yw, H, W))
        if not k.size:
            continue
        px, py = np.floor(xw[k]).astype(np.int64), np.floor(yw[k]).astype(np.int64)
        kI = 4 * int(np.bincount(py * Wc + px).max())
        s = (Wm[py, px] + Wm[py, px + 1] + Wm[py + 1, px] + Wm[py + 1, px + 1]) * np.abs(pb[k])
        J = np.abs(jacobian(kind, xb[k], yb[k], db[k], prm, centre)).sum(axis=0).T      # (n, K): |dx'/dp_k| + |dy'/dp_k|
        out[b] = (s[:, None] * J).sum(axis=0)
        cnt[b] = k.size + kI
    return out, cnt


def jacobian(kind, x, y, d, prm, centre=(120.0, 90.0)):
    """(2, K, n) f64 rows dx'/dp_k, dy'/dp_k (the closed forms of contrast_max/warps.py)"""
    x, y, d = (np.asarray(a, np.float64) for a in (x, y, d))
    z = np.zeros_like(d)
    if kind == "linvel":
        return np.array([[-d, z], [z, -d]])
    if kind == "rotation":
        cx, cy, om = (float(v) for v in prm)
        a = om * d
        c, s = np.cos(a), np.sin(a)
        u, v = x - cx, y - cy
        return np.array([[1 - c, -s, d * (c * v - s * u)], [s, 1 - c, -d * (c * u + s * v)]])
    u, v = x - centre[0], y - centre[1]
    return np.array([[-d, z, -d * u, d * v], [z, -d, -d * v, -d * u]])
