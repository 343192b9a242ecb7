"""Batched motion fit (motion_contrast_fit_torch) against a per-window scipy BFGS loop and a 300-step Adam loop on the
batched loss, on synthetic windows with a known motion each.

    python tools/bench_motion_fit.py [--scipy-windows 16] [--out DIR]

Rows (DESIGN.md section 6):
    rotation  256 windows x 30 k events, 180x240, grid 5^3, one level, blur (2, 1)
    linvel   1024 windows x 10 k events, grid 5^2, two levels
    4-DoF      64 windows x 100 k events, from x0 within 15 % of the truth
The scipy path runs on the first --scipy-windows windows only (it takes seconds per window); its windows/s is over those.
Every path starts from the same point: the fit's grid-search result where the fit searches a grid.  Times are wall
times that end in a device synchronise.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from event_utils_b200.contrast_max import (linvel_warp, motion_contrast_fit_torch, motion_contrast_objective_torch,  # noqa: E402
                                           pure_rotation_warp, xyztheta_warp)
from event_utils_b200.contrast_max.motion_fit import _grid_search  # noqa: E402
from event_utils_b200.contrast_max.motion_objective import _candidates  # noqa: E402
from event_utils_b200.contrast_max._batched import _batch_events, _model  # noqa: E402

CENTRE = (120.0, 90.0)


def _scene(rng, n_pts, per_pt, centre, radius):
    ang, rad = rng.uniform(0, 2 * np.pi, n_pts), radius * np.sqrt(rng.uniform(0.05, 1, n_pts))
    x0, y0 = np.repeat(centre[0] + rad * np.cos(ang), per_pt), np.repeat(centre[1] + rad * np.sin(ang), per_pt)
    ps = np.repeat(rng.integers(0, 2, n_pts) * 2.0 - 1.0, per_pt)
    order = rng.permutation(x0.size)
    return x0[order], y0[order], ps[order]


def windows(kind, truths, duration, rng, n_pts, per_pt):
    """one window per true motion: a scene of points seen during `duration`, moving with that motion"""
    xs, ys, ts, ps, ends = [], [], [], [], []
    for tr in truths:
        centre = (tr[0], tr[1]) if kind == "rotation" else CENTRE
        x0, y0, p = _scene(rng, n_pts, per_pt, centre, 60.0)
        t = np.sort(rng.uniform(0, duration, x0.size))
        dt = t - t[-1]
        if kind == "linvel":
            x, y = x0 + dt * tr[0], y0 + dt * tr[1]
        elif kind == "rotation":
            a = tr[2] * dt
            u, v = x0 - tr[0], y0 - tr[1]
            x, y = tr[0] + np.cos(a) * u - np.sin(a) * v, tr[1] + np.sin(a) * u + np.cos(a) * v
        else:
            hx, hy, hz, th = tr
            bx, by = (x0 - CENTRE[0]) + dt * hx, (y0 - CENTRE[1]) + dt * hy
            m00, m01, m10, m11 = 1 - dt * hz, dt * th, -dt * th, 1 - dt * hz
            det = m00 * m11 - m01 * m10
            x, y = CENTRE[0] + (m11 * bx - m01 * by) / det, CENTRE[1] + (m00 * by - m10 * bx) / det
        xs.append(x), ys.append(y), ts.append(t), ps.append(p)
        ends.append(sum(len(a) for a in xs))
    return [np.concatenate(a) for a in (xs, ys, ts, ps)], ends


def truths_of(kind, rng, B):
    s = lambda: rng.choice([-1, 1], B)
    if kind == "linvel":
        return np.column_stack((rng.uniform(20, 60, B) * s(), rng.uniform(20, 60, B) * s())), 0.2
    if kind == "rotation":
        return np.column_stack((rng.uniform(110, 130, B), rng.uniform(80, 100, B), rng.uniform(3, 8, B) * s())), 0.05
    return np.column_stack((rng.uniform(15, 30, B) * s(), rng.uniform(15, 30, B) * s(), rng.uniform(2, 4, B),
                            rng.uniform(2, 4, B) * s())), 0.2


def recovered(kind, got, truths):
    if kind == "rotation":
        return (np.abs(got[:, 2] - truths[:, 2]) <= 0.03 * np.abs(truths[:, 2])) & \
            (np.hypot(got[:, 0] - truths[:, 0], got[:, 1] - truths[:, 1]) <= 2.0)
    return np.all(np.abs(got - truths) <= 0.05 * np.abs(truths), axis=1)


WARPS = {"linvel": linvel_warp, "rotation": pure_rotation_warp, "xyztheta": lambda: xyztheta_warp(center=CENTRE)}
SCALE = {"linvel": [1.0, 1.0], "rotation": [0.5, 0.5, 0.05], "xyztheta": [1.0, 1.0, 0.1, 0.1]}
ROWS = [
    dict(kind="rotation", B=256, n_pts=300, per_pt=100, fit=dict(param_ranges=[[105.0, 135.0], [75.0, 105.0], [-10.0, 10.0]],
                                                               num_samples_per_param=5, grid_levels=1, blur_sigma=(2.0, 1.0))),
    dict(kind="linvel", B=1024, n_pts=100, per_pt=100, fit=dict(param_ranges=[[-80.0, 80.0], [-80.0, 80.0]],
                                                              num_samples_per_param=5, grid_levels=2, blur_sigma=1.0)),
    dict(kind="xyztheta", B=64, n_pts=500, per_pt=200, fit=dict(blur_sigma=1.0)),
]


def timed(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, time.perf_counter() - t


def run_row(row, scipy_windows):
    import scipy.optimize as opt
    kind, B = row["kind"], row["B"]
    rng = np.random.default_rng({"rotation": 1, "linvel": 2, "xyztheta": 3}[kind])
    truths, duration = truths_of(kind, rng, B)
    (x, y, t, p), ends = windows(kind, truths, duration, rng, row["n_pts"], row["per_pt"])
    ev = [torch.from_numpy(a).float().cuda() for a in (x, y)] + [torch.from_numpy(t).cuda(), torch.from_numpy(p).float().cuda()]
    ends_d = torch.tensor(ends, device="cuda")
    warp = WARPS[kind]()
    kw = dict(row["fit"])
    if "param_ranges" in kw:
        kw["param_ranges"] = torch.tensor(kw["param_ranges"], device="cuda")
    else:
        start = truths * (1 + rng.uniform(-0.15, 0.15, truths.shape))
        kw["x0"] = torch.tensor(start, device="cuda")
        kw["param_scale"] = SCALE[kind]
    sigmas = kw["blur_sigma"] if isinstance(kw["blur_sigma"], tuple) else (kw["blur_sigma"],)
    motion_contrast_fit_torch(*ev, warp, batch_end_indices=ends_d, **kw)               # warm-up
    fit, t_fit = timed(lambda: motion_contrast_fit_torch(*ev, warp, batch_end_indices=ends_d, **kw))
    # the common start of the other paths: x0, or the fit's own grid-search result
    if "x0" in kw:
        start = kw["x0"]
    else:
        xd, yd, td, pd, off = _batch_events(*ev, None, ends_d, B, ev[0].device, "windows")
        opts = _model(_code(kind), warp, "variance", sigmas[0], None, 180, 240)
        ranges = kw["param_ranges"].to(torch.float64).unsqueeze(0).expand(B, -1, -1).contiguous()
        start = _grid_search(lambda c: _candidates(xd, yd, td, pd, off, c, opts), ranges, kw["num_samples_per_param"],
                             kw["grid_levels"], False)
    f_fit = fit.f.cpu().numpy()
    got_fit = fit.params.cpu().numpy()
    # per-window scipy BFGS from the same start, at each stage's blur
    S = min(scipy_windows, B)
    e = [0] + list(ends)
    f_sp, got_sp = np.empty(S), np.empty((S, truths.shape[1]))
    t0 = time.perf_counter()
    for b in range(S):
        wev = [a[e[b]:e[b + 1]] for a in ev]
        q = start[b].cpu().numpy()
        for sigma in sigmas:
            def fun(v):
                prm = torch.tensor(v, device="cuda", requires_grad=True)
                f = motion_contrast_objective_torch(*wev, prm, warp, blur_sigma=sigma)
                f.sum().backward()
                return f.item(), prm.grad.cpu().numpy()
            res = opt.minimize(fun, q, jac=True, method="BFGS")
            q = res.x
        f_sp[b], got_sp[b] = res.fun, res.x
    torch.cuda.synchronize()
    t_sp = time.perf_counter() - t0
    # Adam, 300 steps with a cosine schedule on the summed loss, from the same start (the existing test's loop)
    s = torch.tensor(SCALE[kind], device="cuda", dtype=torch.float64)

    def adam():
        base = start.clone().to(torch.float64)
        z = torch.zeros_like(base, requires_grad=True)
        o = torch.optim.Adam([z], lr=0.3)
        sch = torch.optim.lr_scheduler.CosineAnnealingLR(o, T_max=300, eta_min=0.003)
        for _ in range(300):
            o.zero_grad()
            f = motion_contrast_objective_torch(*ev, base + s * z, warp, blur_sigma=sigmas[-1], batch_end_indices=ends_d)
            f.sum().backward()
            o.step()
            sch.step()
        return (base + s * z).detach()
    got_adam, t_adam = timed(adam)
    f_adam = motion_contrast_objective_torch(*ev, got_adam, warp, blur_sigma=sigmas[-1], batch_end_indices=ends_d).cpu().numpy()
    got_adam = got_adam.cpu().numpy()
    rel = lambda a, b: float(np.max(np.abs(a - b) / np.maximum(np.abs(b), 1e-30)))
    return {"kind": kind, "windows": B, "events_per_window": row["n_pts"] * row["per_pt"],
            "fit": {"s": t_fit, "windows_per_s": B / t_fit, "recovered": float(recovered(kind, got_fit, truths).mean()),
                    "status_counts": np.bincount(fit.status.cpu().numpy(), minlength=4).tolist()},
            "scipy": {"windows": S, "s": t_sp, "windows_per_s": S / t_sp,
                      "recovered": float(recovered(kind, got_sp, truths[:S]).mean()),
                      "max_rel_df_fit_vs_scipy": rel(f_fit[:S], f_sp),
                      "fit_minus_scipy_max": float(np.max(f_fit[:S] - f_sp))},
            "adam": {"s": t_adam, "windows_per_s": B / t_adam, "recovered": float(recovered(kind, got_adam, truths).mean()),
                     "max_rel_df_fit_vs_adam": rel(f_fit, f_adam), "fit_minus_adam_max": float(np.max(f_fit - f_adam))}}


def _code(kind):
    from event_utils_b200 import _lib
    return {"linvel": _lib.WARP_LINVEL, "rotation": _lib.WARP_ROTATION, "xyztheta": _lib.WARP_XYZTHETA}[kind]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scipy-windows", type=int, default=16)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    print("card: %s" % card)
    rows = []
    for row in ROWS:
        r = run_row(row, a.scipy_windows)
        r["card"] = card
        print(json.dumps(r))
        rows.append(r)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_motion_fit.json"), "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
