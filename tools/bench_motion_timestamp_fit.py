"""Batched fit of the average-timestamp loss (motion_timestamp_fit_torch) against a per-window scipy BFGS loop and a
300-step Adam loop on the batched loss, on the synthetic windows of tools/bench_motion_fit.py; and one candidates pass
of B x 32 candidates against 32 calls of the batched forward.

    python tools/bench_motion_timestamp_fit.py [--scipy-windows 16] [--out DIR]

Rows (DESIGN.md section 6), 180x240, blur 2 (the loss's default):
    rotation  256 windows x 30 k events, grid 5^3, one level
    linvel   1024 windows x 10 k events, grid 5^2, two levels
    4-DoF      64 windows x 100 k events, from x0 within 15 % of the truth, bounded to +-30 % of it
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
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_motion_fit import SCALE, WARPS, _code, recovered, timed, truths_of, windows  # noqa: E402
from event_utils_b200.contrast_max import (motion_timestamp_candidates_torch, motion_timestamp_fit_torch,  # noqa: E402
                                           motion_timestamp_objective_torch)
from event_utils_b200.contrast_max._batched import _timestamp_events, _ts_model  # noqa: E402
from event_utils_b200.contrast_max.motion_fit import _grid_search  # noqa: E402
from event_utils_b200.contrast_max.motion_timestamp_objective import _ts_candidates  # noqa: E402

SIGMA = 2.0
ROWS = [
    dict(kind="rotation", B=256, n_pts=300, per_pt=100, fit=dict(param_ranges=[[105.0, 135.0], [75.0, 105.0], [-10.0, 10.0]],
                                                               num_samples_per_param=5, grid_levels=1)),
    dict(kind="linvel", B=1024, n_pts=100, per_pt=100, fit=dict(param_ranges=[[-80.0, 80.0], [-80.0, 80.0]],
                                                              num_samples_per_param=5, grid_levels=2)),
    dict(kind="xyztheta", B=64, n_pts=500, per_pt=200, fit=dict()),
]


def candidates_pass(kind, ev, ends_d, warp, start, rng, reps=5):
    """one pass of B x 32 candidates against 32 calls of the batched forward (no autograd graph), same values"""
    B, K = start.shape
    cand = start.unsqueeze(1) * (1 + 0.05 * torch.tensor(rng.uniform(-1, 1, (B, 32, K)), device="cuda"))
    one = lambda: motion_timestamp_candidates_torch(*ev, cand, warp, blur_sigma=SIGMA, batch_end_indices=ends_d)

    def each():
        with torch.no_grad():
            return torch.stack([motion_timestamp_objective_torch(*ev, cand[:, j], warp, blur_sigma=SIGMA,
                                                                 batch_end_indices=ends_d) for j in range(32)], 1)
    one(), each()
    f1, t1 = timed(lambda: [one() for _ in range(reps)][-1])
    f2, t2 = timed(lambda: [each() for _ in range(reps)][-1])
    rel = float(((f1 - f2).abs() / f2.abs().clamp_min(1e-30)).max())
    return {"candidates_pass_ms": 1e3 * t1 / reps, "forward_x32_ms": 1e3 * t2 / reps, "max_rel_diff": rel}


def run_row(row, scipy_windows):
    import scipy.optimize as opt
    kind, B = row["kind"], row["B"]
    rng = np.random.default_rng({"rotation": 1, "linvel": 2, "xyztheta": 3}[kind])
    truths, duration = truths_of(kind, rng, B)
    (x, y, t, p), ends = windows(kind, truths, duration, rng, row["n_pts"], row["per_pt"])
    ev = [torch.from_numpy(a).float().cuda() for a in (x, y)] + [torch.from_numpy(t).cuda(), torch.from_numpy(p).float().cuda()]
    ends_d = torch.tensor(ends, device="cuda")
    warp = WARPS[kind]()
    kw = dict(row["fit"], blur_sigma=SIGMA)
    if "param_ranges" in kw:
        kw["param_ranges"] = torch.tensor(kw["param_ranges"], device="cuda")
        lo, hi = (np.tile(kw["param_ranges"][:, i].cpu().numpy(), (B, 1)) for i in (0, 1))
    else:
        start = truths * (1 + rng.uniform(-0.15, 0.15, truths.shape))
        half = np.maximum(0.3 * np.abs(start), 1.0)
        lo, hi = start - half, start + half
        kw["x0"] = torch.tensor(start, device="cuda")
        kw["bounds"] = torch.tensor(np.stack((lo, hi), -1), device="cuda")
        kw["param_scale"] = SCALE[kind]
    motion_timestamp_fit_torch(*ev, warp, batch_end_indices=ends_d, **kw)               # warm-up
    fit, t_fit = timed(lambda: motion_timestamp_fit_torch(*ev, warp, batch_end_indices=ends_d, **kw))
    if "x0" in kw:
        start = kw["x0"]
    else:
        xd, yd, td, tau, pd, off = _timestamp_events(*ev, None, ends_d, B, ev[0].device, "windows", False)
        opts = _ts_model(_code(kind), warp, SIGMA, 180, 240)
        ranges = kw["param_ranges"].to(torch.float64).unsqueeze(0).expand(B, -1, -1).contiguous()
        start = _grid_search(lambda c: _ts_candidates(xd, yd, td, tau, pd, off, c, opts), ranges, kw["num_samples_per_param"],
                             kw["grid_levels"], False)
    f_fit = fit.f.cpu().numpy()
    got_fit = fit.params.cpu().numpy()
    S = min(scipy_windows, B)
    e = [0] + list(ends)
    f_sp, got_sp = np.empty(S), np.empty((S, truths.shape[1]))
    t0 = time.perf_counter()
    for b in range(S):
        wev = [a[e[b]:e[b + 1]] for a in ev]

        def fun(v):
            prm = torch.tensor(v, device="cuda", requires_grad=True)
            f = motion_timestamp_objective_torch(*wev, prm, warp, blur_sigma=SIGMA)
            f.sum().backward()
            return f.item(), prm.grad.cpu().numpy()
        res = opt.minimize(fun, start[b].cpu().numpy(), jac=True, method="BFGS")
        f_sp[b], got_sp[b] = res.fun, res.x
    torch.cuda.synchronize()
    t_sp = time.perf_counter() - t0
    s = torch.tensor(SCALE[kind], device="cuda", dtype=torch.float64)

    def adam():
        base = start.clone().to(torch.float64)
        z = torch.zeros_like(base, requires_grad=True)
        o = torch.optim.Adam([z], lr=0.3)
        sch = torch.optim.lr_scheduler.CosineAnnealingLR(o, T_max=300, eta_min=0.003)
        for _ in range(300):
            o.zero_grad()
            f = motion_timestamp_objective_torch(*ev, base + s * z, warp, blur_sigma=SIGMA, batch_end_indices=ends_d)
            f.sum().backward()
            o.step()
            sch.step()
        return (base + s * z).detach()
    got_adam, t_adam = timed(adam)
    f_adam = motion_timestamp_objective_torch(*ev, got_adam, warp, blur_sigma=SIGMA, batch_end_indices=ends_d).cpu().numpy()
    got_adam = got_adam.cpu().numpy()
    inside = lambda g: float(np.all((g >= lo[:len(g)]) & (g <= hi[:len(g)]), axis=1).mean())
    rel = lambda a, b: float(np.max(np.abs(a - b) / np.maximum(np.abs(b), 1e-30)))
    return {"kind": kind, "windows": B, "events_per_window": row["n_pts"] * row["per_pt"],
            "fit": {"s": t_fit, "windows_per_s": B / t_fit, "recovered": float(recovered(kind, got_fit, truths).mean()),
                    "status_counts": np.bincount(fit.status.cpu().numpy(), minlength=4).tolist()},
            "scipy": {"windows": S, "s": t_sp, "windows_per_s": S / t_sp,
                      "recovered": float(recovered(kind, got_sp, truths[:S]).mean()), "inside_bounds": inside(got_sp),
                      "max_rel_df_fit_vs_scipy": rel(f_fit[:S], f_sp), "fit_minus_scipy_max": float(np.max(f_fit[:S] - f_sp))},
            "adam": {"s": t_adam, "windows_per_s": B / t_adam, "recovered": float(recovered(kind, got_adam, truths).mean()),
                     "inside_bounds": inside(got_adam), "max_rel_df_fit_vs_adam": rel(f_fit, f_adam),
                     "fit_minus_adam_max": float(np.max(f_fit - f_adam))},
            "pass": candidates_pass(kind, ev, ends_d, warp, start.to(torch.float64), rng)}


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
        print(json.dumps(r), flush=True)
        rows.append(r)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_motion_timestamp_fit.json"), "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
