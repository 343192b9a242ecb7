"""The grid-flow average-timestamp loss, its candidates pass and its fit (contrast_max/grid_flow_timestamp.py), against
what a user would otherwise write.

  (a) forward + backward of grid_flow_timestamp_objective_torch against the composed path F.interpolate(nodes,
      align_corners=True) -> flow_timestamp_objective_torch -> autograd, at the dense-flow loss's bench sizes and node
      grids 12x16 and 48x64; and each event pass alone (CUDA time from torch.profiler) against its floor of 20 bytes per
      event read at the HBM bandwidth of an H100 SXM (3.35 TB/s).
  (b) one candidates pass with J = 8 grids against 8 forward calls.
  (c) grid_flow_timestamp_fit_torch on synthetic windows (wall time, windows/s) against a per-window scipy loop on the
      same loss, stages, start and box for the first 16 windows (L-BFGS-B, scipy's BFGS with bounds).

    python tools/bench_grid_flow_timestamp.py [--reps 20] [--warmup 3] [--fit-windows 64]

Prints the card's name and power limit, then one JSON line per measurement."""
import argparse
import json
import os
import sys
import time

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_grid_flow import GRIDS, SIZES, card, fit_windows, kernel_ms, make, timed  # noqa: E402
from event_utils_b200.contrast_max import (charbonnier_smoothness, flow_timestamp_objective_torch,  # noqa: E402
                                           grid_flow_timestamp_candidates_torch, grid_flow_timestamp_fit_torch,
                                           grid_flow_timestamp_objective_torch)

SIGMA = 2.0
HBM_BYTES_PER_S = 3.35e12


def loss_tables(a):
    for B, n, H, W in SIZES:
        for grid in GRIDS:
            x, y, t, p, nodes, ends = make(B, n, H, W, grid)
            nd = nodes.clone().requires_grad_(True)

            def fused():
                nd.grad = None
                f = grid_flow_timestamp_objective_torch(x, y, t, p, nd, (H, W), blur_sigma=SIGMA, batch_end_indices=ends)
                f.sum().backward()
                return f

            def comp():
                nd.grad = None
                dense = F.interpolate(nd, (H, W), mode="bilinear", align_corners=True)
                f = flow_timestamp_objective_torch(x, y, t, p, dense, blur_sigma=SIGMA, batch_end_indices=ends)
                f.sum().backward()
                return f

            f1, g1 = fused().detach(), nd.grad.clone()
            f2, g2 = comp().detach(), nd.grad.clone()
            ms_f = timed(fused, a.reps, a.warmup)
            ms_c = timed(comp, a.reps, a.warmup)
            k = kernel_ms(fused, ("grid_flow_cand_kernel", "grid_flow_grad_kernel"), a.reps)
            floor_ms = 20.0 * B * n / HBM_BYTES_PER_S * 1e3
            print(json.dumps({"table": "a", "batch": B, "events_per_window": n, "H": H, "W": W, "grid": list(grid),
                              "grid_fwd_bwd_ms": round(ms_f, 3), "composed_fwd_bwd_ms": round(ms_c, 3),
                              "speedup": round(ms_c / ms_f, 2),
                              "forward_event_pass_ms": round(k["grid_flow_cand_kernel"], 3),
                              "backward_event_pass_ms": round(k["grid_flow_grad_kernel"], 3),
                              "event_pass_floor_ms": round(floor_ms, 3),
                              "f_max_rel_diff": float(((f1 - f2).abs() / f2.abs()).max()),
                              "grad_max_rel_diff": float((g1 - g2).abs().max() / g2.abs().max())}), flush=True)
            if grid == GRIDS[0]:
                J = 8
                cand = nodes.unsqueeze(1) * torch.linspace(0.5, 1.5, J, device="cuda").view(1, J, 1, 1, 1)

                def one_pass():
                    return grid_flow_timestamp_candidates_torch(x, y, t, p, cand, (H, W), blur_sigma=SIGMA,
                                                                batch_end_indices=ends)

                def forwards():
                    return torch.stack([grid_flow_timestamp_objective_torch(x, y, t, p, cand[:, j], (H, W),
                                                                            blur_sigma=SIGMA, batch_end_indices=ends)
                                        for j in range(J)], 1)

                ms_p = timed(one_pass, a.reps, a.warmup)
                with torch.no_grad():
                    ms_s = timed(forwards, a.reps, a.warmup)
                print(json.dumps({"table": "b", "batch": B, "events_per_window": n, "H": H, "W": W, "grid": list(grid),
                                  "candidates": J, "one_pass_ms": round(ms_p, 3), "forward_calls_ms": round(ms_s, 3),
                                  "speedup": round(ms_s / ms_p, 2)}), flush=True)


def scipy_fit(x, y, t, p, H, W, shapes, lam, max_iter, box):
    """scipy L-BFGS-B per stage on one window, the same loss, stages, start (zero) and box"""
    from scipy.optimize import minimize
    flow = torch.zeros((1, 2) + shapes[0], dtype=torch.float64, device="cuda")
    for gh, gw in shapes:
        flow = F.interpolate(flow, (gh, gw), mode="bilinear", align_corners=True)

        def fun(v):
            g = torch.from_numpy(v).cuda().view(1, 2, gh, gw).requires_grad_(True)
            f = grid_flow_timestamp_objective_torch(x, y, t, p, g, (H, W), blur_sigma=SIGMA)
            R, dR = charbonnier_smoothness(g.detach(), 1.0)
            f.sum().backward()
            return float(f.item() + lam * R.item()), (g.grad + lam * dR).cpu().numpy().reshape(-1)
        r = minimize(fun, flow.cpu().numpy().reshape(-1), jac=True, method="L-BFGS-B", bounds=[box] * (2 * gh * gw),
                     options={"maxiter": max_iter})
        flow = torch.from_numpy(r.x).cuda().view(1, 2, gh, gw)
    return r.fun


def fit_table(a):
    H, W, n = 180, 240, 30000
    shapes = ((3, 4), (6, 8), (12, 16))
    lam, max_iter, box = 1e-2, 30, (-100.0, 100.0)
    ev, ends = fit_windows(a.fit_windows, n, H, W)
    x0 = torch.zeros((a.fit_windows, 2, 3, 4), dtype=torch.float64, device="cuda")

    def gpu():
        return grid_flow_timestamp_fit_torch(*ev, (H, W), grid_shapes=shapes, smoothness=lam, batch_end_indices=ends,
                                             x0=x0, bounds=[box, box], max_iter=max_iter, blur_sigma=SIGMA)
    gpu()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fit = gpu()
    torch.cuda.synchronize()
    t_gpu = time.perf_counter() - t0
    k = min(16, a.fit_windows)
    t0 = time.perf_counter()
    fs = [scipy_fit(*(c[b * n:(b + 1) * n] for c in ev), H, W, shapes, lam, max_iter, box) for b in range(k)]
    t_cpu = time.perf_counter() - t0
    print(json.dumps({"table": "c", "windows": a.fit_windows, "events_per_window": n, "H": H, "W": W,
                      "grid_shapes": [list(s) for s in shapes], "max_iter_per_stage": max_iter,
                      "fit_s": round(t_gpu, 3), "windows_per_s": round(a.fit_windows / t_gpu, 1),
                      "scipy_windows": k, "scipy_s": round(t_cpu, 3), "scipy_windows_per_s": round(k / t_cpu, 2),
                      "speedup_per_window": round((t_cpu / k) / (t_gpu / a.fit_windows), 1),
                      "fit_F_first": float(fit.f[0]), "scipy_F_first": fs[0],
                      "fit_F_le_scipy_windows": int(sum(float(fit.f[b]) <= fs[b] + 1e-9 * abs(fs[b]) for b in range(k)))}),
          flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--fit-windows", type=int, default=64)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a GPU")
    print("card: %s" % card(), flush=True)
    loss_tables(a)
    fit_table(a)


if __name__ == "__main__":
    main()
