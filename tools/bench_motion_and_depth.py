"""The joint motion-and-depth contrast loss (contrast_max/motion_and_depth.py) beside the depth-grid loss on the same
events, on the workloads of tools/bench_depth_grid.py (64 x 30 k events at 180 x 240, 16 x 500 k at 480 x 640): the
forward, forward + joint backward beside the depth grid's forward + node backward, one J = 8 joint candidates pass and
a whole motion_and_depth_fit_torch with its defaults (3 x 4, 6 x 8, 12 x 16 nodes).  Every function is warmed up on its
shape before it is timed with device events; the losses alternate within each of three rounds, so the rounds give the
spread.  The depth grid is 12 x 16 nodes.

Then the recovery table of tests/test_gpu_motion_and_depth.py (the three scenes of tests/test_gpu_depth_grid.py, started
with w off by 0.1 rad/s per axis and v turned by 10 degrees): the remaining w and heading errors as fractions of the
start's, the median relative rho error of the joint fit, of depth_grid_fit_torch at the wrong start and at the truth,
and F against depth_grid_fit_torch's F at the truth; with --sweep, at other scales and smoothness, which is how the
fit's defaults were chosen.

    python tools/bench_motion_and_depth.py [--reps 10] [--warmup 2] [--rounds 3] [--recovery-runs 3] [--sweep]

Prints the card's name and power limit, then one JSON line per round, workload and loss with median milliseconds, then
one JSON line per recovery run."""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from event_utils_b200.contrast_max import (camera_motion_warp, depth_grid_contrast_objective_torch,  # noqa: E402
                                           motion_and_depth_contrast_candidates_torch,
                                           motion_and_depth_contrast_objective_torch, motion_and_depth_fit_torch)

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_camera_motion import WORKLOADS, make  # noqa: E402
from bench_cmax_motion_objective import card  # noqa: E402
from bench_planar_motion import timed  # noqa: E402

GRID = (12, 16)


def speed(a):
    for rnd in range(a.rounds):
        for B, n, H, W, intr in WORKLOADS:
            xs, ys, ts, ps, _, motion = make(B, n, H, W)
            ev = [torch.tensor(v, device="cuda", dtype=torch.float32 if i != 2 else torch.float64)
                  for i, v in enumerate((xs, ys, ts, ps))]
            ends = torch.arange(1, B + 1, device="cuda") * n
            warp = camera_motion_warp(intr)
            kw = dict(img_size=(H, W), batch_end_indices=ends)
            mt = torch.tensor(motion, device="cuda")
            grid = torch.from_numpy(np.random.default_rng(1).uniform(0.125, 1.0, (B,) + GRID)).cuda()
            scales = torch.linspace(0.8, 1.2, 8, device="cuda", dtype=torch.float64)
            gcand = grid.unsqueeze(1) * scales[:, None, None]
            mcand = mt.unsqueeze(1) * scales[:, None]

            def joint_f():
                with torch.no_grad():
                    motion_and_depth_contrast_objective_torch(*ev, grid, mt, warp, **kw)

            def joint_fb():
                g, m = grid.clone().requires_grad_(True), mt.clone().requires_grad_(True)
                motion_and_depth_contrast_objective_torch(*ev, g, m, warp, **kw).sum().backward()

            def joint_cand():
                motion_and_depth_contrast_candidates_torch(*ev, mcand, gcand, warp, **kw)

            def joint_fit():
                motion_and_depth_fit_torch(*ev, warp, x0=mt, inv_depth_range=(0.05, 2.0), **kw)

            def grid_fb():
                g = grid.clone().requires_grad_(True)
                depth_grid_contrast_objective_torch(*ev, g, mt, warp, **kw).sum().backward()

            for kind, fns in (("motion_and_depth", (("forward_ms", joint_f), ("fb_ms", joint_fb),
                                                    ("candidates_j8_ms", joint_cand), ("fit_ms", joint_fit))),
                              ("depth_grid", (("fb_ms", grid_fb),))):
                row = {"round": rnd, "windows": B, "events_per_window": n, "H": H, "W": W, "loss": kind}
                for name, fn in fns:
                    reps, warmup = (max(1, a.reps // 5), 1) if name == "fit_ms" else (a.reps, a.warmup)
                    med, lo, hi = timed(fn, reps, warmup)
                    row[name] = round(med, 3)
                    row[name.replace("_ms", "_range_ms")] = [round(lo, 3), round(hi, 3)]
                print(json.dumps(row), flush=True)
            del ev


def accuracy(a):
    import test_gpu_motion_and_depth as T
    settings = [{}]
    if a.sweep:
        settings += [dict(rotation_scale=r, direction_scale=s) for r in (0.02, 0.05, 0.2) for s in (0.02, 0.05, 0.2)]
        settings += [dict(smoothness=s) for s in (1e-3, 1e-1)]
    for opts in settings:
        for run in range(a.recovery_runs if not opts else 1):
            r = T.recovery(**({"opts": opts} if opts else {}))
            print(json.dumps({"settings": opts or "defaults", "run": run,
                              **{k: [round(float(x), 5) for x in v] for k, v in r.items()}}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--recovery-runs", type=int, default=3)
    ap.add_argument("--sweep", action="store_true")
    ap.add_argument("--skip-speed", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_motion_and_depth needs a GPU")
    print("card:", card())
    if not a.skip_speed:
        speed(a)
    accuracy(a)


if __name__ == "__main__":
    main()
