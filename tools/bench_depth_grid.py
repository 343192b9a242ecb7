"""The depth-grid contrast loss (contrast_max/depth_grid.py) beside the per-event-rho camera_motion_warp loss on the same
events, on the workloads of tools/bench_camera_motion.py: forward + backward of both losses, one J = 8 candidates pass of
each, and a whole depth_grid_fit_torch with its defaults (3 x 4, 6 x 8, 12 x 16 nodes).  The losses alternate within each
of three rounds, so the rounds give the spread.  The depth grid is 12 x 16 nodes.

Then the recovery table of tests/test_gpu_depth_grid.py (a slanted plane, a step between two planes, a slanted plane
seen with a forward component of v; 180 x 240, 50 ms, rho 0.2-1 per metre): the median relative error of the fitted
rho at the scene's points, of the best constant inverse depth, and, with --sweep, of the fit at other smoothness and
Charbonnier eps values, which is how the fit's defaults were chosen.

    python tools/bench_depth_grid.py [--reps 10] [--warmup 2] [--rounds 3] [--sweep]

Prints the card's name and power limit, then one JSON line per round, workload and loss with median milliseconds, then
the recovery table."""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from event_utils_b200.contrast_max import (camera_motion_warp, depth_grid_contrast_candidates_torch,  # noqa: E402
                                           depth_grid_contrast_objective_torch, depth_grid_fit_torch,
                                           motion_contrast_candidates_torch, motion_contrast_objective_torch)

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_camera_motion import WORKLOADS, make  # noqa: E402
from bench_cmax_motion_objective import card  # noqa: E402
from bench_planar_motion import timed  # noqa: E402

GRID = (12, 16)


def speed(a):
    for rnd in range(a.rounds):
        for B, n, H, W, intr in WORKLOADS:
            xs, ys, ts, ps, rho, motion = make(B, n, H, W)
            ev = [torch.tensor(v, device="cuda", dtype=torch.float32 if i != 2 else torch.float64)
                  for i, v in enumerate((xs, ys, ts, ps))]
            depth = torch.tensor(rho, device="cuda", dtype=torch.float32)
            ends = torch.arange(1, B + 1, device="cuda") * n
            warp = camera_motion_warp(intr)
            kw = dict(img_size=(H, W), batch_end_indices=ends)
            mt = torch.tensor(motion, device="cuda")
            grid = torch.from_numpy(np.random.default_rng(1).uniform(0.125, 1.0, (B,) + GRID)).cuda()
            scales = torch.linspace(0.8, 1.2, 8, device="cuda", dtype=torch.float64)
            gcand = grid.unsqueeze(1) * scales[:, None, None]
            mcand = mt.unsqueeze(1) * scales[:, None]

            def grid_fb():
                g = grid.clone().requires_grad_(True)
                depth_grid_contrast_objective_torch(*ev, g, mt, warp, **kw).sum().backward()

            def grid_cand():
                depth_grid_contrast_candidates_torch(*ev, gcand, mt, warp, **kw)

            def grid_fit():
                depth_grid_fit_torch(*ev, mt, warp, inv_depth_range=(0.05, 2.0), **kw)

            def event_fb():
                m = mt.clone().requires_grad_(True)
                motion_contrast_objective_torch(*ev, m, warp, inv_depth=depth, **kw).sum().backward()

            def event_cand():
                motion_contrast_candidates_torch(*ev, mcand, warp, inv_depth=depth, **kw)

            for kind, fns in (("depth_grid", (("fb_ms", grid_fb), ("candidates_j8_ms", grid_cand), ("fit_ms", grid_fit))),
                              ("camera_motion_per_event_rho", (("fb_ms", event_fb), ("candidates_j8_ms", event_cand)))):
                row = {"round": rnd, "windows": B, "events_per_window": n, "H": H, "W": W, "loss": kind}
                for name, fn in fns:
                    reps, warmup = (max(1, a.reps // 5), 1) if name == "fit_ms" else (a.reps, a.warmup)
                    med, lo, hi = timed(fn, reps, warmup)
                    row[name] = round(med, 3)
                    row[name.replace("_ms", "_range_ms")] = [round(lo, 3), round(hi, 3)]
                print(json.dumps(row), flush=True)
            del ev, depth


def accuracy(sweep):
    from test_gpu_depth_grid import RANGE, SCENE_INTR, SCENES, median_errors, recovery_windows
    (x, y, t, p), ends, motion, truth = recovery_windows()
    ev = [torch.from_numpy(a).cuda() for a in (x, y, t, p)]
    kw = dict(batch_end_indices=torch.from_numpy(ends).cuda())
    mt = torch.from_numpy(motion).cuda()
    warp = camera_motion_warp(SCENE_INTR)
    consts = np.linspace(RANGE[0], RANGE[1], 32)
    cand = torch.from_numpy(np.broadcast_to(consts[None, :, None, None], (len(SCENES), 32, 3, 4)).copy()).cuda()
    best = consts[depth_grid_contrast_candidates_torch(*ev, cand, mt, warp, (180, 240), **kw).cpu().numpy().argmin(1)]
    print("median relative rho error at the scene's points (windows: slanted plane, two planes, plane with forward v):")
    print("| fit | " + " | ".join("window %d" % b for b in range(len(SCENES))) + " |")
    print("|---|" + "---|" * len(SCENES))
    print("| best constant | " + " | ".join("%.4f" % float(np.median(np.abs(best[b] - r) / r))
                                           for b, (_, _, r) in enumerate(truth)) + " |")
    settings = [{}]
    if sweep:
        settings += [dict(smoothness=s, charbonnier_eps=e) for s in (0.0, 1e-3, 1e-2, 1e-1) for e in (0.01, 0.05, 0.2)]
        settings += [dict(num_samples=n, grid_levels=lv) for n, lv in ((9, 1), (15, 1), (9, 2))]
    for opts in settings:
        fit = depth_grid_fit_torch(*ev, mt, warp, (180, 240), RANGE, **kw, **opts)
        err = median_errors(fit.inv_depth.cpu().numpy(), truth)
        print("| %s | " % (opts or "defaults") + " | ".join("%.4f" % e for e in err) + " |", flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--sweep", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_depth_grid needs a GPU")
    print("card:", card())
    speed(a)
    accuracy(a.sweep)


if __name__ == "__main__":
    main()
