"""The depth-grid average-timestamp loss (contrast_max/depth_grid_timestamp.py) beside the per-event-rho camera_motion_warp
timestamp loss and the depth-grid contrast loss on the same events and (w, v), on the workloads of
tools/bench_camera_motion.py: forward + backward of each loss, one J = 8 candidates pass of each, and a whole
depth_grid_timestamp_fit_torch with its defaults (3 x 4, 6 x 8, 12 x 16 nodes).  The losses alternate within each of
three rounds, so the rounds give the spread.  The depth grids are 12 x 16 nodes.

Then the recovery table of tests/test_gpu_depth_grid.py's scenes (a slanted plane, a step between two planes, a slanted
plane seen with a forward component of v; 180 x 240, 50 ms, rho 0.2-1 per metre) for both fits side by side: the median
relative error of the fitted rho at the scene's points, the best constant inverse depth of each loss, and, with --sweep,
the timestamp fit at other smoothness and Charbonnier eps values, which is how its defaults were chosen.  Then, for both
fits, whether the box had to stop border nodes: the fit's line search rejects a point outside the box rather than
projecting it onto a face, so a node driven towards hi stops at its last accepted point inside the box.  So the table
gives the share of each window's nodes within 1 % of (hi - lo) of a face, the median relative error of the outer ring of
nodes and of the inner nodes against the true surface at the node pixels, and the share of the window's events warped
off the canvas at the fitted grid beside that share at the true-surface grid.

    python tools/bench_depth_grid_timestamp.py [--reps 10] [--warmup 2] [--rounds 3] [--sweep] [--no-speed]

Prints the card's name and power limit, then one JSON line per round, workload and loss with median milliseconds, then
the recovery tables."""
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
                                           depth_grid_timestamp_candidates_torch, depth_grid_timestamp_fit_torch,
                                           depth_grid_timestamp_objective_torch, motion_timestamp_candidates_torch,
                                           motion_timestamp_objective_torch)

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

            def ts_fb():
                g = grid.clone().requires_grad_(True)
                depth_grid_timestamp_objective_torch(*ev, g, mt, warp, **kw).sum().backward()

            def ts_cand():
                depth_grid_timestamp_candidates_torch(*ev, gcand, mt, warp, **kw)

            def ts_fit():
                depth_grid_timestamp_fit_torch(*ev, mt, warp, inv_depth_range=(0.05, 2.0), **kw)

            def event_fb():
                m = mt.clone().requires_grad_(True)
                motion_timestamp_objective_torch(*ev, m, warp, inv_depth=depth, **kw).sum().backward()

            def event_cand():
                motion_timestamp_candidates_torch(*ev, mcand, warp, inv_depth=depth, **kw)

            def contrast_fb():
                g = grid.clone().requires_grad_(True)
                depth_grid_contrast_objective_torch(*ev, g, mt, warp, **kw).sum().backward()

            def contrast_cand():
                depth_grid_contrast_candidates_torch(*ev, gcand, mt, warp, **kw)

            for kind, fns in (("depth_grid_timestamp", (("fb_ms", ts_fb), ("candidates_j8_ms", ts_cand),
                                                        ("fit_ms", ts_fit))),
                              ("camera_motion_timestamp_per_event_rho", (("fb_ms", event_fb),
                                                                         ("candidates_j8_ms", event_cand))),
                              ("depth_grid_contrast", (("fb_ms", contrast_fb), ("candidates_j8_ms", contrast_cand)))):
                row = {"round": rnd, "windows": B, "events_per_window": n, "H": H, "W": W, "loss": kind}
                for name, fn in fns:
                    reps, warmup = (max(1, a.reps // 5), 1) if name == "fit_ms" else (a.reps, a.warmup)
                    med, lo, hi = timed(fn, reps, warmup)
                    row[name] = round(med, 3)
                    row[name.replace("_ms", "_range_ms")] = [round(lo, 3), round(hi, 3)]
                print(json.dumps(row), flush=True)
            del ev, depth


def near_face(D, box, rel=0.01):
    """the share of each window's nodes within rel (hi - lo) of lo or hi"""
    lo, hi = box
    tol = rel * (hi - lo)
    return [float(np.mean((d - lo < tol) | (hi - d < tol))) for d in D]


def true_grids(scenes, intr, shape, H, W):
    """the scenes' true inverse depth at the node pixels of a (gh, gw) grid"""
    gh, gw = shape
    py, px = np.meshgrid(np.arange(gh) * (H - 1) / (gh - 1), np.arange(gw) * (W - 1) / (gw - 1), indexing="ij")
    return np.stack([surface(px, py, intr) for surface, _, _ in scenes])


def ring_errors(D, G):
    """median relative error of the outer ring of nodes and of the inner nodes of every window, against G"""
    ring = np.ones(D.shape[1:], bool)
    ring[1:-1, 1:-1] = False
    err = np.abs(D - G) / G
    return [(float(np.median(e[ring])), float(np.median(e[~ring]))) for e in err]


def off_canvas(D, x, y, t, ends, motion, intr, H, W):
    """the share of every window's events whose warp at the grid D (t0: the window's last stamp) is not kept"""
    import camera_motion_reference as CM
    import depth_grid_reference as DR
    from motion_objective_reference import contributes
    out, lo = [], 0
    for b, hi in enumerate(ends):
        xb, yb = x[lo:hi].astype(np.float32), y[lo:hi].astype(np.float32)
        d = (t[lo:hi] - t[hi - 1]).astype(np.float32)
        r = DR.event_rho_f32(xb, yb, D[b], H, W)
        xw, yw = CM.warp(xb, yb, d, r, motion[b, :3], motion[b, 3:], intr)
        out.append(float(1.0 - np.mean(contributes(xw, yw, H, W))))
        lo = hi
    return out


def accuracy(sweep):
    from test_gpu_depth_grid import RANGE, SCENE_INTR, SCENES, median_errors, recovery_windows
    (x, y, t, p), ends, motion, truth = recovery_windows()
    ev = [torch.from_numpy(a).cuda() for a in (x, y, t, p)]
    kw = dict(batch_end_indices=torch.from_numpy(ends).cuda())
    mt = torch.from_numpy(motion).cuda()
    warp = camera_motion_warp(SCENE_INTR)
    nw = len(SCENES)
    consts = np.linspace(RANGE[0], RANGE[1], 32)
    cand = torch.from_numpy(np.broadcast_to(consts[None, :, None, None], (nw, 32, 3, 4)).copy()).cuda()
    print("median relative rho error at the scene's points (windows: slanted plane, two planes, plane with forward v):")
    print("| fit | " + " | ".join("window %d" % b for b in range(nw)) + " |")
    print("|---|" + "---|" * nw)
    for name, fn in (("contrast", depth_grid_contrast_candidates_torch),
                     ("timestamp", depth_grid_timestamp_candidates_torch)):
        best = consts[fn(*ev, cand, mt, warp, (180, 240), **kw).cpu().numpy().argmin(1)]
        print("| best constant, %s loss | " % name + " | ".join("%.4f" % float(np.median(np.abs(best[b] - r) / r))
                                                              for b, (_, _, r) in enumerate(truth)) + " |")
    runs = [("contrast fit, defaults", depth_grid_fit_torch, {}),
            ("timestamp fit, defaults", depth_grid_timestamp_fit_torch, {})]
    if sweep:
        runs += [("timestamp fit, %s" % o, depth_grid_timestamp_fit_torch, o)
                 for o in [dict(smoothness=s, charbonnier_eps=e) for s in (0.0, 0.1, 1.0, 10.0, 100.0)
                           for e in (0.01, 0.05, 0.2)]]
    fits = {}
    for label, fit, opts in runs:
        D = fit(*ev, mt, warp, (180, 240), RANGE, **kw, **opts).inv_depth.cpu().numpy()
        fits.setdefault(label, D)
        print("| %s | " % label + " | ".join("%.4f" % e for e in median_errors(D, truth)) + " |", flush=True)
    G = true_grids(SCENES, SCENE_INTR, GRID, 180, 240)
    off_true = off_canvas(G, x, y, t, ends, motion, SCENE_INTR, 180, 240)
    print("\nthe box and the border nodes, per window: nodes within 1 %% of (hi - lo) of a face / median relative error "
          "of the outer ring / of the inner nodes / events off the canvas at the fit (at the true surface: %s):"
          % " / ".join("%.4f" % o for o in off_true))
    print("| fit | " + " | ".join("window %d" % b for b in range(nw)) + " |")
    print("|---|" + "---|" * nw)
    for label in ("contrast fit, defaults", "timestamp fit, defaults"):
        D = fits[label]
        cols = zip(near_face(D, RANGE), ring_errors(D, G), off_canvas(D, x, y, t, ends, motion, SCENE_INTR, 180, 240))
        print("| %s | " % label + " | ".join("%.2f / %.4f / %.4f / %.4f" % (f, r, i, o) for f, (r, i), o in cols) + " |",
              flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--sweep", action="store_true")
    ap.add_argument("--no-speed", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_depth_grid_timestamp needs a GPU")
    print("card:", card())
    if not a.no_speed:
        speed(a)
    accuracy(a.sweep)


if __name__ == "__main__":
    main()
