"""The camera-motion model (camera_motion_warp, K = 6, with an inverse depth per event) beside camera_rotation_warp (K = 3)
and homography_warp (K = 8) on the same events: forward + backward of the batched contrast loss and of the batched
timestamp loss, and one contrast candidates pass at J = 8.  Every window's motion is an angular velocity w, with a linear
velocity v for the camera motion; the homography gets the first-order embedding of w
(tests/camera_rotation_reference.embedding_matrix).  The models alternate within each of three rounds, so the rounds give
the spread.

Then the recovery table of tests/test_gpu_camera_motion.py on its scene with depth (6 windows, points 1-8 m away,
|w| = 1.4-3.6 rad/s, |v| = 1.6-2.7 m/s, 180 x 240, 50 ms): the w error of a camera_rotation_warp fit from a grid
search, and the w and v errors of the camera_motion_warp fit started from it with v = 0, for both losses.

    python tools/bench_camera_motion.py [--reps 10] [--warmup 2] [--rounds 3]

Prints the card's name and power limit, then one JSON line per round, workload and model with median milliseconds, then
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

import camera_rotation_reference as CR  # noqa: E402
from event_utils_b200.contrast_max import (camera_motion_warp, camera_rotation_warp, homography_warp,  # noqa: E402
                                           motion_contrast_candidates_torch, motion_contrast_objective_torch,
                                           motion_timestamp_objective_torch)

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_cmax_motion_objective import card  # noqa: E402
from bench_planar_motion import timed  # noqa: E402

# (windows, events per window, H, W, (fx, fy, cx, cy))
WORKLOADS = [(64, 30000, 180, 240, (199.1, 198.7, 132.1, 110.8)), (16, 500000, 480, 640, (530.0, 528.0, 322.0, 238.0))]


def make(B, n, H, W, seed=0):
    """B windows of n events in the sensor, t in [0, 0.05] per window, inverse depths in [1/8, 1] per metre, and one
    (w, v) per window"""
    rng = np.random.default_rng(seed)
    xs = (rng.random((B, n)) * (W - 1)).reshape(-1)
    ys = (rng.random((B, n)) * (H - 1)).reshape(-1)
    ts = (np.sort(rng.random((B, n)), axis=1) * 0.05 + np.arange(B)[:, None] * 0.05).reshape(-1)
    ps = (rng.integers(0, 2, (B, n)) * 2.0 - 1.0).reshape(-1)
    rho = rng.uniform(0.125, 1.0, B * n)
    return xs, ys, ts, ps, rho, np.column_stack((rng.uniform(-6, 6, (B, 3)), rng.uniform(-2, 2, (B, 3))))


def models(motion, intr):
    cx, cy = intr[2:]
    hom = motion[:, :3] @ CR.embedding_matrix(intr).T
    return [("camera_motion", camera_motion_warp(intr), motion), ("camera_rotation", camera_rotation_warp(intr), motion[:, :3]),
            ("homography", homography_warp(center=(cx, cy)), hom)]


def speed(a):
    for rnd in range(a.rounds):
        for B, n, H, W, intr in WORKLOADS:
            xs, ys, ts, ps, rho, motion = make(B, n, H, W)
            ev = [torch.tensor(v, device="cuda", dtype=torch.float32 if i != 2 else torch.float64)
                  for i, v in enumerate((xs, ys, ts, ps))]
            depth = torch.tensor(rho, device="cuda", dtype=torch.float32)
            ends = torch.arange(1, B + 1, device="cuda") * n
            for kind, warp, params in models(motion, intr):
                kw = dict(img_size=(H, W), batch_end_indices=ends)
                if kind == "camera_motion":
                    kw["inv_depth"] = depth
                base = torch.tensor(params, device="cuda")
                cand = base.unsqueeze(1) * torch.linspace(0.8, 1.2, 8, device="cuda", dtype=torch.float64)[:, None]

                def contrast():
                    prm = base.clone().requires_grad_(True)
                    motion_contrast_objective_torch(*ev, prm, warp, **kw).sum().backward()

                def timestamp():
                    prm = base.clone().requires_grad_(True)
                    motion_timestamp_objective_torch(*ev, prm, warp, **kw).sum().backward()

                def candidates():
                    motion_contrast_candidates_torch(*ev, cand, warp, **kw)

                row = {"round": rnd, "windows": B, "events_per_window": n, "H": H, "W": W, "model": kind, "K": warp.dims}
                for name, fn in (("contrast_fb_ms", contrast), ("timestamp_fb_ms", timestamp), ("candidates_j8_ms", candidates)):
                    med, lo, hi = timed(fn, a.reps, a.warmup)
                    row[name] = round(med, 3)
                    row[name.replace("_ms", "_range_ms")] = [round(lo, 3), round(hi, 3)]
                print(json.dumps(row), flush=True)
            del ev, depth


def accuracy():
    from test_gpu_camera_motion import TRUTHS, recover
    print("recovery on the scene with depth (|w - w_true| rad/s, |v - v_true| m/s):")
    print("| loss | window | |w_true| | |v_true| | rotation-only w | camera motion w | camera motion v |")
    print("|---|---|---|---|---|---|---|")
    for loss_name in ("contrast", "timestamp"):
        rot, got = recover(loss_name)
        for b, m in enumerate(TRUTHS):
            print("| %s | %d | %.2f | %.2f | %.4f | %.4f | %.4f |" % (
                loss_name, b, np.linalg.norm(m[:3]), np.linalg.norm(m[3:]), np.linalg.norm(rot[b] - m[:3]),
                np.linalg.norm(got[b, :3] - m[:3]), np.linalg.norm(got[b, 3:] - m[3:])), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_camera_motion needs a GPU")
    print("card:", card())
    speed(a)
    accuracy()


if __name__ == "__main__":
    main()
