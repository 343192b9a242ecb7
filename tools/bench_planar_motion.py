"""The planar motion models (affine_warp, K = 6; homography_warp, K = 8) beside xyztheta_warp (K = 4) on the same events:
forward + backward of the batched contrast loss (motion_contrast_objective_torch), forward + backward of the batched
timestamp loss (motion_timestamp_objective_torch), and a contrast fit (motion_contrast_fit_torch) from an x0 near each
window's motion.  The parameters are the embeddings of one xyztheta vector per window, (hx, hy, hz, -theta, theta, hz) and
g = (0.01, -0.01), so every model sees the same motion up to the homography's small projective part.

    python tools/bench_planar_motion.py [--reps 10] [--warmup 2] [--fit-iters 20]

Prints the card's name and power limit, then one JSON line per workload and model with the median milliseconds."""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from event_utils_b200.contrast_max import (affine_warp, homography_warp, motion_contrast_fit_torch,  # noqa: E402
                                           motion_contrast_objective_torch, motion_timestamp_objective_torch,
                                           xyztheta_warp)

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_cmax_motion_objective import card  # noqa: E402

# (windows, events per window, H, W)
WORKLOADS = [(64, 30000, 180, 240), (16, 500000, 480, 640)]


def make(B, n, H, W, seed=0):
    """B windows of n events in the sensor, t in [0, 0.05] per window, one xyztheta vector per window"""
    rng = np.random.default_rng(seed)
    xs = (rng.random((B, n)) * (W - 1)).reshape(-1)
    ys = (rng.random((B, n)) * (H - 1)).reshape(-1)
    ts = (np.sort(rng.random((B, n)), axis=1) * 0.05 + np.arange(B)[:, None] * 0.05).reshape(-1)
    ps = (rng.integers(0, 2, (B, n)) * 2.0 - 1.0).reshape(-1)
    xyz = np.column_stack((rng.uniform(-30, 30, (B, 2)), rng.uniform(-2, 2, (B, 2))))
    return xs, ys, ts, ps, xyz


def models(xyz, centre):
    hx, hy, hz, th = xyz.T
    aff = np.column_stack((hx, hy, hz, -th, th, hz))
    hom = np.column_stack((aff, np.full(len(hx), 0.01), np.full(len(hx), -0.01)))
    return [("xyztheta", xyztheta_warp(center=centre), xyz), ("affine", affine_warp(center=centre), aff),
            ("homography", homography_warp(center=centre), hom)]


def timed(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        out.append(a.elapsed_time(b))
    return float(np.median(out)), float(np.min(out)), float(np.max(out))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--fit-iters", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_planar_motion needs a GPU")
    print("card:", card())
    for B, n, H, W in WORKLOADS:
        xs, ys, ts, ps, xyz = make(B, n, H, W)
        ev = [torch.tensor(v, device="cuda", dtype=torch.float32 if i != 2 else torch.float64)
              for i, v in enumerate((xs, ys, ts, ps))]
        ends = torch.arange(1, B + 1, device="cuda") * n
        for kind, warp, params in models(xyz, (W / 2, H / 2)):
            base = torch.tensor(params, device="cuda")
            kw = dict(img_size=(H, W), batch_end_indices=ends)

            def contrast():
                prm = base.clone().requires_grad_(True)
                motion_contrast_objective_torch(*ev, prm, warp, **kw).sum().backward()

            def timestamp():
                prm = base.clone().requires_grad_(True)
                motion_timestamp_objective_torch(*ev, prm, warp, **kw).sum().backward()

            start = base * 1.1

            def fit():
                motion_contrast_fit_torch(*ev, warp, x0=start, max_iter=a.fit_iters, **kw)

            row = {"windows": B, "events_per_window": n, "H": H, "W": W, "model": kind, "K": warp.dims}
            for name, fn, reps in (("contrast_fb_ms", contrast, a.reps), ("timestamp_fb_ms", timestamp, a.reps),
                                   ("contrast_fit_ms", fit, max(1, a.reps // 3))):
                med, lo, hi = timed(fn, reps, a.warmup)
                row[name] = round(med, 3)
                row[name.replace("_ms", "_range_ms")] = [round(lo, 3), round(hi, 3)]
            print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
