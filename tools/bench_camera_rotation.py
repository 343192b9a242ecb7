"""The camera-rotation model (camera_rotation_warp, K = 3) beside homography_warp (K = 8) and xyztheta_warp (K = 4) on the
same events: forward + backward of the batched contrast loss and of the batched timestamp loss, one contrast candidates
pass at J = 32, and a grid-started contrast fit of 256 windows.  Every window's motion is one angular velocity w; the
homography gets its first-order embedding K'[w]x K'^-1 (tests/camera_rotation_reference.embedding_matrix) and xyztheta
its translation and in-plane part (-fx wy, fy wx, 0, -wz).  The models alternate within each of three rounds, so the
rounds give the spread.

Then an accuracy table on the rotation scene of tests/test_gpu_camera_rotation.py (8 windows, |w| = 2.1 .. 7.8 rad/s,
180 x 240, 50 ms): the angular-velocity error of the camera fit (grid search over [-10, 10]^3, 3 levels, blur 4, 2, 1)
against the w read off a homography fit, which starts from the embedded xyztheta fit and whose w is the least-squares
projection of its 8 parameters onto the rotation subspace (the inverse of the embedding).

    python tools/bench_camera_rotation.py [--reps 10] [--warmup 2] [--rounds 3]

Prints the card's name and power limit, then one JSON line per round, workload and model with median milliseconds, then
the accuracy table."""
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
from event_utils_b200.contrast_max import (camera_rotation_warp, homography_warp, motion_contrast_candidates_torch,  # noqa: E402
                                           motion_contrast_fit_torch, motion_contrast_objective_torch,
                                           motion_timestamp_objective_torch, xyztheta_warp)

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_cmax_motion_objective import card  # noqa: E402
from bench_planar_motion import timed  # noqa: E402

# (windows, events per window, H, W, (fx, fy, cx, cy))
WORKLOADS = [(64, 30000, 180, 240, (199.1, 198.7, 132.1, 110.8)), (16, 500000, 480, 640, (530.0, 528.0, 322.0, 238.0))]
FIT_WINDOWS = 256


def make(B, n, H, W, seed=0):
    """B windows of n events in the sensor, t in [0, 0.05] per window, one angular velocity per window"""
    rng = np.random.default_rng(seed)
    xs = (rng.random((B, n)) * (W - 1)).reshape(-1)
    ys = (rng.random((B, n)) * (H - 1)).reshape(-1)
    ts = (np.sort(rng.random((B, n)), axis=1) * 0.05 + np.arange(B)[:, None] * 0.05).reshape(-1)
    ps = (rng.integers(0, 2, (B, n)) * 2.0 - 1.0).reshape(-1)
    return xs, ys, ts, ps, rng.uniform(-6, 6, (B, 3))


def models(omega, intr):
    fx, fy, cx, cy = intr
    hom = omega @ CR.embedding_matrix(intr).T
    xyz = np.column_stack((-fx * omega[:, 1], fy * omega[:, 0], np.zeros(len(omega)), -omega[:, 2]))
    return [("camera_rotation", camera_rotation_warp(intr), omega), ("homography", homography_warp(center=(cx, cy)), hom),
            ("xyztheta", xyztheta_warp(center=(cx, cy)), xyz)]


def device_events(xs, ys, ts, ps):
    return [torch.tensor(v, device="cuda", dtype=torch.float32 if i != 2 else torch.float64)
            for i, v in enumerate((xs, ys, ts, ps))]


def speed(a):
    for rnd in range(a.rounds):
        for B, n, H, W, intr in WORKLOADS:
            xs, ys, ts, ps, omega = make(B, n, H, W)
            ev = device_events(xs, ys, ts, ps)
            ends = torch.arange(1, B + 1, device="cuda") * n
            kw = dict(img_size=(H, W), batch_end_indices=ends)
            for kind, warp, params in models(omega, intr):
                base = torch.tensor(params, device="cuda")
                cand = (base.unsqueeze(1) * torch.linspace(0.8, 1.2, 32, device="cuda", dtype=torch.float64)[:, None])

                def contrast():
                    prm = base.clone().requires_grad_(True)
                    motion_contrast_objective_torch(*ev, prm, warp, **kw).sum().backward()

                def timestamp():
                    prm = base.clone().requires_grad_(True)
                    motion_timestamp_objective_torch(*ev, prm, warp, **kw).sum().backward()

                def candidates():
                    motion_contrast_candidates_torch(*ev, cand, warp, **kw)

                row = {"round": rnd, "windows": B, "events_per_window": n, "H": H, "W": W, "model": kind, "K": warp.dims}
                for name, fn in (("contrast_fb_ms", contrast), ("timestamp_fb_ms", timestamp),
                                 ("candidates_j32_ms", candidates)):
                    med, lo, hi = timed(fn, a.reps, a.warmup)
                    row[name] = round(med, 3)
                    row[name.replace("_ms", "_range_ms")] = [round(lo, 3), round(hi, 3)]
                print(json.dumps(row), flush=True)
            del ev
        # the grid-started fit: camera rotation from a grid over [-10, 10]^3, xyztheta from a grid over its ranges, the
        # homography (no grid at K = 8) from its embedding scaled by 1.1
        B, n, H, W, intr = FIT_WINDOWS, 30000, 180, 240, WORKLOADS[0][4]
        xs, ys, ts, ps, omega = make(B, n, H, W, seed=1)
        ev = device_events(xs, ys, ts, ps)
        kw = dict(img_size=(H, W), batch_end_indices=torch.arange(1, B + 1, device="cuda") * n)
        for kind, warp, params in models(omega, intr):
            if kind == "camera_rotation":
                go = dict(param_ranges=[[-10.0, 10.0]] * 3, grid_levels=3)
            elif kind == "xyztheta":
                go = dict(param_ranges=[[-2000.0, 2000.0]] * 2 + [[-2.0, 2.0], [-10.0, 10.0]], grid_levels=3)
            else:
                go = dict(x0=torch.tensor(params * 1.1, device="cuda"))
            med, lo, hi = timed(lambda: motion_contrast_fit_torch(*ev, warp, blur_sigma=[4.0, 2.0, 1.0], **go, **kw),
                                max(1, a.reps // 3), 1)
            print(json.dumps({"round": rnd, "windows": B, "events_per_window": n, "model": kind, "K": warp.dims,
                              "start": "x0" if "x0" in go else "grid", "fit_ms": round(med, 1),
                              "fit_range_ms": [round(lo, 1), round(hi, 1)]}), flush=True)
        del ev


def accuracy():
    camera = (199.1, 198.7, 132.1, 110.8)
    truths = np.array([(1.3, -1.1, 1.2), (-2.5, 1.5, 0.8), (0.5, 3.5, -2.0), (4.0, 2.5, 1.0), (-3.0, -3.5, 2.0),
                       (2.0, -4.5, -3.0), (-5.0, 2.0, 3.5), (6.0, 4.0, -3.0)])
    rng = np.random.default_rng(81)
    parts = [CR.rotation_scene(om, camera, rng, t_end=0.05, duration=0.05) for om in truths]
    x, y, t, p = (np.concatenate(a) for a in zip(*parts))
    ev = device_events(x, y, t, p)
    kw = dict(batch_end_indices=torch.tensor(np.cumsum([a[0].size for a in parts]), device="cuda"), t0=0.05,
              blur_sigma=[4.0, 2.0, 1.0])
    cam = motion_contrast_fit_torch(*ev, camera_rotation_warp(camera), param_ranges=[[-10.0, 10.0]] * 3, grid_levels=3,
                                    **kw).params.cpu().numpy()
    cxy = camera[2:]
    four_start = np.column_stack((-camera[0] * truths[:, 1] * 0.9, camera[1] * truths[:, 0] * 0.9, np.zeros(len(truths)),
                                  -truths[:, 2] * 0.9))
    four = motion_contrast_fit_torch(*ev, xyztheta_warp(center=cxy), x0=torch.tensor(four_start, device="cuda"),
                                     **kw).params.cpu().numpy()
    hx, hy, hz, th = four.T
    start = np.column_stack((hx, hy, hz, -th, th, hz, np.zeros((len(truths), 2))))
    hom = motion_contrast_fit_torch(*ev, homography_warp(center=cxy), x0=torch.tensor(start, device="cuda"),
                                    **kw).params.cpu().numpy()
    E = CR.embedding_matrix(camera)
    from_hom = np.linalg.lstsq(E, hom.T, rcond=None)[0].T
    print("accuracy on the rotation scene (|w - w_true| rad/s; the homography's w is its least-squares projection):")
    print("| window | |w_true| rad/s | camera rotation | homography |")
    print("|---|---|---|---|")
    for b, om in enumerate(truths):
        print("| %d | %.2f | %.4f | %.4f |" % (b, np.linalg.norm(om), np.linalg.norm(cam[b] - om),
                                              np.linalg.norm(from_hom[b] - om)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_camera_rotation needs a GPU")
    print("card:", card())
    speed(a)
    accuracy()


if __name__ == "__main__":
    main()
