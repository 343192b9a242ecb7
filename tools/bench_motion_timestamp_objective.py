"""Forward + backward of the batched parametric average-timestamp loss (motion_timestamp_objective_torch: one event pass
each way for the whole batch) against what a user runs today: per window zhu_timestamp_objective.evaluate_function plus
a K+1-point forward-difference gradient (the objective has no derivative, has_derivative=False, so optimize_contrast
takes finite differences).  That objective warps and masks on the host, so there is nothing to pin.  The events stay
strictly inside the canvas under every window's motion, so both paths compute the same loss (f of one is -f of the
other); they must agree on f before anything is timed.

    python tools/bench_motion_timestamp_objective.py [--reps 10] [--warmup 2]

Prints the card's name and power limit, then one JSON line per workload: the batched path through the torch function,
the same two C entries called alone on prepared events (its GPU side), the per-window loop (at 180x240, the canvas of
zhu_timestamp_objective), and the byte floor of the batched path: 20 B per event per pass (x, y, d, tau, p as f32),
two passes, at the H100 SXM's 3.35 TB/s."""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from event_utils_b200 import _lib  # noqa: E402
from event_utils_b200.contrast_max import (motion_timestamp_objective_torch, pure_rotation_warp, xyztheta_warp,  # noqa: E402
                                           zhu_timestamp_objective)
from event_utils_b200.contrast_max._batched import _normalised_stamps  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_cmax_motion_objective import card  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
# (model, windows, events per window, H, W, time the per-window loop too)
WORKLOADS = [("rotation", 64, 30000, 180, 240, True), ("xyztheta", 8, 500000, 180, 240, True),
             ("xyztheta", 16, 500000, 480, 640, False)]
SIGMA = 2.0          # zhu_timestamp_objective's default_blur
FD_STEP = 1e-3


def make(kind, B, n, H, W, seed=0):
    """B windows of n events at least 40 px inside the sensor, t in [0, 0.05] per window; the warp and one parameter
    vector per window, small enough that no event leaves the canvas"""
    rng = np.random.default_rng(seed)
    xs = 40 + rng.random((B, n)) * (W - 81)
    ys = 40 + rng.random((B, n)) * (H - 81)
    ts = np.sort(rng.random((B, n)), axis=1) * 0.05 + np.arange(B)[:, None] * 0.05
    ps = rng.integers(0, 2, (B, n)) * 2.0 - 1.0
    if kind == "rotation":
        warp = pure_rotation_warp()
        params = np.column_stack((W / 2 + rng.uniform(-5, 5, B), H / 2 + rng.uniform(-5, 5, B), rng.uniform(-2, 2, B)))
    else:
        warp = xyztheta_warp(center=(W / 2, H / 2))
        params = np.column_stack((rng.uniform(-30, 30, (B, 2)), rng.uniform(-2, 2, (B, 2))))
    return xs, ys, ts, ps, warp, params


def entries_only(kind, warp, x, y, t, p, ends, base, H, W, reps, warmup):
    """The two C entries alone (evk_motion_timestamp_objective_f32 + _grad_f32) on events already prepared as they take
    them (t - t0_b as f32, tau, sample offsets): the GPU side of the batched path without the Python and autograd
    layers."""
    L = _lib.lib()
    B, K = base.shape
    n = x.shape[0] // B
    t_rel = (t.view(B, n) - t.view(B, n)[:, -1:]).reshape(-1).float().contiguous()
    offsets = torch.cat((torch.zeros(1, dtype=torch.int64, device="cuda"), ends))
    sample = torch.arange(B, device="cuda").repeat_interleave(n)
    tau = _normalised_stamps(t, sample, offsets, False)
    code = {"rotation": _lib.WARP_ROTATION, "xyztheta": _lib.WARP_XYZTHETA}[kind]
    cx, cy = warp.center if kind == "xyztheta" else (0.0, 0.0)
    f = torch.empty(B, dtype=torch.float64, device="cuda")
    T = torch.empty((B, 2, H + 1, W + 1), device="cuda")
    C = torch.empty_like(T)
    gf = torch.ones(B, device="cuda")
    gp = torch.empty_like(base)
    ws = torch.empty(L.evk_motion_timestamp_objective_workspace_bytes(B, H, W), dtype=torch.uint8, device="cuda")
    ev = [_lib.ptr(v) for v in (x, y, t_rel, tau, p, offsets)]

    def once():
        _lib.check(L.evk_motion_timestamp_objective_f32(*ev, B, x.shape[0], code, _lib.ptr(base), K, cx, cy, H, W, SIGMA,
                                                        _lib.ptr(f), _lib.ptr(T), _lib.ptr(C), _lib.ptr(ws), ws.numel(),
                                                        _lib.stream()))
        _lib.check(L.evk_motion_timestamp_objective_grad_f32(*ev, B, x.shape[0], code, _lib.ptr(base), K, cx, cy, H, W, SIGMA,
                                                             _lib.ptr(T), _lib.ptr(C), _lib.ptr(gf), _lib.ptr(gp),
                                                             _lib.ptr(ws), ws.numel(), _lib.stream()))
    for _ in range(warmup):
        once()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        once()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a GPU")
    print("card: %s" % card())
    obj = zhu_timestamp_objective()
    for kind, B, n, H, W, loop in WORKLOADS:
        xs, ys, ts, ps, warp, params = make(kind, B, n, H, W)
        x, y, p = (torch.from_numpy(v.reshape(-1)).float().cuda() for v in (xs, ys, ps))
        t = torch.from_numpy(ts.reshape(-1)).cuda()
        ends = torch.arange(1, B + 1, device="cuda", dtype=torch.int64) * n
        base = torch.tensor(params, device="cuda")

        def batched(r):
            prm = (base + 1e-4 * r).requires_grad_(True)
            f = motion_timestamp_objective_torch(x, y, t, p, prm, warp, blur_sigma=SIGMA, img_size=(H, W),
                                                 batch_end_indices=ends)
            f.sum().backward()
            return f.detach(), prm.grad

        for r in range(a.warmup):
            batched(-1 - r)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for r in range(a.reps):
            batched(r)
        e1.record()
        torch.cuda.synchronize()
        ms_batched = e0.elapsed_time(e1) / a.reps
        ms_entries = entries_only(kind, warp, x, y, t, p, ends, base, H, W, a.reps, a.warmup)
        floor_ms = 2 * 20.0 * B * n / HBM_BYTES_PER_S * 1e3
        out = {"model": kind, "windows": B, "events_per_window": n, "H": H, "W": W, "sigma": SIGMA,
               "batched_fwd_bwd_ms": round(ms_batched, 3), "entries_only_fwd_bwd_ms": round(ms_entries, 3),
               "byte_floor_ms": round(floor_ms, 3)}
        if loop:
            K = params.shape[1]

            def per_window(r):
                fs = []
                for b in range(B):
                    q = params[b] + 1e-4 * r
                    w = (xs[b], ys[b], ts[b], ps[b])
                    f0 = obj.evaluate_function(q, *w, warp, (H, W), SIGMA)
                    for k in range(K):       # the K+1-point forward-difference gradient
                        obj.evaluate_function(q + FD_STEP * np.eye(K)[k], *w, warp, (H, W), SIGMA)
                    fs.append(f0)
                return np.array(fs)

            for r in range(a.warmup):
                per_window(-1 - r)
            f_loop = per_window(0)
            f_b, _ = batched(0)
            rel_f = float(np.max(np.abs(f_b.cpu().numpy() + f_loop) / np.abs(f_loop)))
            assert rel_f <= 4 * 2.0 ** -15, ("f disagrees", rel_f)
            reps = max(2, a.reps // 4)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for r in range(1, reps + 1):
                per_window(r)
            torch.cuda.synchronize()
            ms_loop = (time.perf_counter() - t0) * 1e3 / reps
            out.update(loop_fwd_fd_grad_ms=round(ms_loop, 3), speedup=round(ms_loop / ms_batched, 2), f_max_rel_diff=rel_f)
        print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
