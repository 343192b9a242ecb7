"""Forward + backward of the batched parametric contrast loss (motion_contrast_objective_torch: one event pass each way
for the whole batch) against the per-window loop a user writes today: objective.evaluate_function +
evaluate_gradient in precision="f32", each window inside pinned_events (uploaded once, before the timing).  Both
paths must agree on f.  The parameters move by 1e-4 per repetition, so that the loop's memoisation of (params -> f, g)
does not skip evaluations.

    python tools/bench_cmax_motion_objective.py [--reps 10] [--warmup 2]

Prints the card's name and power limit, then one JSON line per workload: the batched path through the torch function,
the same two C entries called alone on prepared events (its GPU side), the per-window loop, and the byte floor of the
batched path: 16 B per event per pass (x, y, t, p as f32), two passes, at the H100 SXM's 3.35 TB/s."""
import argparse
import contextlib
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from event_utils_b200.contrast_max import motion_contrast_objective_torch, pure_rotation_warp, xyztheta_warp  # noqa: E402
from event_utils_b200 import _lib  # noqa: E402
from event_utils_b200.contrast_max import objectives as OB  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
# (model, windows, events per window, H, W, time the per-window loop too)
WORKLOADS = [("rotation", 64, 30000, 180, 240, True), ("xyztheta", 8, 500000, 180, 240, True),
             ("xyztheta", 16, 500000, 480, 640, False)]
SIGMA = 1.0


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def make(kind, B, n, H, W, seed=0):
    """B windows of n events in the sensor, t in [0, 0.05] per window; the warp and one parameter vector per window"""
    rng = np.random.default_rng(seed)
    xs = rng.random((B, n)) * (W - 1)
    ys = rng.random((B, n)) * (H - 1)
    ts = np.sort(rng.random((B, n)), axis=1) * 0.05 + np.arange(B)[:, None] * 0.05
    ps = rng.integers(0, 2, (B, n)) * 2.0 - 1.0
    if kind == "rotation":
        warp = pure_rotation_warp()
        params = np.column_stack((W / 2 + rng.uniform(-5, 5, B), H / 2 + rng.uniform(-5, 5, B), rng.uniform(-6, 6, B)))
    else:
        warp = xyztheta_warp(center=(W / 2, H / 2))
        params = np.column_stack((rng.uniform(-30, 30, (B, 2)), rng.uniform(-3, 3, (B, 2))))
    return xs, ys, ts, ps, warp, params


def entries_only(kind, warp, x, y, t, p, ends, base, H, W, reps, warmup):
    """The two C entries alone (evk_cmax_motion_objective_f32 + _grad_f32) on events already prepared as they take them
    (t - t0_b as f32, sample offsets): the GPU side of the batched path without the Python and autograd layers."""
    L = _lib.lib()
    B, K = base.shape
    n = x.shape[0] // B
    t_rel = (t.view(B, n) - t.view(B, n)[:, -1:]).reshape(-1).float().contiguous()
    offsets = torch.cat((torch.zeros(1, dtype=torch.int64, device="cuda"), ends))
    code = {"rotation": _lib.WARP_ROTATION, "xyztheta": _lib.WARP_XYZTHETA}[kind]
    cx, cy = warp.center if kind == "xyztheta" else (0.0, 0.0)
    f = torch.empty(B, dtype=torch.float64, device="cuda")
    iwe = torch.empty((B, H + 1, W + 1), device="cuda")
    gf = torch.ones(B, device="cuda")
    gp = torch.empty_like(base)
    ws = torch.empty(L.evk_cmax_motion_objective_workspace_bytes(B, H, W), dtype=torch.uint8, device="cuda")
    ev = [_lib.ptr(v) for v in (x, y, t_rel, p, offsets)]

    def once():
        _lib.check(L.evk_cmax_motion_objective_f32(*ev, B, x.shape[0], code, _lib.ptr(base), K, cx, cy, H, W, SIGMA, 0, 0.0,
                                                   _lib.ptr(f), _lib.ptr(iwe), _lib.ptr(ws), ws.numel(), _lib.stream()))
        _lib.check(L.evk_cmax_motion_objective_grad_f32(*ev, B, x.shape[0], code, _lib.ptr(base), K, cx, cy, H, W, SIGMA, 0, 0.0,
                                                        _lib.ptr(iwe), _lib.ptr(gf), _lib.ptr(gp), _lib.ptr(ws), ws.numel(),
                                                        _lib.stream()))
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
    obj = OB.variance_objective()
    for kind, B, n, H, W, loop in WORKLOADS:
        xs, ys, ts, ps, warp, params = make(kind, B, n, H, W)
        x, y, p = (torch.from_numpy(v.reshape(-1)).float().cuda() for v in (xs, ys, ps))
        t = torch.from_numpy(ts.reshape(-1)).cuda()
        ends = torch.arange(1, B + 1, device="cuda", dtype=torch.int64) * n
        base = torch.tensor(params, device="cuda")

        def batched(r):
            prm = (base + 1e-4 * r).requires_grad_(True)
            f = motion_contrast_objective_torch(x, y, t, p, prm, warp, blur_sigma=SIGMA, img_size=(H, W), batch_end_indices=ends)
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
        floor_ms = 2 * 16.0 * B * n / HBM_BYTES_PER_S * 1e3
        out = {"model": kind, "windows": B, "events_per_window": n, "H": H, "W": W, "sigma": SIGMA,
               "batched_fwd_bwd_ms": round(ms_batched, 3), "entries_only_fwd_bwd_ms": round(ms_entries, 3),
               "byte_floor_ms": round(floor_ms, 3)}
        if loop:
            OB.precision, OB.event_pass = "f32", None
            try:
                # the same array objects go to pinned_events and to every evaluation: pinned_events matches by identity,
                # and a fresh slice xs[b] per call would miss it (a content hash, and a re-upload once the two-slot
                # cache has cycled, per call)
                wins = [(xs[b], ys[b], ts[b], ps[b]) for b in range(B)]
                with contextlib.ExitStack() as stack:
                    for w in wins:
                        stack.enter_context(OB.pinned_events(*w))
                    assert all(OB.pinned_events.lookup(*w) is not None for w in wins)

                    def per_window(r):
                        fs, gs = [], []
                        for b, w in enumerate(wins):
                            q = params[b] + 1e-4 * r
                            fs.append(obj.evaluate_function(q, *w, warp, (H, W), SIGMA))
                            gs.append(obj.evaluate_gradient(q, *w, warp, (H, W), SIGMA))
                        return np.array(fs), np.array(gs)

                    for r in range(a.warmup):
                        per_window(-1 - r)
                    f_loop, _ = per_window(0)
                    f_b, _ = batched(0)
                    rel_f = float(np.max(np.abs(f_b.cpu().numpy() - f_loop) / np.abs(f_loop)))
                    assert rel_f <= 1e-5, ("f disagrees", rel_f)
                    reps = max(2, a.reps // 2)
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    for r in range(1, reps + 1):
                        per_window(r)
                    torch.cuda.synchronize()
                    ms_loop = (time.perf_counter() - t0) * 1e3 / reps
            finally:
                OB.precision, OB.event_pass = "f64", None
                OB.clear_cache()
            out.update(loop_fwd_bwd_ms=round(ms_loop, 3), speedup=round(ms_loop / ms_batched, 2), f_max_rel_diff=rel_f)
        print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
