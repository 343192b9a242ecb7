"""Forward + backward of the voxel grids through the CUDA autograd path (event_utils_b200.autograd.VoxelGrid) and
through the torch-op ports of the reference (tests/autograd_voxel_ports.py) on the same GPU, at B x 480 x 640, B = 5:

    voxel      events_to_voxel_torch, ps and ts requiring grad, loss sum(grid * R)        (20 M and 50 M events)
    negpos     events_to_neg_pos_voxel_torch, ts requiring grad                            (20 M)
    fixed_n    voxel_grids_fixed_n_torch, 100 windows, ps and ts requiring grad            (20 M)
    bwd_kernel evk_voxel_grad_f32 by itself (interleave + event pass + end-stamp terms), and the plain forward
               (events_to_voxel_torch without grad) beside it, CUDA events over `--reps` back-to-back calls

Prints the card's name and power limit, then one JSON line per measurement: median (min, max) ms of a step, CUDA
events around forward + backward.  Algorithmic bytes of the backward: 16 B/event of events in, 8 B/event of
gradients out, and the re-layout of the incoming gradient (B*H*W*4 B read, H*W*roundup(B,4)*4 B written per grid).

    python tools/bench_voxel_grad.py [--sizes 20000000 50000000] [--reps 10] [--warmup 3]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import autograd_voxel_ports as P  # noqa: E402
from event_utils_b200 import _lib  # noqa: E402
from event_utils_b200.representations.voxel_grid import (events_to_neg_pos_voxel_torch, events_to_voxel_torch,  # noqa: E402
                                                         voxel_grids_fixed_n_torch)

B, H, W = 5, 480, 640
HBM_BYTES_PER_S = 3.35e12   # H100 SXM data sheet


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        q = "unknown"
    return name, q


def events(n, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    xs = torch.rand(n, device="cuda", generator=g) * (W - 1)
    ys = torch.rand(n, device="cuda", generator=g) * (H - 1)
    ts = torch.sort(torch.rand(n, device="cuda", generator=g))[0] * 0.05
    ps = (torch.rand(n, device="cuda", generator=g) < 0.5).float() * 2 - 1
    return xs, ys, ts, ps


def timed(fn, reps, warmup, calls=1):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(calls):
            fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b) / calls)
    times.sort()
    return times[len(times) // 2], times[0], times[-1]


def regrid_bytes(grids, windows=1):
    return windows * grids * (B * H * W * 4 + H * W * ((B + 3) // 4 * 4) * 4)


def step_fn(kind, arm, ev, R):
    xs, ys, ts0, ps0 = ev
    fns = {"cuda": (events_to_voxel_torch, events_to_neg_pos_voxel_torch),
           "torch_port": (P.events_to_voxel_torch, P.events_to_neg_pos_voxel_torch)}[arm]

    def step():
        ts = ts0.clone().requires_grad_(True)
        if kind == "voxel":
            ps = ps0.clone().requires_grad_(True)
            loss = (fns[0](xs, ys, ts, ps, B, sensor_size=(H, W)) * R).sum()
        elif kind == "negpos":
            pos, neg = fns[1](xs, ys, ts, ps0, B, sensor_size=(H, W))
            loss = (pos * R).sum() - (neg * R).sum()
        else:
            ps = ps0.clone().requires_grad_(True)
            n = xs.shape[0] // 100
            if arm == "cuda":
                grids = voxel_grids_fixed_n_torch(xs, ys, ts, ps, B, n, sensor_size=(H, W))
            else:
                grids = [P.events_to_voxel_torch(xs[i:i + n], ys[i:i + n], ts[i:i + n], ps[i:i + n], B, sensor_size=(H, W))
                         for i in range(0, xs.shape[0] - n, n)]
            loss = sum((gr * R).sum() for gr in grids)
        loss.backward()
    return step


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[20_000_000, 50_000_000])
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_voxel_grad needs a GPU")
    name, power = card()
    print("card: %s; power.limit, clocks.max.sm: %s" % (name, power))
    R = torch.randn(B, H, W, device="cuda", generator=torch.Generator(device="cuda").manual_seed(1))
    L = _lib.lib()

    def emit(rec):
        rec.update(gpu=name, power=power)
        print(json.dumps(rec), flush=True)

    for n in args.sizes:
        ev = events(n)
        xs, ys, ts, ps = ev
        kinds = ["voxel"] + (["negpos", "fixed_n"] if n == args.sizes[0] else [])
        for kind in kinds:
            for arm in ("cuda", "torch_port"):
                med, lo, hi = timed(step_fn(kind, arm, ev, R), args.reps, args.warmup)
                emit(dict(what=kind + " fwd+bwd", events=n, grid=[B, H, W], arm=arm, ms_median=round(med, 3),
                          ms_min=round(lo, 3), ms_max=round(hi, 3)))
            torch.cuda.empty_cache()
        # the backward entry point by itself, and the plain forward beside it
        gp, gt = torch.empty_like(ps), torch.empty_like(ts)
        ws = torch.empty(L.evk_voxel_grad_workspace_bytes(1, B, H, W, 0), dtype=torch.uint8, device="cuda")

        def bwd():
            _lib.check(L.evk_voxel_grad_f32(_lib.ptr(xs), _lib.ptr(ys), _lib.ptr(ts), _lib.ptr(ps), n, None, 1, B, H, W, 0,
                                            _lib.ptr(R), _lib.ptr(gp), _lib.ptr(gt), _lib.ptr(ws), ws.numel(), _lib.stream()))

        def fwd():
            events_to_voxel_torch(xs, ys, ts, ps, B, sensor_size=(H, W))
        for what, fn in (("bwd_kernel", bwd), ("fwd_plain", fwd)):
            med, lo, hi = timed(fn, args.reps, args.warmup, calls=10)
            rec = dict(what=what, events=n, grid=[B, H, W], arm="cuda", ms_median=round(med, 4), ms_min=round(lo, 4),
                       ms_max=round(hi, 4))
            if what == "bwd_kernel":
                by = 24 * n + regrid_bytes(1)
                rec.update(bytes=by, bytes_per_event_events=24, bytes_regrid=regrid_bytes(1),
                           algorithmic_GBps=round(by / (med * 1e-3) / 1e9, 1),
                           share_of_hbm_datasheet=round(by / (med * 1e-3) / HBM_BYTES_PER_S, 3))
            emit(rec)
        del ev, xs, ys, ts, ps, gp, gt, ws
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
