"""Forward + backward of the batched dense-flow average-timestamp loss: the fused path (flow_timestamp_objective_torch,
two passes over the events) against the composed per-sample autograd path a user would otherwise write
(warp_events_flow_torch -> events_to_timestamp_image_torch -> torch reflect-padded Gaussian blur -> sum of squares,
one Python iteration per sample).  The flows keep every event inside the canvas, so both paths compute the same loss;
they must agree on f and the gradient before anything is timed.  Also the two event passes alone (CUDA events around
them, evk_prof_*) against their byte floor: 20 B per event (x, y, d, tau, p) at 3.35 TB/s.

    python tools/bench_flow_timestamp_objective.py [--reps 20] [--warmup 3]

Prints the card's name and power limit, then one JSON line per size and sigma."""
import argparse
import ctypes
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from event_utils_b200 import _lib  # noqa: E402
from event_utils_b200.contrast_max import flow_timestamp_objective_torch  # noqa: E402
from event_utils_b200.representations.image import events_to_timestamp_image_torch  # noqa: E402
from event_utils_b200.transforms.optic_flow import warp_events_flow_torch  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_cmax_flow_objective import blur_torch, card, make, timed  # noqa: E402

SIZES = [(8, 500000, 480, 640), (16, 100000, 260, 346)]
SIGMAS = (0.0, 2.0)
HBM_BYTES_PER_S = 3.35e12


def composed(x, y, t, p, flow, ends_host, H, W, sigma):
    fs = []
    lo = 0
    for b, hi in enumerate(ends_host):
        xw, yw = warp_events_flow_torch(x[lo:hi], y[lo:hi], t[lo:hi], p[lo:hi], flow[b])
        f = 0.0
        for img in events_to_timestamp_image_torch(xw, yw, t[lo:hi], p[lo:hi], sensor_size=(H, W)):
            G = blur_torch(img, sigma) if sigma > 0 else img
            f = f + (G.double() ** 2).sum()
        fs.append(f)
        lo = hi
    return torch.stack(fs)


def event_pass_ms(fn, reps):
    """mean time of the event pass each call of fn brackets (evk_prof_*), over reps calls"""
    L = _lib.lib()
    torch.cuda.synchronize()
    L.evk_prof_collect(None, None, None)
    L.evk_prof_enable(1)
    for _ in range(reps):
        fn()
    ms, n = ctypes.c_double(), ctypes.c_longlong()
    _lib.check(L.evk_prof_collect(ctypes.byref(ms), ctypes.byref(n), None))
    L.evk_prof_enable(0)
    return ms.value / max(n.value, 1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a GPU")
    print("card: %s" % card())
    for B, n, H, W in SIZES:
        x, y, t, p, flow, ends = make(B, n, H, W)
        ends_host = [int(e) for e in ends.cpu()]
        fl = flow.clone().requires_grad_(True)
        for sigma in SIGMAS:
            def fused():
                fl.grad = None
                f = flow_timestamp_objective_torch(x, y, t, p, fl, blur_sigma=sigma, batch_end_indices=ends)
                f.sum().backward()
                return f

            def comp():
                fl.grad = None
                f = composed(x, y, t, p, fl, ends_host, H, W, sigma)
                f.sum().backward()
                return f

            f1 = fused().detach()
            g1 = fl.grad.clone()
            f2 = comp().detach()
            g2 = fl.grad.clone()
            rel_f = float(((f1 - f2).abs() / f2.abs()).max())
            rel_g = float((g1 - g2).abs().max() / g2.abs().max())
            assert rel_f <= 1e-4 and rel_g <= 1e-3, ("the two paths disagree", rel_f, rel_g)
            ms_fused = timed(fused, a.reps, a.warmup)
            ms_comp = timed(comp, max(3, a.reps // 4), 1)
            with torch.no_grad():
                fwd_ms = event_pass_ms(lambda: flow_timestamp_objective_torch(x, y, t, p, fl, blur_sigma=sigma,
                                                                              batch_end_indices=ends), a.reps)
            f = flow_timestamp_objective_torch(x, y, t, p, fl, blur_sigma=sigma, batch_end_indices=ends)
            bwd_ms = event_pass_ms(lambda: torch.autograd.grad(f.sum(), fl, retain_graph=True), a.reps)
            floor_ms = 20.0 * B * n / HBM_BYTES_PER_S * 1e3
            print(json.dumps({"batch": B, "events_per_sample": n, "H": H, "W": W, "sigma": sigma,
                              "fused_fwd_bwd_ms": round(ms_fused, 3), "composed_fwd_bwd_ms": round(ms_comp, 3),
                              "speedup": round(ms_comp / ms_fused, 2),
                              "fwd_event_pass_ms": round(fwd_ms, 4), "bwd_event_pass_ms": round(bwd_ms, 4),
                              "event_bytes_floor_ms": round(floor_ms, 4),
                              "f_max_rel_diff": rel_f, "grad_max_rel_diff": rel_g}))


if __name__ == "__main__":
    main()
