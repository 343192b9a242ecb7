"""Forward + backward of the batched dense-flow contrast loss: the fused path (flow_contrast_objective_torch, two passes
over the events) against the composed per-sample autograd path a user would otherwise write (warp_events_flow_torch ->
events_to_image_torch(bilinear) -> torch Gaussian blur -> -var, one Python iteration per sample).  The flows keep every
event inside the canvas, so the composed path does not raise; both paths must agree on f.

    python tools/bench_cmax_flow_objective.py [--reps 20] [--warmup 3]

Prints the card's name and power limit, then one JSON line per size."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from event_utils_b200.contrast_max import flow_contrast_objective_torch  # noqa: E402
from event_utils_b200.representations.image import events_to_image_torch  # noqa: E402
from event_utils_b200.transforms.optic_flow import warp_events_flow_torch  # noqa: E402

SIZES = [(8, 500000, 480, 640), (16, 100000, 260, 346)]
SIGMA = 1.0


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def make(B, n, H, W, seed=0):
    """B samples of n events 12 px inside the sensor, t in [0, 0.05] per sample, flows of at most 200 px/s (10 px)"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = 12 + torch.rand(B * n, device="cuda", generator=g) * (W - 25)
    y = 12 + torch.rand(B * n, device="cuda", generator=g) * (H - 25)
    t = (torch.rand(B, n, device="cuda", generator=g).sort(dim=1).values * 0.05).reshape(-1)
    p = torch.randint(0, 2, (B * n,), device="cuda", generator=g).float() * 2 - 1
    yy, xx = torch.meshgrid(torch.arange(H, device="cuda"), torch.arange(W, device="cuda"), indexing="ij")
    ph = torch.rand(B, 2, 1, 1, device="cuda", generator=g) * 6.28
    flow = torch.stack((torch.cos(xx / 37.0 + ph[:, 0]), torch.sin(yy / 23.0 + ph[:, 1])), dim=1) * 200.0
    ends = torch.arange(1, B + 1, device="cuda", dtype=torch.int64) * n
    return x, y, t, p, flow.float().contiguous(), ends


def blur_torch(img, sigma):
    """scipy.ndimage.gaussian_filter(img, sigma) (truncate 4, mode reflect) with torch ops"""
    r = int(4.0 * sigma + 0.5)
    k = torch.exp(-0.5 * (torch.arange(-r, r + 1, device=img.device, dtype=torch.float64) / sigma) ** 2)
    k = (k / k.sum()).float()

    def reflect(n):
        i = torch.arange(-r, n + r, device=img.device)
        i = torch.remainder(i, 2 * n)
        return torch.where(i < n, i, 2 * n - 1 - i)

    H, W = img.shape
    a = img[reflect(H)].t().unsqueeze(1)                      # (W, 1, H + 2r)
    a = F.conv1d(a, k.view(1, 1, -1)).squeeze(1).t()          # (H, W)
    b = a[:, reflect(W)].unsqueeze(1)                         # (H, 1, W + 2r)
    return F.conv1d(b, k.view(1, 1, -1)).squeeze(1)


def composed(x, y, t, p, flow, ends_host, H, W):
    fs = []
    lo = 0
    for b, hi in enumerate(ends_host):
        xw, yw = warp_events_flow_torch(x[lo:hi], y[lo:hi], t[lo:hi], p[lo:hi], flow[b])
        img = events_to_image_torch(xw, yw, p[lo:hi], sensor_size=(H, W), interpolation='bilinear')
        G = blur_torch(img, SIGMA)
        fs.append(-((G - G.mean()) ** 2).mean())
        lo = hi
    return torch.stack(fs)


def timed(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


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

        def fused():
            fl.grad = None
            f = flow_contrast_objective_torch(x, y, t, p, fl, objective="variance", blur_sigma=SIGMA, batch_end_indices=ends)
            f.sum().backward()
            return f

        def comp():
            fl.grad = None
            f = composed(x, y, t, p, fl, ends_host, H, W)
            f.sum().backward()
            return f

        f1 = fused().detach()
        g1 = fl.grad.clone()
        f2 = comp().detach()
        g2 = fl.grad.clone()
        rel_f = float(((f1 - f2).abs() / f2.abs()).max())
        rel_g = float((g1 - g2).abs().max() / g2.abs().max())
        assert rel_f <= 1e-4, ("f disagrees", f1, f2)
        ms_fused = timed(fused, a.reps, a.warmup)
        ms_comp = timed(comp, max(3, a.reps // 4), 1)
        print(json.dumps({"batch": B, "events_per_sample": n, "H": H, "W": W, "sigma": SIGMA,
                          "fused_fwd_bwd_ms": round(ms_fused, 3), "composed_fwd_bwd_ms": round(ms_comp, 3),
                          "speedup": round(ms_comp / ms_fused, 2), "f_max_rel_diff": rel_f, "grad_max_rel_diff": rel_g}))


if __name__ == "__main__":
    main()
