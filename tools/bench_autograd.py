"""Forward + backward of the two training chains through the CUDA autograd path and through the torch-op ports of the
reference (tests/autograd_ports.py: the reference's own formulation, ATen index_put_ and grid_sample backward) on the
same GPU:

    image      flow (requires grad) -> warp_events_flow_torch -> events_to_image_torch (bilinear) -> sum(img^2)
    timestamp  flow (requires grad) -> warp_events_flow_torch -> events_to_timestamp_image_torch -> sum(pos^2 + neg^2)

at 1 M and 20 M events with a 480x640 flow.  Prints the card's name and power limit, then one JSON line per chain,
size and arm: median time of a step (CUDA events around forward + backward), and the algorithmic event-array bytes
per event of our path (computed from the arrays each kernel reads and writes) with the rate they imply.

    python tools/bench_autograd.py [--sizes 1000000 20000000] [--reps 10] [--warmup 3]
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
import autograd_ports as P  # noqa: E402
from event_utils_b200.representations.image import events_to_image_torch, events_to_timestamp_image_torch  # noqa: E402
from event_utils_b200.transforms.optic_flow import warp_events_flow_torch  # noqa: E402

H, W = 480, 640
HBM_BYTES_PER_S = 3.35e12   # H100 SXM data sheet

# bytes of event arrays (4-byte floats) each kernel of our chain reads + writes per event; the images and the flow
# (at most 10 MB each) stay in L2
BYTES = {
    "image": {"warp fwd (x,y,t -> xw,yw)": 12 + 8, "image fwd (xw,yw,p)": 12,
              "image bwd (xw,yw,p -> gxw,gyw)": 12 + 8, "warp bwd (x,y,t,gxw,gyw)": 20},
    "timestamp": {"warp fwd (x,y,t -> xw,yw)": 12 + 8, "tsimg fwd (xw,yw,t,p)": 16,
                  "tsimg bwd (xw,yw,t,p -> gxw,gyw)": 16 + 8, "warp bwd (x,y,t,gxw,gyw)": 20},
}


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
    flow = torch.randn(2, H, W, device="cuda", generator=g) * 20
    return xs, ys, ts, ps, flow


def step(chain, fns, ev):
    image, tsimg, warp = fns
    xs, ys, ts, ps, flow0 = ev
    flow = flow0.clone().requires_grad_(True)
    xw, yw = warp(xs, ys, ts, ps, flow)
    if chain == "image":
        img = image(xw, yw, ps, sensor_size=(H, W), interpolation='bilinear')
        loss = (img * img).sum()
    else:
        pos, neg = tsimg(xw, yw, ts, ps, sensor_size=(H, W))
        loss = (pos * pos).sum() + (neg * neg).sum()
    loss.backward()
    return flow.grad


def time_steps(chain, fns, ev, reps, warmup):
    for _ in range(warmup):
        step(chain, fns, ev)
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        step(chain, fns, ev)
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    times.sort()
    return times[len(times) // 2], times[0], times[-1]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[1_000_000, 20_000_000])
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_autograd needs a GPU")
    name, power = card()
    print("card: %s; power.limit, clocks.max.sm: %s" % (name, power))
    arms = {"cuda": (events_to_image_torch, events_to_timestamp_image_torch, warp_events_flow_torch),
            "torch_port": (P.events_to_image_torch, P.events_to_timestamp_image_torch, P.warp_events_flow_torch)}
    for n in args.sizes:
        ev = events(n)
        for chain in ("image", "timestamp"):
            for arm, fns in arms.items():
                med, lo, hi = time_steps(chain, fns, ev, args.reps, args.warmup)
                rec = dict(chain=chain, events=n, flow=[2, H, W], arm=arm, ms_median=round(med, 3), ms_min=round(lo, 3),
                           ms_max=round(hi, 3), gpu=name, power=power)
                if arm == "cuda":
                    bpe = sum(BYTES[chain].values())
                    rec.update(bytes_per_event=bpe, bytes_per_event_by_kernel=BYTES[chain],
                               algorithmic_GBps=round(bpe * n / (med * 1e-3) / 1e9, 1),
                               share_of_hbm_datasheet=round(bpe * n / (med * 1e-3) / HBM_BYTES_PER_S, 3))
                print(json.dumps(rec), flush=True)
        del ev
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
