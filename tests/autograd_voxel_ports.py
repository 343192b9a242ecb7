"""Torch-op ports of the reference's torch voxel grids -- TEST / BASELINE INFRASTRUCTURE ONLY.

Written from the reference's semantics with the ops it uses: per bin b a weight ps * max(0, 1 - |tn - b|) with
tn = ((ts - ts[0]) / dt) * (B-1), dt = ts[-1] - ts[0], scattered by `index_put_(accumulate=True)` at the truncated
(wrapping) pixel, so that autograd on these ports gives the reference's gradients w.r.t. ps and ts.  Unlike the
reference they build their constants on the inputs' device, so they run on CUDA too.  tests/test_autograd_voxel_port.py
pins them to the real reference through tests/golden/autograd_voxel.npz; tests/test_gpu_voxel_autograd.py and
tools/bench_voxel_grad.py compare the CUDA backward against them.

  events_to_voxel_torch          lib/representations/voxel_grid.py:114-153
  events_to_neg_pos_voxel_torch  lib/representations/voxel_grid.py:155-182
"""
import torch


def events_to_voxel_torch(xs, ys, ts, ps, B, device=None, sensor_size=(180, 240)):
    dev = xs.device
    dt = ts[-1] - ts[0]
    tn = (ts - ts[0]) / dt * (B - 1)
    zeros = torch.zeros(tn.shape, device=dev)
    iy, ix = ys.long(), xs.long()
    bins = []
    for b in range(B):
        w = ps * torch.max(zeros, 1.0 - torch.abs(tn - b))
        img = torch.zeros(tuple(sensor_size), device=dev)
        bins.append(img.index_put_((iy, ix), w, accumulate=True))
    out = torch.stack(bins)
    return out if device is None else out.to(device)


def events_to_neg_pos_voxel_torch(xs, ys, ts, ps, B, device=None, sensor_size=(180, 240)):
    one, zero = torch.ones((), device=xs.device), torch.zeros((), device=xs.device)
    pos = events_to_voxel_torch(xs, ys, ts, torch.where(ps > 0, one, zero), B, device, sensor_size)
    neg = events_to_voxel_torch(xs, ys, ts, torch.where(ps <= 0, one, zero), B, device, sensor_size)
    return pos, neg
