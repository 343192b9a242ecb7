"""Torch-op ports of the three differentiable reference functions -- TEST / BASELINE INFRASTRUCTURE ONLY.

Written from the reference's documented semantics with the same torch ops it uses (`index_put_(accumulate=True)`
with weights built from `x - floor(x)`, `grid_sample`), so that autograd on these ports gives the reference's
gradients on any machine and any device, the GPU one included.  tests/test_autograd_port.py pins them to the real
reference through tests/golden/autograd*.npz; tests/test_gpu_autograd.py and tools/bench_autograd.py compare the
CUDA backward passes against them.

  events_to_image_torch            lib/representations/image.py:46-100 (interpolate_to_image :102-115)
  events_to_timestamp_image_torch  lib/representations/image.py:286-353
  warp_events_flow_torch           lib/transforms/optic_flow.py:5-46
"""
import torch
import torch.nn.functional as F


def _clip_mask(xs, ys, img_size, interpolation, padding):
    # a coordinate at or beyond the last usable column / row is clipped; nearest without padding may use them all
    clipx = img_size[1] if interpolation is None and padding == False else img_size[1] - 1  # noqa: E712
    clipy = img_size[0] if interpolation is None and padding == False else img_size[0] - 1  # noqa: E712
    one, zero = torch.ones((), device=xs.device), torch.zeros((), device=xs.device)
    return torch.where(xs >= clipx, zero, one) * torch.where(ys >= clipy, zero, one)


def _splat_bilinear(img, px, py, dx, dy, w):
    img.index_put_((py, px), w * (1.0 - dx) * (1.0 - dy), accumulate=True)
    img.index_put_((py, px + 1), w * dx * (1.0 - dy), accumulate=True)
    img.index_put_((py + 1, px), w * (1.0 - dx) * dy, accumulate=True)
    img.index_put_((py + 1, px + 1), w * dx * dy, accumulate=True)
    return img


def events_to_image_torch(xs, ys, ps, sensor_size=(180, 240), clip_out_of_range=True, interpolation=None, padding=True,
                          default=0):
    """Nearest: img[trunc(y)*m, trunc(x)*m] += p (the weight is not masked).  Bilinear: four taps of p*m at
    floor(x)*m, floor(y)*m with the unmasked fractions, on an (H+1,W+1) canvas with padding."""
    dev = xs.device
    if interpolation == 'bilinear' and padding:
        img_size = (sensor_size[0] + 1, sensor_size[1] + 1)
    else:
        img_size = tuple(sensor_size)
    mask = torch.ones(xs.shape, device=dev)
    if clip_out_of_range:
        mask = _clip_mask(xs, ys, img_size, interpolation, padding)
    img = torch.ones(img_size, device=dev) * default
    if interpolation == 'bilinear' and xs.dtype is not torch.long:
        fx, fy = xs.floor().float(), ys.floor().float()
        dx, dy = (xs - fx).float(), (ys - fy).float()
        return _splat_bilinear(img, (fx * mask).long(), (fy * mask).long(), dx, dy, ps.squeeze() * mask)
    m = mask.long()
    return img.index_put_((ys.long() * m, xs.long() * m), ps, accumulate=True)


def events_to_timestamp_image_torch(xs, ys, ts, ps, sensor_size=(180, 240), clip_out_of_range=True,
                                    interpolation='bilinear', padding=True, timestamp_reverse=False):
    """Average normalised timestamp of the positive / negative events per pixel: bilinear sums of tn*[p>0] and of
    [p>0] (the count starts at one), divided; likewise for p<=0.  A clipped event keeps its weight, only its index
    is zeroed."""
    dev = xs.device
    xs, ys, ts, ps = xs.squeeze(), ys.squeeze(), ts.squeeze(), ps.squeeze()
    img_size = (sensor_size[0] + 1, sensor_size[1] + 1) if padding else tuple(sensor_size)
    mask = torch.ones(xs.shape, device=dev)
    if clip_out_of_range:
        mask = _clip_mask(xs, ys, img_size, interpolation, padding)
    one, zero = torch.ones((), device=dev), torch.zeros((), device=dev)
    pos, neg = torch.where(ps > 0, one, zero), torch.where(ps <= 0, one, zero)
    denom = ts[-1] - ts[0] + 1e-6
    tn = ((ts[-1] - ts) if timestamp_reverse else (ts - ts[0])) / denom
    fx, fy = xs.floor().float(), ys.floor().float()
    dx, dy = (xs - fx).float(), (ys - fy).float()
    px, py = (fx * mask).long(), (fy * mask).long()
    out = []
    for sel in (pos, neg):
        s = _splat_bilinear(torch.zeros(img_size, device=dev), px, py, dx, dy, (tn * sel).float())
        c = _splat_bilinear(torch.ones(img_size, device=dev), px, py, dx, dy, sel)
        c = torch.where(c == 0, one, c)
        out.append(s / c)
    return out[0], out[1]


def warp_events_flow_torch(xt, yt, tt, pt, flow_field, t0=None):
    """x' = x + u(x,y) (t - t0), y' = y + v(x,y) (t - t0) with the flow sampled bilinearly over integer pixel centres
    (grid_sample, align_corners=True, zero padding); t0 defaults to the last timestamp."""
    if xt.dim() > 1:
        xt, yt, tt = xt.squeeze(), yt.squeeze(), tt.squeeze()
    if t0 is None:
        t0 = tt[-1]
    flow = flow_field
    while flow.dim() < 4:
        flow = flow.unsqueeze(0)
    H, W = flow.shape[-2], flow.shape[-1]
    grid = torch.stack((xt / (W - 1) * 2.0 - 1.0, yt / (H - 1) * 2.0 - 1.0), dim=1).reshape(1, 1, -1, 2)
    uv = F.grid_sample(flow, grid, align_corners=True)
    dt = (tt - t0).squeeze()
    return xt + uv[:, 0].squeeze() * dt, yt + uv[:, 1].squeeze() * dt
