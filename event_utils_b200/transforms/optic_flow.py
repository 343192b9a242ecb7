"""Dense-flow event warp -- drop-in for the reference's lib/transforms/optic_flow.py."""
import torch

from .. import _lib
from ..representations import _events as E


def warp_events_flow_torch(xt, yt, tt, pt, flow_field, t0=None,
        batched=False, batch_indices=None):
    """
    Warp events by a per-pixel flow field: x' = x + u(x,y)*(t-t0), y' = y + v(x,y)*(t-t0).
    Drop-in for optic_flow.py:5-46: flow sampled bilinearly at the event position over integer
    pixel centres (grid_sample, align_corners=True), neighbours outside the field count as zero.
    @param xt, yt, tt, pt event components, shape (N,) or (N,1) (pt is unused, as in the reference)
    @param flow_field (2,H,W) or (1,2,H,W) tensor
    @param t0 reference time (default: the last timestamp)
    @returns warped_xt, warped_yt (shape (N,))
    Differentiable like the reference w.r.t. xt, yt, tt, flow_field and t0 (event_utils_b200.autograd).
    """
    _lib.lib()
    xt, yt, tt = (E.as_tensor(a) for a in (xt, yt, tt))
    out_device = xt.device
    if len(xt.shape) > 1:
        xt, yt, tt = xt.squeeze(), yt.squeeze(), tt.squeeze()
    if t0 is None:
        t0 = tt[-1]
    if E.needs_grad(xt, yt, tt, t0, flow_field):
        from ..autograd import WarpFlow
        if not isinstance(t0, torch.Tensor):
            t0 = torch.tensor(t0, dtype=torch.float64)
        return WarpFlow.apply(xt, yt, tt, t0, flow_field, out_device)
    t0 = float(t0)
    dev, x, y, t, f = _flow_inputs(xt, yt, tt, flow_field)
    with torch.cuda.device(dev):
        if t.dtype != torch.float32:
            # the reference forms dt = tt - t0 in the INPUT dtype (optic_flow.py:33): absolute float64 / integer
            # stamps must not be rounded to float32 before the subtraction.  Pass the relative times, t0 = 0.
            t = (t - t0).to(torch.float32).contiguous()
            t0 = 0.0
        else:
            t = t.contiguous()
        xw, yw = _warp_device(x, y, t, f, t0)
    if xw.device != out_device:
        xw, yw = xw.to(out_device), yw.to(out_device)
    return xw, yw


def _flow_inputs(xt, yt, tt, flow_field):
    """warp_events_flow_torch's kernel inputs: compute device, f32 x, y, the stamps on the device (input dtype) and the
    f32 [2][H][W] flow."""
    flow = E.as_tensor(flow_field)
    while flow.dim() < 4:
        flow = flow.unsqueeze(0)
    if flow.shape[0] != 1 or flow.shape[1] != 2:
        raise RuntimeError("flow_field must have shape (2,H,W) or (1,2,H,W), got %s" % (tuple(flow_field.shape),))
    dev = E.compute_device(xt, yt, tt, flow)
    with torch.cuda.device(dev):
        x, y = (a.reshape(-1).to(dev).to(torch.float32).contiguous() for a in (xt, yt))
        t = tt.reshape(-1).to(dev)
        f = flow[0].to(dev).to(torch.float32).contiguous()
    return dev, x, y, t, f


def _warp_device(x, y, t, f, t0):
    L = _lib.lib()
    with torch.cuda.device(x.device):
        xw, yw = torch.empty_like(x), torch.empty_like(y)
        ws = _lib.scratch("flow_ws", L.evk_warp_flow_workspace_bytes(f.shape[1], f.shape[2]), x.device)
        _lib.check(L.evk_warp_flow_f32(_lib.ptr(x), _lib.ptr(y), _lib.ptr(t), x.shape[0], _lib.ptr(f),
                                       f.shape[1], f.shape[2], t0, _lib.ptr(xw), _lib.ptr(yw), _lib.ptr(ws), ws.numel(),
                                       _lib.stream()))
    return xw, yw
