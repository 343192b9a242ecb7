"""Autograd for the torch functions whose reference versions are plain, differentiable torch ops.

The reference builds its event images, timestamp images and flow warp from `index_put_(accumulate=True)`,
`grid_sample` and weights made of `xs - floor(xs)` (image.py:46-100, image.py:286-353, optic_flow.py:5-46), so
autograd runs through them: flow -> warp -> event image -> loss -> backward() into the flow.  Our forwards are
CUDA kernels, so each function gets a torch.autograd.Function here whose forward is the existing kernel path
(bit-identical outputs) and whose backward is one pass of a kernel of csrc/evk_grad.cu.

Which inputs get a gradient (as in the reference; the others get None):
    events_to_image_torch            bilinear: xs, ys, ps;  nearest (or integer coordinates): ps
    events_to_timestamp_image_torch  xs, ys, ts
    warp_events_flow_torch           xt, yt, tt, flow_field, t0 (when it is a tensor; t0=None means tt[-1])
    events_to_voxel_torch            ps, ts (voxel_grid.py:114-153); also through voxel_grids_fixed_n/_t_torch and
                                     events_to_voxel_timesync_torch
    events_to_neg_pos_voxel_torch    ts (voxel_grid.py:155-182)
    flow_contrast_objective_torch    flow only (contrast_max/flow_objective.py; the events are data)
    flow_timestamp_objective_torch   flow only (contrast_max/flow_timestamp_objective.py; the events are data)
    grid_flow_contrast_objective_torch  the node grid only (contrast_max/grid_flow.py; the events are data)
    grid_flow_timestamp_objective_torch  the node grid only (contrast_max/grid_flow_timestamp.py; the events are data)
    depth_grid_contrast_objective_torch  the inverse-depth grid only (contrast_max/depth_grid.py; events and motion are data)
    motion_contrast_objective_torch  params only (contrast_max/motion_objective.py; the events are data)
    motion_segmentation_objective_torch  params and weights (contrast_max/motion_segmentation.py; the events are data)
    motion_timestamp_objective_torch params only (contrast_max/motion_timestamp_objective.py; the events are data)

The public functions take this path only when grad mode is on and one of those inputs requires grad; every
other call runs the plain forward.  Gradients come back in each input's shape, dtype and device.  The
backwards are not themselves differentiable (no double backward).
"""
import numpy as np
import torch
from torch.autograd.function import once_differentiable

from . import _lib


def _meta(t):
    return (t.shape, t.dtype, t.device) if isinstance(t, torch.Tensor) else None


def _as_input(g, meta):
    """A per-event gradient (flat f32 on the compute device) in the shape, dtype and device of its input."""
    if g is None or meta is None:
        return None
    shape, dtype, device = meta
    return g.reshape(shape).to(device=device, dtype=dtype)


def _grad_in(g, dev):
    """The incoming gradient as contiguous f32 on the compute device (autograd hands zeros for an unused output, and
    an expanded gradient such as the one of img.sum() has stride 0).  The backward kernels work in f32, so an f64
    incoming gradient (e.g. of the contrast objectives' f64 f) is rounded to f32 here."""
    return g.to(device=dev, dtype=torch.float32).contiguous()


class EventImage(torch.autograd.Function):
    """events_to_image_torch (image.py:46-100)."""

    @staticmethod
    def forward(ctx, xs, ys, ps, opts):
        from .representations.image import _image_device, _image_inputs
        device, sensor_size, clip, interpolation, padding, default = opts
        dev, (H, W), clipx, clipy, flags, x, y, p = _image_inputs(xs, ys, ps, sensor_size, clip, interpolation, padding)
        img = _image_device(x, y, p, H, W, clipx, clipy, flags, default)
        ctx.save_for_backward(x, y, p)
        ctx.geom = (dev, H, W, clipx, clipy, flags)
        ctx.metas = tuple(_meta(t) for t in (xs, ys, ps))
        return img if img.device == device else img.to(device)

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        x, y, p = ctx.saved_tensors
        dev, H, W, clipx, clipy, flags = ctx.geom
        bil = bool(flags & _lib.BILINEAR)
        need = ctx.needs_input_grad
        L = _lib.lib()
        with torch.cuda.device(dev):
            g = _grad_in(g, dev)
            gx = torch.empty_like(x) if bil and need[0] else None
            gy = torch.empty_like(y) if bil and need[1] else None
            gp = torch.empty_like(p) if need[2] else None
            _lib.check(L.evk_image_grad_f32(_lib.ptr(x), _lib.ptr(y), _lib.ptr(p), x.shape[0], H, W, clipx, clipy, flags,
                                            _lib.ptr(g), _lib.ptr(gx), _lib.ptr(gy), _lib.ptr(gp), _lib.stream()))
        return _as_input(gx, ctx.metas[0]), _as_input(gy, ctx.metas[1]), _as_input(gp, ctx.metas[2]), None


class TimestampImages(torch.autograd.Function):
    """events_to_timestamp_image_torch (image.py:286-353).  The forward also keeps the two count images."""

    @staticmethod
    def forward(ctx, xs, ys, ts, ps, opts):
        from .representations.image import _timestamp_images, _timestamp_inputs, _ts_canvas_and_clip, _ts_flags
        device, sensor_size, clip, interpolation, padding, reverse = opts
        dev, x, y, t, p, fl = _timestamp_inputs(xs, ys, ts, ps)
        pos, neg, cpos, cneg = _timestamp_images(x, y, t, p, fl[0], fl[1], sensor_size, clip, interpolation, padding,
                                                 reverse, counts=True)
        ctx.save_for_backward(x, y, t, p, pos, neg, cpos, cneg)
        _, clipx, clipy = _ts_canvas_and_clip(sensor_size, interpolation, padding)
        ctx.geom = (dev, fl[0], fl[1], clipx, clipy, _ts_flags(clip, reverse), reverse)
        ctx.metas = tuple(_meta(a) for a in (xs, ys, ts))
        if pos.device != device:
            pos, neg = pos.to(device), neg.to(device)
        return pos, neg

    @staticmethod
    @once_differentiable
    def backward(ctx, g_pos, g_neg):
        x, y, t, p, pos, neg, cpos, cneg = ctx.saved_tensors
        dev, t_first, t_last, clipx, clipy, flags, reverse = ctx.geom
        need = ctx.needs_input_grad
        H, W = pos.shape
        L = _lib.lib()
        with torch.cuda.device(dev):
            g_pos, g_neg = _grad_in(g_pos, dev), _grad_in(g_neg, dev)
            gx = torch.empty_like(x) if need[0] else None
            gy = torch.empty_like(y) if need[1] else None
            gt = torch.empty_like(t) if need[2] else None
            sums = torch.empty(2, dtype=torch.float64, device=dev)
            ws = torch.empty(L.evk_timestamp_image_grad_workspace_bytes(H, W), dtype=torch.uint8, device=dev)
            _lib.check(L.evk_timestamp_image_grad_f32(
                _lib.ptr(x), _lib.ptr(y), _lib.ptr(t), _lib.ptr(p), x.shape[0], t_first, t_last, H, W, clipx, clipy, flags,
                _lib.ptr(g_pos), _lib.ptr(g_neg), _lib.ptr(pos), _lib.ptr(neg), _lib.ptr(cpos), _lib.ptr(cneg),
                _lib.ptr(gx), _lib.ptr(gy), _lib.ptr(gt), _lib.ptr(sums), _lib.ptr(ws), ws.numel(), _lib.stream()))
            if gt is not None and gt.numel():
                # tn's denominator D = ts[-1] - ts[0] + 1e-6 (f32, as the kernels form it) also depends on ts[0], ts[-1]
                D = float(np.float32(np.float32(t_last) - np.float32(t_first)) + np.float32(1e-6))
                s0, s1 = sums[0], sums[1]
                if reverse:
                    d_first, d_last = s1 / D, (s0 - s1) / D
                else:
                    d_first, d_last = (s1 - s0) / D, -s1 / D
                gt[0] += d_first.to(torch.float32)
                gt[-1] += d_last.to(torch.float32)
        return _as_input(gx, ctx.metas[0]), _as_input(gy, ctx.metas[1]), _as_input(gt, ctx.metas[2]), None, None


class WarpFlow(torch.autograd.Function):
    """warp_events_flow_torch (optic_flow.py:5-46), with t0 a tensor (tt[-1] when the caller gave none, so that its
    gradient reaches the last event)."""

    @staticmethod
    def forward(ctx, xt, yt, tt, t0, flow_field, out_device):
        from .transforms.optic_flow import _flow_inputs, _warp_device
        dev, x, y, t, f = _flow_inputs(xt, yt, tt, flow_field)
        with torch.cuda.device(dev):
            # dt = tt - t0 in the dtype the plain path forms it in (the kernel's f32 subtraction for f32 stamps, the
            # input dtype's otherwise), then the kernel runs with t0 = 0: the same warped coordinates, bit for bit
            rt = torch.result_type(t, 1.0)
            t_rel = (t.to(rt) - t0.detach().to(device=dev, dtype=rt)).to(torch.float32).contiguous()
            xw, yw = _warp_device(x, y, t_rel, f, 0.0)
        ctx.save_for_backward(x, y, t_rel, f)
        ctx.dev = dev
        ctx.metas = tuple(_meta(a) for a in (xt, yt, tt, t0, flow_field))
        if xw.device != out_device:
            xw, yw = xw.to(out_device), yw.to(out_device)
        return xw, yw

    @staticmethod
    @once_differentiable
    def backward(ctx, g_xw, g_yw):
        x, y, t, f = ctx.saved_tensors
        dev = ctx.dev
        need = ctx.needs_input_grad
        H, W = f.shape[1], f.shape[2]
        L = _lib.lib()
        with torch.cuda.device(dev):
            g_xw, g_yw = _grad_in(g_xw, dev), _grad_in(g_yw, dev)
            gx = torch.empty_like(x) if need[0] else None
            gy = torch.empty_like(y) if need[1] else None
            gt = torch.empty_like(t) if need[2] or need[3] else None
            gf = torch.empty_like(f)
            s = torch.empty(1, dtype=torch.float64, device=dev)
            ws = torch.empty(L.evk_warp_flow_grad_workspace_bytes(H, W), dtype=torch.uint8, device=dev)
            _lib.check(L.evk_warp_flow_grad_f32(
                _lib.ptr(x), _lib.ptr(y), _lib.ptr(t), x.shape[0], _lib.ptr(f), H, W, 0.0, _lib.ptr(g_xw), _lib.ptr(g_yw),
                _lib.ptr(gx), _lib.ptr(gy), _lib.ptr(gt), _lib.ptr(gf), _lib.ptr(s), _lib.ptr(ws), ws.numel(), _lib.stream()))
        m = ctx.metas
        g_t0 = _as_input(-s, m[3]) if need[3] else None
        return (_as_input(gx, m[0]), _as_input(gy, m[1]), _as_input(gt, m[2]) if need[2] else None, g_t0,
                _as_input(gf, m[4]) if need[4] else None, None)


def _loss_entry(L, entry, events, offsets, d):
    """The arguments every entry of a batched loss starts with, and its scratch.  entry = (stem, scratch key, (M,) for
    a multi-model loss, the arguments in front of and behind the differentiable input d, (H, W), the arguments the
    workspace query takes in front of (H, W) besides the batch and M)."""
    stem, key, ms, pre, post, (H, W), query = entry
    B = d.shape[0]
    lead = tuple(_lib.ptr(a) for a in events) + ms + (_lib.ptr(offsets), B, events[0].shape[0]) + pre + (_lib.ptr(d),) + post
    ws = _lib.scratch(key, getattr(L, stem + "_workspace_bytes")(B, *ms, *query, H, W), d.device)
    return lead, ws


def _loss_forward(ctx, stem, key, inp, dtype, pre, post, size, events, offsets, images, weights=None, query=()):
    """The forward the batched losses share: f (B,) f64 of `stem`_f32 from inp in `dtype` on the events' device and the
    prepared device events.  `images` are the canvases per sample of each image the entry hands to `stem`_grad_f32.
    With the memberships `weights` (N,M), as f32 the last of the event arrays, the loss has M models: f is (B,M).
    `query`: the arguments `stem`_workspace_bytes takes between the batch and (H, W)."""
    dev = events[0].device
    L = _lib.lib()
    with torch.cuda.device(dev):
        d = inp.detach().to(device=dev, dtype=dtype).contiguous()
        ms = ()
        if weights is not None:
            events += (weights.detach().to(device=dev, dtype=torch.float32).contiguous(),)
            ms = (weights.shape[1],)
        B, (H, W) = d.shape[0], size
        f = torch.empty((B,) + ms, dtype=torch.float64, device=dev)
        imgs = [torch.empty((B, c, H + 1, W + 1), dtype=torch.float32, device=dev) for c in images]
        ctx.entry = (stem, key, ms, pre, post, size, query)
        lead, ws = _loss_entry(L, ctx.entry, events, offsets, d)
        _lib.check(getattr(L, stem + "_f32")(*lead, _lib.ptr(f), *(_lib.ptr(i) for i in imgs), _lib.ptr(ws), ws.numel(),
                                             _lib.stream()))
    ctx.save_for_backward(*events, offsets, d, *imgs)
    ctx.n_images = len(imgs)
    ctx.metas = (_meta(inp), _meta(weights))
    return f


def _loss_backward(ctx, g, weights_grad=False):
    """The backward the batched losses share: (gradient of inp, gradient of the memberships or None), one pass over the
    events (`stem`_grad_f32).  The membership gradient is only computed with weights_grad."""
    saved = ctx.saved_tensors
    k = len(saved) - ctx.n_images
    events, (offsets, d), imgs = saved[:k - 2], saved[k - 2:k], saved[k:]
    stem, ms = ctx.entry[0], ctx.entry[2]
    dev = d.device
    L = _lib.lib()
    with torch.cuda.device(dev):
        g = _grad_in(g, dev)
        gd = torch.empty_like(d)
        gw = torch.zeros_like(events[-1]) if weights_grad else None      # rows outside every window: 0
        lead, ws = _loss_entry(L, ctx.entry, events, offsets, d)
        _lib.check(getattr(L, stem + "_grad_f32")(*lead, *(_lib.ptr(i) for i in imgs), _lib.ptr(g), _lib.ptr(gd),
                                                  *((_lib.ptr(gw),) if ms else ()), _lib.ptr(ws), ws.numel(), _lib.stream()))
    return _as_input(gd, ctx.metas[0]), _as_input(gw, ctx.metas[1])


class FlowObjective(torch.autograd.Function):
    """The batched dense-flow contrast objective of contrast_max/flow_objective.py (draw_flow.py:15-26 followed by an
    objective of objectives.py): f (B,) f64 from flow (B,2,H,W) and the prepared device events.  Only the flow gets a
    gradient: the exact derivative of f, one pass over the events (evk_cmax_flow_objective_grad_f32)."""

    @staticmethod
    def forward(ctx, flow, x, y, t_rel, p, offsets, opts):
        objective, sigma, param = opts
        H, W = flow.shape[2:]
        return _loss_forward(ctx, "evk_cmax_flow_objective", "flow_objective", flow, torch.float32, (),
                             (H, W, sigma, objective, param), (H, W), (x, y, t_rel, p), offsets, (1,))

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        return _loss_backward(ctx, g)[:1] + (None,) * 6


class GridFlowObjective(torch.autograd.Function):
    """The batched grid-flow contrast objective of contrast_max/grid_flow.py (the dense-flow objective with the flow
    bilinearly interpolated from a gh x gw grid of nodes): f (B,) f64 from grid_flow (B,2,gh,gw) and the prepared device
    events.  Only the nodes get a gradient: the exact derivative of f, one pass over the events
    (evk_cmax_grid_flow_objective_grad_f32).  opts = (H, W, objective, sigma, obj_param)."""

    @staticmethod
    def forward(ctx, grid_flow, x, y, t_rel, p, offsets, opts):
        H, W, objective, sigma, param = opts
        gh, gw = grid_flow.shape[2:]
        return _loss_forward(ctx, "evk_cmax_grid_flow_objective", "grid_flow_objective", grid_flow, torch.float32, (),
                             (gh, gw, H, W, sigma, objective, param), (H, W), (x, y, t_rel, p), offsets, (1,),
                             query=(gh, gw))

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        return _loss_backward(ctx, g)[:1] + (None,) * 6


class DepthGridObjective(torch.autograd.Function):
    """The batched depth-grid contrast objective of contrast_max/depth_grid.py (the camera-motion contrast loss with each
    event's inverse depth bilinearly interpolated from a gh x gw grid of nodes): f (B,) f64 from inv_depth_grid
    (B,gh,gw) and the prepared device events.  Only the nodes get a gradient: the exact derivative of f, one pass over
    the events (evk_cmax_depth_grid_objective_grad_f32).  opts = (rows, cx, cy, H, W, sigma, objective, obj_param) with
    rows the device motion rows (B,8) f64 (_batched._rows)."""

    @staticmethod
    def forward(ctx, inv_depth_grid, x, y, t_rel, p, offsets, opts):
        rows, cx, cy, H, W, sigma, objective, param = opts
        gh, gw = inv_depth_grid.shape[1:]
        ctx.rows = rows   # the entries read the rows through a pointer, in the backward too
        return _loss_forward(ctx, "evk_cmax_depth_grid_objective", "depth_grid_objective", inv_depth_grid, torch.float32,
                             (_lib.ptr(rows), cx, cy), (gh, gw, H, W, sigma, objective, param), (H, W), (x, y, t_rel, p),
                             offsets, (1,), query=(gh, gw))

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        return _loss_backward(ctx, g)[:1] + (None,) * 6


class MotionAndDepthObjective(torch.autograd.Function):
    """The depth-grid contrast objective of DepthGridObjective, differentiable in the camera motion as well as in the
    nodes (contrast_max/motion_and_depth.py): f (B,) f64 from inv_depth_grid (B,gh,gw), motion (B,6) and the prepared
    device events.  The forward is evk_cmax_depth_grid_objective_f32's; the backward is one pass over the events
    (evk_cmax_depth_grid_joint_grad_f32) that returns both gradients.  opts = (centre (cx, cy, fx, fy), H, W, sigma,
    objective, obj_param)."""

    @staticmethod
    def forward(ctx, inv_depth_grid, motion, x, y, t_rel, p, offsets, opts):
        from .contrast_max._batched import _rows
        centre, H, W, sigma, objective, param = opts
        gh, gw = inv_depth_grid.shape[1:]
        with torch.cuda.device(x.device):
            rows = _rows(motion.detach().to(device=x.device, dtype=torch.float64), centre).contiguous()
        ctx.rows = rows   # the entries read the rows through a pointer, in the backward too
        ctx.motion_meta = _meta(motion)
        return _loss_forward(ctx, "evk_cmax_depth_grid_objective", "depth_grid_objective", inv_depth_grid, torch.float32,
                             (_lib.ptr(rows), centre[0], centre[1]), (gh, gw, H, W, sigma, objective, param), (H, W),
                             (x, y, t_rel, p), offsets, (1,), query=(gh, gw))

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        saved = ctx.saved_tensors
        events, offsets, d, iwe = saved[:4], saved[4], saved[5], saved[6]
        dev = d.device
        L = _lib.lib()
        with torch.cuda.device(dev):
            g = _grad_in(g, dev)
            gd = torch.empty_like(d)
            gm = torch.empty((d.shape[0], 6), dtype=torch.float64, device=dev)
            entry = ("evk_cmax_depth_grid_joint_grad",) + ctx.entry[1:]
            lead, ws = _loss_entry(L, entry, events, offsets, d)
            _lib.check(L.evk_cmax_depth_grid_joint_grad_f32(*lead, _lib.ptr(iwe), _lib.ptr(g), _lib.ptr(gd), _lib.ptr(gm),
                                                            _lib.ptr(ws), ws.numel(), _lib.stream()))
        return (_as_input(gd, ctx.metas[0]), _as_input(gm, ctx.motion_meta)) + (None,) * 6


class FlowTimestampObjective(torch.autograd.Function):
    """The batched dense-flow average-timestamp loss of contrast_max/flow_timestamp_objective.py (optic_flow.py:5-46,
    image.py:286-353, then the sum of squares of objectives.py:524-551): f (B,) f64 from flow (B,2,H,W) and the prepared
    device events with their normalised stamps tau.  Only the flow gets a gradient: the exact derivative of f, one pass
    over the events (evk_flow_timestamp_objective_grad_f32).  The forward keeps the timestamp and count images."""

    @staticmethod
    def forward(ctx, flow, x, y, t_rel, tau, p, offsets, sigma):
        H, W = flow.shape[2:]
        return _loss_forward(ctx, "evk_flow_timestamp_objective", "flow_timestamp_objective", flow, torch.float32, (),
                             (H, W, sigma), (H, W), (x, y, t_rel, tau, p), offsets, (2, 2))

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        return _loss_backward(ctx, g)[:1] + (None,) * 7


class GridFlowTimestampObjective(torch.autograd.Function):
    """The batched grid-flow average-timestamp loss of contrast_max/grid_flow_timestamp.py (the dense-flow timestamp loss
    with the flow bilinearly interpolated from a gh x gw grid of nodes): f (B,) f64 from grid_flow (B,2,gh,gw) and the
    prepared device events with their normalised stamps tau.  Only the nodes get a gradient: the exact derivative of f,
    one pass over the events (evk_grid_flow_timestamp_objective_grad_f32).  The forward keeps the timestamp and count
    images.  opts = (H, W, sigma)."""

    @staticmethod
    def forward(ctx, grid_flow, x, y, t_rel, tau, p, offsets, opts):
        H, W, sigma = opts
        gh, gw = grid_flow.shape[2:]
        return _loss_forward(ctx, "evk_grid_flow_timestamp_objective", "grid_flow_timestamp_objective", grid_flow,
                             torch.float32, (), (gh, gw, H, W, sigma), (H, W), (x, y, t_rel, tau, p), offsets, (2, 2),
                             query=(gh, gw))

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        return _loss_backward(ctx, g)[:1] + (None,) * 7


class DepthGridTimestampObjective(torch.autograd.Function):
    """The batched depth-grid average-timestamp loss of contrast_max/depth_grid_timestamp.py (the camera-motion timestamp
    loss with each event's inverse depth bilinearly interpolated from a gh x gw grid of nodes): f (B,) f64 from
    inv_depth_grid (B,gh,gw) and the prepared device events with their normalised stamps tau.  Only the nodes get a
    gradient: the exact derivative of f, one pass over the events (evk_depth_grid_timestamp_objective_grad_f32).  The
    forward keeps the timestamp and count images.  opts = (rows, cx, cy, H, W, sigma) with rows the device motion rows
    (B,8) f64 (_batched._rows)."""

    @staticmethod
    def forward(ctx, inv_depth_grid, x, y, t_rel, tau, p, offsets, opts):
        rows, cx, cy, H, W, sigma = opts
        gh, gw = inv_depth_grid.shape[1:]
        ctx.rows = rows   # the entries read the rows through a pointer, in the backward too
        return _loss_forward(ctx, "evk_depth_grid_timestamp_objective", "depth_grid_timestamp_objective", inv_depth_grid,
                             torch.float32, (_lib.ptr(rows), cx, cy), (gh, gw, H, W, sigma), (H, W), (x, y, t_rel, tau, p),
                             offsets, (2, 2), query=(gh, gw))

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        return _loss_backward(ctx, g)[:1] + (None,) * 7


class MotionObjective(torch.autograd.Function):
    """The batched parametric contrast objective of contrast_max/motion_objective.py (get_iwe, objectives.py:184-192, with
    the linvel, rotation or 4-DoF model, then an objective of objectives.py): f (B,) f64 from params (B,K) and the
    prepared device events.  Only the parameters get a gradient: the exact derivative of f, one pass over the events
    (evk_cmax_motion_objective_grad_f32).  opts = (warp code, centre, H, W, objective, sigma, obj_param); params are the
    rows the entries take (contrast_max/_batched._rows), so K = 5 for the camera rotation and 8 for the camera motion.
    rho: None, or camera_motion_warp's inverse depth of every event (f32 on the events' device), which routes the loss to
    the depth entries (evk_cmax_motion_depth_objective_f32 / _grad_f32); it gets no gradient."""

    @staticmethod
    def forward(ctx, params, x, y, t_rel, p, offsets, opts, rho=None):
        from .contrast_max._batched import _depth_entry
        warp, centre, H, W, objective, sigma, param = opts
        cx, cy = centre[:2]
        stem, events = _depth_entry("evk_cmax_motion_objective", (x, y, t_rel, p), rho)
        return _loss_forward(ctx, stem, "motion_objective", params, torch.float64, (warp,),
                             (params.shape[-1], cx, cy, H, W, sigma, objective, param), (H, W), events, offsets, (1,))

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        return _loss_backward(ctx, g)[:1] + (None,) * 7


class MotionSegmentationObjective(torch.autograd.Function):
    """The weighted multi-model contrast of contrast_max/motion_segmentation.py: f (B,M) f64 from params (B,M,K), the
    memberships weights (N,M) and the prepared device events.  The parameters and the memberships get gradients, one
    pass over the events for both (evk_cmax_motion_segment_grad_f32); the membership gradient only when weights
    requires grad.  opts = (warp code, centre, H, W, objective, sigma, obj_param); params are the entries' rows
    (_batched._rows)."""

    @staticmethod
    def forward(ctx, params, weights, x, y, t_rel, p, offsets, opts):
        warp, centre, H, W, objective, sigma, param = opts
        cx, cy = centre[:2]
        return _loss_forward(ctx, "evk_cmax_motion_segment", "motion_segment", params, torch.float64, (warp,),
                             (params.shape[-1], cx, cy, H, W, sigma, objective, param), (H, W), (x, y, t_rel, p), offsets,
                             (weights.shape[1],), weights)

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        return _loss_backward(ctx, g, ctx.needs_input_grad[1]) + (None,) * 6


class MotionTimestampObjective(torch.autograd.Function):
    """The batched parametric average-timestamp loss of contrast_max/motion_timestamp_objective.py
    (zhu_timestamp_objective, objectives.py:524-558, with the linvel, rotation or 4-DoF model): f (B,) f64 from params
    (B,K) and the prepared device events with their normalised stamps tau.  Only the parameters get a gradient: the exact
    derivative of f, one pass over the events (evk_motion_timestamp_objective_grad_f32).  The forward keeps the timestamp
    and count images.  opts = (warp code, centre, H, W, sigma); params are the entries' rows (_batched._rows).  rho is
    MotionObjective's: camera_motion_warp's inverse depth, through the depth entries, or None."""

    @staticmethod
    def forward(ctx, params, x, y, t_rel, tau, p, offsets, opts, rho=None):
        from .contrast_max._batched import _depth_entry
        warp, centre, H, W, sigma = opts
        cx, cy = centre[:2]
        stem, events = _depth_entry("evk_motion_timestamp_objective", (x, y, t_rel, tau, p), rho)
        return _loss_forward(ctx, stem, "motion_timestamp_objective", params, torch.float64,
                             (warp,), (params.shape[-1], cx, cy, H, W, sigma), (H, W), events, offsets, (2, 2))

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        return _loss_backward(ctx, g)[:1] + (None,) * 8


class VoxelGrid(torch.autograd.Function):
    """events_to_voxel_torch (voxel_grid.py:114-153), both grids of events_to_neg_pos_voxel_torch (:155-182, one
    (2,B,H,W) output) and the stacked (nw,B,H,W) windows of voxel_grids_fixed_n/_t_torch (:37-80).  opts = (device,
    B, H, W, negpos, windows) with windows None or (starts, ends).  Each grid or window is normalised by its own first
    and last stamp, so those two stamps get extra gradient terms (evk.h, evk_voxel_grad_f32)."""

    @staticmethod
    def forward(ctx, xs, ys, ts, ps, opts):
        from .representations import _events as E
        from .representations.voxel_grid import _device_events, _negpos_device, _voxel_device, _windows_device
        device, B, H, W, negpos, windows = opts
        dev = E.compute_device(xs, ys, ts, ps)
        aos = pairs = None
        overlap = False
        if windows is not None:
            starts, ends = windows
            x, y, t, p = xs, ys, ts, ps
            out, pairs = _windows_device(xs, ys, ts, ps, starts, ends, B, H, W)
            s, e = np.asarray(starts), np.asarray(ends)
            order = np.argsort(s, kind="stable")
            s, e = s[order], e[order]
            # searchsorted ends of voxel_grids_fixed_t_torch can reach past the next window's start through rounding
            overlap = bool(len(s) > 1 and (np.maximum.accumulate(e)[:-1] > s[1:]).any())
        else:
            # host inputs are uploaded: the backward runs on the device
            aos, x, y, t, p, t0, dt, flags = _device_events(xs, ys, ts, ps, dev, aos_ok=not negpos)
            out = _negpos_device(x, y, t, p, t0, dt, B, H, W, flags) if negpos else \
                _voxel_device(x, y, t, p, t0, dt, B, H, W, flags=flags, aos=aos)
        ctx.save_for_backward(aos, x, y, t, p, pairs)
        ctx.geom = (dev, B, H, W, negpos, overlap)
        ctx.metas = (_meta(ts), _meta(ps))
        return out if out.device == device else out.to(device)

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        aos, x, y, t, p, pairs = ctx.saved_tensors
        dev, B, H, W, negpos, overlap = ctx.geom
        need = ctx.needs_input_grad
        n = (aos if aos is not None else x).shape[0]
        nw = 1 if pairs is None else pairs.shape[0] // 2
        flags = ((_lib.WINDOW_NEGPOS if negpos else 0) | (_lib.WINDOW_OVERLAP if overlap else 0) |
                 (_lib.EVENTS_AOS if aos is not None else 0))
        L = _lib.lib()
        with torch.cuda.device(dev):
            g = _grad_in(g, dev)
            gt = torch.empty(n, dtype=torch.float32, device=dev) if need[2] else None
            gp = torch.empty(n, dtype=torch.float32, device=dev) if need[3] and not negpos else None
            ws = torch.empty(L.evk_voxel_grad_workspace_bytes(nw, B, H, W, flags), dtype=torch.uint8, device=dev)
            _lib.check(L.evk_voxel_grad_f32(
                _lib.ptr(aos if aos is not None else x), _lib.ptr(y), _lib.ptr(t), _lib.ptr(p), n, _lib.ptr(pairs), nw,
                B, H, W, flags, _lib.ptr(g), _lib.ptr(gp), _lib.ptr(gt), _lib.ptr(ws), ws.numel(), _lib.stream()))
        return None, None, _as_input(gt, ctx.metas[0]), _as_input(gp, ctx.metas[1]), None
