"""Dense-flow contrast maximisation as a batched, differentiable torch loss.

The loss of self-supervised optical-flow training: warp each sample's events by the flow the network predicts
(warp_events_flow_torch, lib/transforms/optic_flow.py:37-44), form the bilinear image of warped events as the
reference's motion_compensate does (lib/visualization/draw_flow.py:15-26) and score its contrast with an objective of
lib/contrast_max/objectives.py.  One call evaluates a whole batch on the GPU (evk_cmax_flow_objective_f32) and its
backward gives the exact gradient of the returned f with respect to the flow (evk_cmax_flow_objective_grad_f32).
"""
from .. import _lib
from ..representations import _events as E
from ._batched import DEFAULT_PARAM, OBJECTIVES, _batch_events, _check_objective, _event_tensors


def flow_contrast_objective_torch(xs, ys, ts, ps, flow, t0=None, objective="variance", blur_sigma=1.0, obj_param=None,
                                  batch_end_indices=None):
    """
    Contrast objective f_b of every sample b of a batch of event windows warped by a dense flow.
    Sample b holds the events [start_b, end_b) of the concatenated stream, end_b = batch_end_indices[b] and start_b the
    previous end (0 for the first sample), and is warped by flow[b]: x' = x + u(x,y) (t - t0_b), y' = y + v(x,y) (t - t0_b)
    (grid_sample bilinear, zero padding, align_corners, optic_flow.py:37-44; t - t0_b is formed in ts' dtype, then f32).
    The image of warped events is the bilinear events_to_image_torch canvas (H+1, W+1) with padding (draw_flow.py:18-21),
    to which an event contributes iff 0 <= x' < W and 0 <= y' < H; other events are dropped (no IndexError, no wrap to
    the opposite border).  An event whose warped position is not finite makes its sample's f NaN.  Then
    G = gaussian_filter(image, blur_sigma) (0: no blur) and
        variance  -var(G)        sos  -mean(G^2)        soe  -mean(exp G)        sosa  -sum(exp(-obj_param G))
    ('moa' and 'isoa' are piecewise constant in the flow and are rejected).
    @param xs, ys, ts, ps the concatenated events, (N,) tensors or arrays; they are data, not differentiable
    @param flow (B,2,H,W) or (2,H,W) for one sample; the only differentiable input (expanded views work)
    @param t0 None (each sample's last timestamp), a number, or B values
    @param batch_end_indices the cumulative end indices of BaseVoxelDataset.collate_fn
           (lib/data_loaders/base_dataset.py:513-539), a list or an int64 tensor; None means one sample of all events
    @returns (B,) tensor of f in flow's dtype, on flow's device.  With every input already on the GPU neither the
           forward nor the backward synchronises with the host.  The backward rounds the incoming gradient g_b to
           f32, as it stores W_b = G(g_b df_b/dG) in f32: the gradient is accurate to f32 rounding whatever
           flow's dtype (an f64 flow does not give an f64-accurate gradient).
    """
    _check_objective(objective, "flow")
    xs, ys, ts, ps = _event_tensors(xs, ys, ts, ps, t0, "flow_contrast_objective_torch", "the flow")
    flow = _flow_batch(flow)
    B, H, W = flow.shape[0], flow.shape[2], flow.shape[3]
    _lib.lib()
    dev = E.compute_device(flow, xs, ys, ts, ps)
    x, y, t_rel, p, offsets = _batch_events(xs, ys, ts, ps, t0, batch_end_indices, B, dev, "flows")
    from ..autograd import FlowObjective
    param = float(obj_param if obj_param is not None else DEFAULT_PARAM.get(objective, 0.0))
    f = FlowObjective.apply(flow, x, y, t_rel, p, offsets, (OBJECTIVES[objective], float(blur_sigma), param))
    return f.to(device=flow.device, dtype=flow.dtype)


def _flow_batch(flow):
    """flow as a (B,2,H,W) tensor ((2,H,W) is one sample)"""
    flow = E.as_tensor(flow)
    if flow.dim() == 3:
        flow = flow.unsqueeze(0)
    if flow.dim() != 4 or flow.shape[1] != 2:
        raise ValueError("flow must have shape (B,2,H,W) or (2,H,W), got %s" % (tuple(flow.shape),))
    return flow
