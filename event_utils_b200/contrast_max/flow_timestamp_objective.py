"""The average-timestamp loss of Zhu et al. (CVPR'19) for a dense flow, as a batched, differentiable torch loss.

The other loss of self-supervised optical-flow training (EV-FlowNet and its successors): warp each sample's events by
the flow the network predicts (warp_events_flow_torch, lib/transforms/optic_flow.py:5-46), form the average-timestamp
images of the warped positive and negative events (events_to_timestamp_image_torch, lib/representations/image.py:286-353)
and sum their squares (zhu_timestamp_objective, lib/contrast_max/objectives.py:524-551).  One call evaluates a whole
batch on the GPU (evk_flow_timestamp_objective_f32) and its backward gives the exact gradient with respect to the flow
(evk_flow_timestamp_objective_grad_f32).
"""
from .. import _lib
from ..representations import _events as E
from ._batched import _normalised_stamps  # noqa: F401  (reached under this module's name as well)
from ._batched import _check_window_count, _event_tensors, _timestamp_events
from .flow_objective import _flow_batch


def flow_timestamp_objective_torch(xs, ys, ts, ps, flow, t0=None, blur_sigma=2.0, timestamp_reverse=False,
                                   batch_end_indices=None):
    """
    Average-timestamp loss f_b of every sample b of a batch of event windows warped by a dense flow.
    Sample b holds the events [start_b, end_b) of the concatenated stream, end_b = batch_end_indices[b] and start_b the
    previous end (0 for the first sample), and is warped by flow[b]:
      1. x' = x + u(x,y) d, y' = y + v(x,y) d with d = t - t0_b formed in ts' dtype, then f32 (grid_sample bilinear,
         zero padding, align_corners, optic_flow.py:37-44), exactly as flow_contrast_objective_torch warps.
      2. tau = (t - t_first_b) / (t_last_b - t_first_b + 1e-6), or (-t + t_last_b) / (...) with timestamp_reverse
         (image.py:324-327), formed in ts' dtype, then f32; t_first_b, t_last_b are the stamps of the sample's first and
         last event.  For f32 stamps this is bit for bit the normalised stamp of events_to_timestamp_image_torch.
      3. An event contributes iff 0 <= x' < W and 0 <= y' < H; other events are dropped (the reference would pile
         clipped events onto row and column 0, or wrap them, or raise IndexError).  An event whose x' or y' is not
         finite makes its sample's f NaN.  p > 0 is positive and p <= 0 negative (image.py:321-322); a NaN p is dropped.
      4. On the (H+1, W+1) canvas, per polarity s with k the bilinear tap weights: S_s = sum tau k, C_s = 1 + sum k (the
         counts start at one, image.py:338-352) and T_s = S_s / C_s.
      5. G_s = gaussian_filter(T_s, blur_sigma) (0: no blur, the paper's form) and
             f_b = sum(G_+^2) + sum(G_-^2),
         Zhu's loss, which training minimises.  It is the negation of zhu_timestamp_objective.evaluate_function, whose
         sign (objectives.py:550) lets the reference's minimiser maximise the loss.  The default blur_sigma 2.0 is that
         objective's default_blur.
    @param xs, ys, ts, ps the concatenated events, (N,) tensors or arrays; they are data, not differentiable
    @param flow (B,2,H,W) or (2,H,W) for one sample; the only differentiable input (expanded views work)
    @param t0 None (each sample's last timestamp), a number, or B values
    @param batch_end_indices the cumulative end indices of BaseVoxelDataset.collate_fn
           (lib/data_loaders/base_dataset.py:513-539), a list or an int64 tensor; None means one sample of all events
    @returns (B,) tensor of f in flow's dtype, on flow's device.  The backward is the exact derivative of f with
           respect to the flow, with the floor and keep decisions held.  It rounds the incoming gradient g_b to f32 and
           works in f32, so the gradient is accurate to f32 rounding whatever flow's dtype.  With every input already on
           the GPU neither the forward nor the backward synchronises with the host.
    """
    xs, ys, ts, ps = _event_tensors(xs, ys, ts, ps, t0, "flow_timestamp_objective_torch", "the flow")
    flow = _flow_batch(flow)
    B, H, W = flow.shape[0], flow.shape[2], flow.shape[3]
    _check_window_count(batch_end_indices, B, "flows")
    _lib.lib()
    dev = E.compute_device(flow, xs, ys, ts, ps)
    x, y, t_rel, tau, p, offsets = _timestamp_events(xs, ys, ts, ps, t0, batch_end_indices, B, dev, "flows", timestamp_reverse)
    from ..autograd import FlowTimestampObjective
    f = FlowTimestampObjective.apply(flow, x, y, t_rel, tau, p, offsets, float(blur_sigma))
    return f.to(device=flow.device, dtype=flow.dtype)

