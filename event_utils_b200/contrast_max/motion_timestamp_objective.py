"""The average-timestamp loss of Zhu et al. (CVPR'19) for the linvel, rotation and 4-DoF motion models, as a batched,
differentiable torch loss.

The reference defines this loss in its parametric form only: zhu_timestamp_objective (lib/contrast_max/objectives.py:
524-558) warps a window's events with a warp_function and sums the squares of the blurred average-timestamp images of the
warped positive and negative events.  Here one call scores every window b with its own parameters params[b] on the GPU
(evk_motion_timestamp_objective_f32), and its backward gives the exact gradient with respect to params
(evk_motion_timestamp_objective_grad_f32), so a network that regresses angular velocity or ego-motion per window can
train on it.
"""
import torch

from .. import _lib
from ..representations import _events as E
from .flow_objective import _batch_events, _event_tensors
from .flow_timestamp_objective import _normalised_stamps
from .motion_objective import _WARPS


def motion_timestamp_objective_torch(xs, ys, ts, ps, params, warpfunc, t0=None, blur_sigma=2.0, timestamp_reverse=False,
                                     img_size=(180, 240), batch_end_indices=None):
    """
    Average-timestamp loss f_b of every sample b of a batch of event windows, each warped by its own motion params[b].
    Sample b holds the events [start_b, end_b) of the concatenated stream, end_b = batch_end_indices[b] and start_b the
    previous end (0 for the first sample):
      1. d = t - t0_b formed in ts' dtype, then f32, and warpfunc's model in f32, in the order written, exactly as
         motion_contrast_objective_torch warps:
             linvel_warp         (vx, vy)              x' = x - d vx,  y' = y - d vy               (warps.py:51-61)
             pure_rotation_warp  (cx, cy, omega)       rotation about (cx, cy) by omega d
             xyztheta_warp       (hx, hy, hz, theta)   about warpfunc.center
      2. tau = (t - t_first_b) / (t_last_b - t_first_b + 1e-6), or (-t + t_last_b) / (...) with timestamp_reverse
         (image.py:324-327), formed in ts' dtype, then f32, as flow_timestamp_objective_torch forms it.
      3. An event contributes iff its f32 x', y' are finite, 0 < x' < W and 0 < y' < H with (H, W) = img_size: those are
         the events whose splat in motion_contrast_objective_torch is not zero (the bounds mask 0 < x' <= W of
         event_util.py:26-27, then the clip that gives x' = W zero weight).  The others add to neither S nor C; a
         non-finite x' or y' contributes nothing and does not make f NaN.  The reference instead zeroes the masked events
         and piles them at (0, 0) as events with p = 0 and t = 0 (objectives.py:543-545), which darkens the negative
         image's corner pixel.  p > 0 is positive and p <= 0 negative (image.py:321-322); a NaN p is dropped.
      4. On the (H+1, W+1) canvas, per polarity s with k the bilinear tap weights: S_s = sum tau k, C_s = 1 + sum k and
         T_s = S_s / C_s.  Then G_s = gaussian_filter(T_s, blur_sigma) (0: no blur) and
             f_b = sum(G_+^2) + sum(G_-^2),
         Zhu's loss, which training minimises.  It is the negation of zhu_timestamp_objective.evaluate_function, whose
         sign (objectives.py:550) lets the reference's minimiser maximise the loss; that class is unchanged.
    @param xs, ys, ts, ps the concatenated events, (N,) tensors or arrays; they are data, not differentiable
    @param params (B,K) or (K,) for one sample, K = warpfunc.dims, any float dtype; the only differentiable input
           (expanded views work)
    @param warpfunc an instance of linvel_warp, pure_rotation_warp or xyztheta_warp
    @param t0 None (each sample's last timestamp, zhu_timestamp_objective's ts[-1]), a number, or B values
    @param img_size (H, W): the bounds of step 3 and the canvas (H+1, W+1)
    @param batch_end_indices the cumulative end indices of BaseVoxelDataset.collate_fn
           (lib/data_loaders/base_dataset.py:513-539), a list or an int64 tensor; None means one sample of all events
    @returns (B,) tensor of f in params' dtype, on params' device, 0 <= B <= 32767.  The backward is the exact derivative
           of f with respect to params, with the floor and keep decisions held.  It rounds the incoming gradient g_b to
           f32 and stores the images in f32, so the gradient is accurate to f32 rounding whatever params' dtype.  With
           every input already on the GPU neither the forward nor the backward synchronises with the host.
    """
    warp = next((code for cls, code in _WARPS if type(warpfunc) is cls), None)
    if warp is None:
        raise ValueError("motion_timestamp_objective_torch supports the models linvel_warp, pure_rotation_warp and "
                         "xyztheta_warp, got %s" % type(warpfunc).__name__)
    xs, ys, ts, ps = _event_tensors(xs, ys, ts, ps, t0, "motion_timestamp_objective_torch", "params")
    params = E.as_tensor(params)
    if not params.is_floating_point():
        raise ValueError("params must be a floating-point tensor, got %s" % params.dtype)
    if params.dim() == 1:
        params = params.unsqueeze(0)
    if params.dim() != 2 or params.shape[1] != warpfunc.dims:
        raise ValueError("params must have shape (B,%d) or (%d,) for %s, got %s"
                         % (warpfunc.dims, warpfunc.dims, type(warpfunc).__name__, tuple(params.shape)))
    B = params.shape[0]
    if batch_end_indices is not None:
        n_samples = (batch_end_indices.reshape(-1).shape[0] if isinstance(batch_end_indices, torch.Tensor)
                     else len(batch_end_indices))
        if n_samples != B:
            raise ValueError("%d samples of events for a batch of %d parameter vectors" % (n_samples, B))
    H, W = int(img_size[0]), int(img_size[1])
    _lib.lib()
    dev = E.compute_device(params, xs, ys, ts, ps)
    x, y, t_rel, p, offsets, t, sample = _batch_events(xs, ys, ts, ps, t0, batch_end_indices, B, dev, "parameter vectors",
                                                       stamps=True)
    with torch.cuda.device(dev):
        tau = _normalised_stamps(t, sample, offsets, timestamp_reverse)
    from ..autograd import MotionTimestampObjective
    centre = tuple(float(c) for c in warpfunc.center) if warp == _lib.WARP_XYZTHETA else (0.0, 0.0)
    f = MotionTimestampObjective.apply(params, x, y, t_rel, tau, p, offsets, (warp, centre, H, W, float(blur_sigma)))
    return f.to(device=params.device, dtype=params.dtype)
