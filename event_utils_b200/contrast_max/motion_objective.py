"""Parametric contrast maximisation (linvel, rotation, 4-DoF motion) as a batched, differentiable torch loss.

Fits of one motion per event window -- angular velocity per window of a rotation sequence, or a network that regresses
ego-motion per window and trains on the contrast -- evaluate many windows at once.  One call scores every window b with
its own parameters params[b], with the semantics of the single-window fast-mode evaluation (evk_cmax_warp_objective_f32 /
evk_cmax_linvel_objective_f32: get_iwe, lib/contrast_max/objectives.py:184-192, then an objective of that file), on the
GPU (evk_cmax_motion_objective_f32); its backward gives the exact gradient of the returned f with respect to params
(evk_cmax_motion_objective_grad_f32).
"""
import torch

from .. import _lib
from ..representations import _events as E
from .flow_objective import DEFAULT_PARAM, OBJECTIVES, _batch_events, _check_objective, _event_tensors
from .warps import linvel_warp, pure_rotation_warp, xyztheta_warp

_WARPS = ((linvel_warp, _lib.WARP_LINVEL), (pure_rotation_warp, _lib.WARP_ROTATION), (xyztheta_warp, _lib.WARP_XYZTHETA))


def motion_contrast_objective_torch(xs, ys, ts, ps, params, warpfunc, t0=None, objective="variance", blur_sigma=1.0,
                                    obj_param=None, img_size=(180, 240), batch_end_indices=None):
    """
    Contrast objective f_b of every sample b of a batch of event windows, each warped by its own motion params[b].
    Sample b holds the events [start_b, end_b) of the concatenated stream, end_b = batch_end_indices[b] and start_b the
    previous end (0 for the first sample).  With d = t - t0_b (formed in ts' dtype, then f32) and warpfunc's model in f32,
    in the order written:
        linvel_warp         (vx, vy)              x' = x - d vx,  y' = y - d vy               (warps.py:51-61)
        pure_rotation_warp  (cx, cy, omega)       rotation about (cx, cy) by omega d
        xyztheta_warp       (hx, hy, hz, theta)   about warpfunc.center
    An event is kept iff 0 < x' <= W and 0 < y' <= H with (H, W) = img_size (events_bounds_mask, event_util.py:26-27; a
    NaN position compares false and is kept, then contributes nothing, as in the single-window evaluation) and is splatted
    bilinearly on the (H+1, W+1) canvas (events_to_image_drv, image.py:179-217).  Then G = gaussian_filter(IWE,
    blur_sigma) (0: no blur) and
        variance  -var(G)        sos  -mean(G^2)        soe  -mean(exp G)        sosa  -sum(exp(-obj_param G))
    ('moa' and 'isoa' are piecewise constant in the parameters and are rejected).  With img_size = (180, 240) the canvas
    is get_iwe's fixed one, and f_b is what objective.evaluate_function returns for window b in precision="f32" mode.
    The backward is the exact derivative of the returned f_b with respect to params[b], with the floor and keep decisions
    held.  For linvel_warp it is therefore not the reference's evaluate_gradient (objectives.py:251-264), which mixes the
    two gradient channels in its 3-D blur and multiplies by the un-blurred IWE; with a blur, the variance and sos
    gradients of evaluate_gradient differ from it for every model for the second reason.
    ps is used as given: pass ps.abs() to match the reference's soe, sosa and isoa objectives (use_polarity=False).
    @param xs, ys, ts, ps the concatenated events, (N,) tensors or arrays; they are data, not differentiable
    @param params (B,K) or (K,) for one sample, K = warpfunc.dims, any float dtype; the only differentiable input
           (expanded views work)
    @param warpfunc an instance of linvel_warp, pure_rotation_warp or xyztheta_warp
    @param t0 None (each sample's last timestamp, get_iwe's ts[-1]), a number, or B values
    @param batch_end_indices the cumulative end indices of BaseVoxelDataset.collate_fn
           (lib/data_loaders/base_dataset.py:513-539), a list or an int64 tensor; None means one sample of all events
    @returns (B,) tensor of f in params' dtype, on params' device.  With every input already on the GPU neither the
           forward nor the backward synchronises with the host.  The backward rounds the incoming gradient g_b to
           f32, as it stores W_b = G(g_b df_b/dG) in f32: the gradient is accurate to f32 rounding whatever
           params' dtype (f64 params do not give an f64-accurate gradient).
    """
    warp = next((code for cls, code in _WARPS if type(warpfunc) is cls), None)
    if warp is None:
        raise ValueError("motion_contrast_objective_torch supports the models linvel_warp, pure_rotation_warp and "
                         "xyztheta_warp, got %s" % type(warpfunc).__name__)
    _check_objective(objective, "parameters")
    xs, ys, ts, ps = _event_tensors(xs, ys, ts, ps, t0, "motion_contrast_objective_torch", "params")
    params = E.as_tensor(params)
    if not params.is_floating_point():
        raise ValueError("params must be a floating-point tensor, got %s" % params.dtype)
    if params.dim() == 1:
        params = params.unsqueeze(0)
    if params.dim() != 2 or params.shape[1] != warpfunc.dims:
        raise ValueError("params must have shape (B,%d) or (%d,) for %s, got %s"
                         % (warpfunc.dims, warpfunc.dims, type(warpfunc).__name__, tuple(params.shape)))
    B = params.shape[0]
    H, W = int(img_size[0]), int(img_size[1])
    _lib.lib()
    dev = E.compute_device(params, xs, ys, ts, ps)
    x, y, t_rel, p, offsets = _batch_events(xs, ys, ts, ps, t0, batch_end_indices, B, dev, "parameter vectors")
    from ..autograd import MotionObjective
    centre = tuple(float(c) for c in warpfunc.center) if warp == _lib.WARP_XYZTHETA else (0.0, 0.0)
    param = float(obj_param if obj_param is not None else DEFAULT_PARAM.get(objective, 0.0))
    f = MotionObjective.apply(params, x, y, t_rel, p, offsets,
                              (warp, centre, H, W, OBJECTIVES[objective], float(blur_sigma), param))
    return f.to(device=params.device, dtype=params.dtype)
