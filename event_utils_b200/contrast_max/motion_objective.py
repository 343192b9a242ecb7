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
from ._batched import MAX_CANDIDATES  # noqa: F401  (a public name of this module)
from ._batched import (_batch_events, _candidates_tensor, _check_objective, _chunked_candidates, _depth_entry,
                       _depth_events, _depth_tensor, _event_tensors, _model, _params_tensor, _rows, _warp_code)


def motion_contrast_objective_torch(xs, ys, ts, ps, params, warpfunc, t0=None, objective="variance", blur_sigma=1.0,
                                    obj_param=None, img_size=(180, 240), batch_end_indices=None, inv_depth=None):
    """
    Contrast objective f_b of every sample b of a batch of event windows, each warped by its own motion params[b].
    Sample b holds the events [start_b, end_b) of the concatenated stream, end_b = batch_end_indices[b] and start_b the
    previous end (0 for the first sample).  With d = t - t0_b (formed in ts' dtype, then f32) and warpfunc's model in f32,
    in the order written:
        linvel_warp         (vx, vy)              x' = x - d vx,  y' = y - d vy               (warps.py:51-61)
        pure_rotation_warp  (cx, cy, omega)       rotation about (cx, cy) by omega d
        xyztheta_warp       (hx, hy, hz, theta)   about warpfunc.center
        affine_warp         (hx, hy, a11, a12, a21, a22)            about warpfunc.center (warps.py has the formulas)
        homography_warp     (hx, hy, a11, a12, a21, a22, g1, g2)    about warpfunc.center; an event past the horizon
                                                                    (w <= 0) is not kept
        camera_rotation_warp (wx, wy, wz)                           exact camera rotation with warpfunc's intrinsics;
                                                                    an event behind the camera (Pz <= 0) is not kept
        camera_motion_warp  (wx, wy, wz, vx, vy, vz)                exact camera rotation and translation with the
                                                                    events' inverse depth inv_depth (warps.py); an
                                                                    event behind the camera or with a negative or
                                                                    non-finite inverse depth is not kept
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
    @param warpfunc an instance of linvel_warp, pure_rotation_warp, xyztheta_warp, affine_warp, homography_warp,
           camera_rotation_warp or camera_motion_warp
    @param t0 None (each sample's last timestamp, get_iwe's ts[-1]), a number, or B values
    @param batch_end_indices the cumulative end indices of BaseVoxelDataset.collate_fn
           (lib/data_loaders/base_dataset.py:513-539), a list or an int64 tensor; None means one sample of all events
    @param inv_depth camera_motion_warp only (required there, rejected with any other model): the inverse depth 1/Z of
           every event's scene point at the event's time, an (N,) float tensor or array aligned with the concatenated
           events; data like them (taken to f32 on their device, no gradient)
    @returns (B,) tensor of f in params' dtype, on params' device.  With every input already on the GPU neither the
           forward nor the backward synchronises with the host.  The backward rounds the incoming gradient g_b to
           f32, as it stores W_b = G(g_b df_b/dG) in f32: the gradient is accurate to f32 rounding whatever
           params' dtype (f64 params do not give an f64-accurate gradient).
    """
    warp = _warp_code(warpfunc, "motion_contrast_objective_torch")
    _check_objective(objective, "parameters")
    xs, ys, ts, ps = _event_tensors(xs, ys, ts, ps, t0, "motion_contrast_objective_torch", "params")
    rho = _depth_tensor(inv_depth, warp, xs.shape[0], "motion_contrast_objective_torch")
    params = _params_tensor(params, warpfunc)
    B = params.shape[0]
    H, W = int(img_size[0]), int(img_size[1])
    _lib.lib()
    dev = E.compute_device(params, xs, ys, ts, ps)
    x, y, t_rel, p, offsets = _batch_events(xs, ys, ts, ps, t0, batch_end_indices, B, dev, "parameter vectors")
    from ..autograd import MotionObjective
    opts = _model(warp, warpfunc, objective, blur_sigma, obj_param, H, W)
    f = MotionObjective.apply(_rows(params, opts[1]), x, y, t_rel, p, offsets, opts, _depth_events(rho, dev))
    return f.to(device=params.device, dtype=params.dtype)


# The workspace of one evk_cmax_motion_candidates_f32 call stays below this many bytes: larger batches of windows run in
# chunks (28 bytes per canvas pixel and candidate: 4 GiB hold 109 windows x 32 candidates at 180x240).
CANDIDATES_WORKSPACE_BYTES = 4 << 30


def motion_contrast_candidates_torch(xs, ys, ts, ps, candidates, warpfunc, t0=None, objective="variance", blur_sigma=1.0,
                                     obj_param=None, img_size=(180, 240), batch_end_indices=None, inv_depth=None):
    """
    The contrast objective of every window b under each of its J candidate parameter vectors candidates[b, j]: f[b, j] is
    the f_b that motion_contrast_objective_torch returns with params[b] = candidates[b, j] (same windows, t0, objective,
    blur and canvas conventions).  Each pass over the events scores up to 32 candidates of every window
    (evk_cmax_motion_candidates_f32): this is the batched form of a grid search per window (grid_search_initial,
    events_cmax.py:241-311) and of the objective surface sample_objective_function draws, and the line search of
    motion_contrast_fit_torch.  J is split into passes of at most 32 candidates, and the windows into chunks whose
    workspace stays under CANDIDATES_WORKSPACE_BYTES; neither split changes a value's arithmetic.
    @param candidates (B,J,K) parameter vectors, any float dtype, K = warpfunc.dims, any J >= 1
    @param inv_depth camera_motion_warp's inverse depth of every event, as in motion_contrast_objective_torch
    @returns (B,J) f64 tensor of values (no autograd graph) on candidates' device
    """
    warp = _warp_code(warpfunc, "motion_contrast_candidates_torch")
    _check_objective(objective, "parameters")
    xs, ys, ts, ps = _event_tensors(xs, ys, ts, ps, t0, "motion_contrast_candidates_torch", "nothing")
    rho = _depth_tensor(inv_depth, warp, xs.shape[0], "motion_contrast_candidates_torch")
    cand = _candidates_tensor(candidates, warpfunc)
    B = cand.shape[0]
    H, W = int(img_size[0]), int(img_size[1])
    _lib.lib()
    dev = E.compute_device(cand, xs, ys, ts, ps)
    x, y, t_rel, p, offsets = _batch_events(xs, ys, ts, ps, t0, batch_end_indices, B, dev, "candidate sets")
    with torch.cuda.device(dev):
        c64 = cand.detach().to(device=dev, dtype=torch.float64)
        f = _candidates(x, y, t_rel, p, offsets, c64, _model(warp, warpfunc, objective, blur_sigma, obj_param, H, W),
                        _depth_events(rho, dev))
    return f.to(cand.device)


def _candidates(x, y, t_rel, p, offsets, c64, opts, rho=None):
    """f (B,J) f64 of the prepared device events under the device candidates c64 (B,J,K) f64, in passes of at most
    MAX_CANDIDATES candidates over chunks of windows whose workspace fits CANDIDATES_WORKSPACE_BYTES; rho: the device
    inverse depth of camera_motion_warp, or None"""
    warp, centre, H, W, objective, sigma, param = opts
    stem, events = _depth_entry("evk_cmax_motion_candidates", (x, y, t_rel, p), rho)
    return _chunked_candidates(stem, "motion_candidates", events, offsets, c64, (warp, centre, H, W), (sigma, objective, param),
                               CANDIDATES_WORKSPACE_BYTES, 65535)
