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
from ._batched import (_candidates_tensor, _check_window_count, _chunked_candidates, _depth_entry, _depth_events,
                       _depth_tensor, _event_tensors, _params_tensor, _rows, _timestamp_events, _ts_model, _warp_code)


def motion_timestamp_objective_torch(xs, ys, ts, ps, params, warpfunc, t0=None, blur_sigma=2.0, timestamp_reverse=False,
                                     img_size=(180, 240), batch_end_indices=None, inv_depth=None):
    """
    Average-timestamp loss f_b of every sample b of a batch of event windows, each warped by its own motion params[b].
    Sample b holds the events [start_b, end_b) of the concatenated stream, end_b = batch_end_indices[b] and start_b the
    previous end (0 for the first sample):
      1. d = t - t0_b formed in ts' dtype, then f32, and warpfunc's model in f32, in the order written, exactly as
         motion_contrast_objective_torch warps:
             linvel_warp         (vx, vy)              x' = x - d vx,  y' = y - d vy               (warps.py:51-61)
             pure_rotation_warp  (cx, cy, omega)       rotation about (cx, cy) by omega d
             xyztheta_warp       (hx, hy, hz, theta)   about warpfunc.center
             affine_warp, homography_warp           about warpfunc.center (warps.py; past the horizon: not kept)
             camera_rotation_warp (wx, wy, wz)      exact camera rotation (warps.py; behind the camera: not kept)
             camera_motion_warp (wx, wy, wz, vx, vy, vz)  exact camera rotation and translation with the events'
                                                  inverse depth inv_depth (warps.py; behind the camera or without a
                                                  finite, non-negative inverse depth: not kept)
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
    @param warpfunc an instance of linvel_warp, pure_rotation_warp, xyztheta_warp, affine_warp, homography_warp,
           camera_rotation_warp or camera_motion_warp
    @param t0 None (each sample's last timestamp, zhu_timestamp_objective's ts[-1]), a number, or B values
    @param img_size (H, W): the bounds of step 3 and the canvas (H+1, W+1)
    @param batch_end_indices the cumulative end indices of BaseVoxelDataset.collate_fn
           (lib/data_loaders/base_dataset.py:513-539), a list or an int64 tensor; None means one sample of all events
    @param inv_depth camera_motion_warp only (required there, rejected with any other model): the (N,) inverse depth of
           every event, as in motion_contrast_objective_torch
    @returns (B,) tensor of f in params' dtype, on params' device, 0 <= B <= 32767.  The backward is the exact derivative
           of f with respect to params, with the floor and keep decisions held.  It rounds the incoming gradient g_b to
           f32 and stores the images in f32, so the gradient is accurate to f32 rounding whatever params' dtype.  With
           every input already on the GPU neither the forward nor the backward synchronises with the host.
    """
    warp = _warp_code(warpfunc, "motion_timestamp_objective_torch")
    xs, ys, ts, ps = _event_tensors(xs, ys, ts, ps, t0, "motion_timestamp_objective_torch", "params")
    rho = _depth_tensor(inv_depth, warp, xs.shape[0], "motion_timestamp_objective_torch")
    params = _params_tensor(params, warpfunc)
    B = params.shape[0]
    _check_window_count(batch_end_indices, B, "parameter vectors")
    H, W = int(img_size[0]), int(img_size[1])
    _lib.lib()
    dev = E.compute_device(params, xs, ys, ts, ps)
    x, y, t_rel, tau, p, offsets = _timestamp_events(xs, ys, ts, ps, t0, batch_end_indices, B, dev, "parameter vectors",
                                                     timestamp_reverse)
    from ..autograd import MotionTimestampObjective
    opts = _ts_model(warp, warpfunc, blur_sigma, H, W)
    f = MotionTimestampObjective.apply(_rows(params, opts[1]), x, y, t_rel, tau, p, offsets, opts, _depth_events(rho, dev))
    return f.to(device=params.device, dtype=params.dtype)


# The workspace of one evk_motion_timestamp_candidates_f32 call stays below this many bytes: larger batches of windows
# run in chunks (96 bytes per canvas pixel and candidate: 16 GiB hold 119 windows x 32 candidates at 180x240, about as
# many windows per chunk as the contrast loss's candidates pass takes).
TIMESTAMP_CANDIDATES_WORKSPACE_BYTES = 16 << 30


def motion_timestamp_candidates_torch(xs, ys, ts, ps, candidates, warpfunc, t0=None, blur_sigma=2.0, timestamp_reverse=False,
                                      img_size=(180, 240), batch_end_indices=None, inv_depth=None):
    """
    The average-timestamp loss of every window b under each of its J candidate parameter vectors candidates[b, j]:
    f[b, j] is the f_b that motion_timestamp_objective_torch returns with params[b] = candidates[b, j] (same windows, t0,
    stamps, keep rule, blur and canvas).  Each pass over the events scores up to 32 candidates of every window
    (evk_motion_timestamp_candidates_f32): the grid search and the line search of motion_timestamp_fit_torch.  J is split
    into passes of at most 32 candidates, and the windows into chunks whose workspace stays under
    TIMESTAMP_CANDIDATES_WORKSPACE_BYTES; neither split changes a value's arithmetic.
    @param candidates (B,J,K) parameter vectors, any float dtype, K = warpfunc.dims, any J >= 1
    @param inv_depth camera_motion_warp's inverse depth of every event, as in motion_timestamp_objective_torch
    @returns (B,J) f64 tensor of values (no autograd graph) on candidates' device
    """
    warp = _warp_code(warpfunc, "motion_timestamp_candidates_torch")
    xs, ys, ts, ps = _event_tensors(xs, ys, ts, ps, t0, "motion_timestamp_candidates_torch", "nothing")
    rho = _depth_tensor(inv_depth, warp, xs.shape[0], "motion_timestamp_candidates_torch")
    cand = _candidates_tensor(candidates, warpfunc)
    B = cand.shape[0]
    H, W = int(img_size[0]), int(img_size[1])
    _lib.lib()
    dev = E.compute_device(cand, xs, ys, ts, ps)
    x, y, t_rel, tau, p, offsets = _timestamp_events(xs, ys, ts, ps, t0, batch_end_indices, B, dev, "candidate sets",
                                                     timestamp_reverse)
    with torch.cuda.device(dev):
        c64 = cand.detach().to(device=dev, dtype=torch.float64)
        f = _ts_candidates(x, y, t_rel, tau, p, offsets, c64, _ts_model(warp, warpfunc, blur_sigma, H, W),
                           _depth_events(rho, dev))
    return f.to(cand.device)


def _ts_candidates(x, y, t_rel, tau, p, offsets, c64, opts, rho=None):
    """f (B,J) f64 of the prepared device events under the device candidates c64 (B,J,K) f64, in passes of at most
    MAX_CANDIDATES candidates over chunks of windows whose workspace fits TIMESTAMP_CANDIDATES_WORKSPACE_BYTES; rho: the
    device inverse depth of camera_motion_warp, or None"""
    warp, centre, H, W, sigma = opts
    stem, events = _depth_entry("evk_motion_timestamp_candidates", (x, y, t_rel, tau, p), rho)
    return _chunked_candidates(stem, "motion_timestamp_candidates", events, offsets, c64, (warp, centre, H, W), (sigma,),
                               TIMESTAMP_CANDIDATES_WORKSPACE_BYTES, 32767)
