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
from .motion_objective import _WARPS, MAX_CANDIDATES, _warp_code


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


# The workspace of one evk_motion_timestamp_candidates_f32 call stays below this many bytes: larger batches of windows
# run in chunks (96 bytes per canvas pixel and candidate: 16 GiB hold 119 windows x 32 candidates at 180x240, about as
# many windows per chunk as the contrast loss's candidates pass takes).
TIMESTAMP_CANDIDATES_WORKSPACE_BYTES = 16 << 30


def motion_timestamp_candidates_torch(xs, ys, ts, ps, candidates, warpfunc, t0=None, blur_sigma=2.0, timestamp_reverse=False,
                                      img_size=(180, 240), batch_end_indices=None):
    """
    The average-timestamp loss of every window b under each of its J candidate parameter vectors candidates[b, j]:
    f[b, j] is the f_b that motion_timestamp_objective_torch returns with params[b] = candidates[b, j] (same windows, t0,
    stamps, keep rule, blur and canvas).  Each pass over the events scores up to 32 candidates of every window
    (evk_motion_timestamp_candidates_f32): the grid search and the line search of motion_timestamp_fit_torch.  J is split
    into passes of at most 32 candidates, and the windows into chunks whose workspace stays under
    TIMESTAMP_CANDIDATES_WORKSPACE_BYTES; neither split changes a value's arithmetic.
    @param candidates (B,J,K) parameter vectors, any float dtype, K = warpfunc.dims, any J >= 1
    @returns (B,J) f64 tensor of values (no autograd graph) on candidates' device
    """
    warp = _warp_code(warpfunc, "motion_timestamp_candidates_torch")
    xs, ys, ts, ps = _event_tensors(xs, ys, ts, ps, t0, "motion_timestamp_candidates_torch", "nothing")
    cand = E.as_tensor(candidates)
    if not cand.is_floating_point():
        raise ValueError("candidates must be a floating-point tensor, got %s" % cand.dtype)
    if cand.dim() != 3 or cand.shape[2] != warpfunc.dims or cand.shape[1] < 1:
        raise ValueError("candidates must have shape (B,J,%d) with J >= 1 for %s, got %s"
                         % (warpfunc.dims, type(warpfunc).__name__, tuple(cand.shape)))
    B = cand.shape[0]
    H, W = int(img_size[0]), int(img_size[1])
    _lib.lib()
    dev = E.compute_device(cand, xs, ys, ts, ps)
    x, y, t_rel, p, offsets, t, sample = _batch_events(xs, ys, ts, ps, t0, batch_end_indices, B, dev, "candidate sets",
                                                       stamps=True)
    with torch.cuda.device(dev):
        tau = _normalised_stamps(t, sample, offsets, timestamp_reverse)
        c64 = cand.detach().to(device=dev, dtype=torch.float64)
        f = _ts_candidates(x, y, t_rel, tau, p, offsets, c64, _ts_model(warp, warpfunc, blur_sigma, H, W))
    return f.to(cand.device)


def _ts_model(warp, warpfunc, blur_sigma, H, W):
    """the scalar arguments the motion timestamp entries share: (warp code, (cx, cy), H, W, sigma)"""
    centre = tuple(float(c) for c in warpfunc.center) if warp == _lib.WARP_XYZTHETA else (0.0, 0.0)
    return warp, centre, H, W, float(blur_sigma)


def _ts_candidates(x, y, t_rel, tau, p, offsets, c64, opts):
    """f (B,J) f64 of the prepared device events under the device candidates c64 (B,J,K) f64, in passes of at most
    MAX_CANDIDATES candidates over chunks of windows whose workspace fits TIMESTAMP_CANDIDATES_WORKSPACE_BYTES"""
    warp, (cx, cy), H, W, sigma = opts
    B, J, K = c64.shape
    L = _lib.lib()
    dev = x.device
    f = torch.empty((B, J), dtype=torch.float64, device=dev)
    if B == 0:
        return f
    jc = min(J, MAX_CANDIDATES)
    per_window = L.evk_motion_timestamp_candidates_workspace_bytes(1, jc, H, W)
    wb = max(1, min(B, TIMESTAMP_CANDIDATES_WORKSPACE_BYTES // per_window, 32767 // jc))
    ws = _lib.scratch("motion_timestamp_candidates", L.evk_motion_timestamp_candidates_workspace_bytes(wb, jc, H, W), dev)
    for b0 in range(0, B, wb):
        b1 = min(B, b0 + wb)
        for j0 in range(0, J, MAX_CANDIDATES):
            j1 = min(J, j0 + MAX_CANDIDATES)
            c = c64[b0:b1, j0:j1].contiguous()
            out = torch.empty((b1 - b0, j1 - j0), dtype=torch.float64, device=dev)
            _lib.check(L.evk_motion_timestamp_candidates_f32(
                _lib.ptr(x), _lib.ptr(y), _lib.ptr(t_rel), _lib.ptr(tau), _lib.ptr(p), _lib.ptr(offsets[b0:]), b1 - b0,
                x.shape[0], warp, _lib.ptr(c), j1 - j0, K, cx, cy, H, W, sigma, _lib.ptr(out), _lib.ptr(ws), ws.numel(),
                _lib.stream()))
            f[b0:b1, j0:j1] = out
    return f
