"""Motion segmentation by motion compensation (Stoffregen, Gallego, Drummond, Kleeman, Scaramuzza, ICCV 2019) on the GPU.

A window rarely holds one motion: a car in front of a panning camera, two people crossing.  The method keeps M motion
models per window and a soft membership w[e, m] of every event in every model, and alternates two steps:
    M-step  with the memberships fixed, maximise each model's contrast of its WEIGHTED image of warped events
    E-step  with the models fixed, reassign each event in proportion to how sharp each model's image is where that
            model sends it
The reference keeps only remnants of this work (segmentation_mask_from_d_iwe and get_hsv_shifted,
lib/contrast_max/events_cmax.py:14-101), which stay out of this library.  Here the weighted images of all M models of a
window come from ONE pass over the events (evk_cmax_motion_segment_f32), as do their gradients with respect to the
parameters and the memberships (evk_cmax_motion_segment_grad_f32), a line search of every model
(evk_cmax_motion_segment_candidates_f32) and the E-step (evk_cmax_motion_segment_assign_f32).
"""
import collections

import torch

from .. import _lib
from ..representations import _events as E
from ._batched import (_batch_events, _check_objective, _chunked_candidates, _chunked_objective, _event_tensors,
                       _float_tensor, _model, _rows, _warp_code, _window_count, fit_window_chunk)
from .motion_fit import FIT_WORKSPACE_BYTES, _batched_bfgs, _check_line_search_steps, _per_window

MAX_MODELS = 8            # motion models per window
MAX_CANVASES = 65535      # images per call of an entry (the image tail's grid limit)
# The workspace of one evk_cmax_motion_segment_candidates_f32 call stays below this many bytes: larger batches of
# windows run in chunks
SEGMENT_CANDIDATES_WORKSPACE_BYTES = 4 << 30

MotionSegmentation = collections.namedtuple("MotionSegmentation", "params weights f status iterations")
MotionSegmentation.__doc__ = """motion_segmentation_fit_torch's result: params (B,M,K) f64, weights (N,M) f32, f (B,M) f64,
status (B,M) int8, iterations (B,M) int32"""


def _segment_warp_code(warpfunc, who):
    """_warp_code of the models segmentation takes: camera_motion_warp needs the inverse depth of every event, which the
    segmentation entries do not take"""
    warp = _warp_code(warpfunc, who)
    if warp == _lib.WARP_CAMERA_MOTION:
        raise ValueError("%s does not take camera_motion_warp: motion segmentation has no inverse-depth input; segment with "
                         "camera_rotation_warp or a planar model" % who)
    return warp


def motion_segmentation_objective_torch(xs, ys, ts, ps, weights, params, warpfunc, t0=None, objective="variance",
                                        blur_sigma=1.0, obj_param=None, img_size=(180, 240), batch_end_indices=None):
    """
    The contrast f[b, m] of every model m of every window b, each image made of the window's events weighted by their
    membership in that model.  Windows, t0, warp models, keep rule, canvas, blur and objectives ('moa' and 'isoa'
    rejected) are exactly those of motion_contrast_objective_torch.  Image (b, m) is the IWE of window b's events warped
    by params[b, m], each event splatted with the weight p_e * weights[e, m] formed in f32: it has exactly the taps of
    motion_contrast_objective_torch(xs, ys, ts, ps * weights[:, m], params[:, m]), and f[b, m] is that image's
    objective.  At M = 1 with weights = 1 this is motion_contrast_objective_torch.  ps is used as given.
    Differentiable in params and weights (the events are data): the backward is the exact derivative with the floor
    and keep decisions held, one pass over the events (evk_cmax_motion_segment_grad_f32).  The weight gradient is only
    computed when weights requires grad; an event of weight 0 (or p = 0) still gets one.
    @param weights (N,M) memberships over the concatenated stream, 1 <= M <= 8 (any float dtype; the kernels take f32)
    @param params (B,M,K), or (M,K) for every window, K = warpfunc.dims
    @returns (B,M) tensor in params' dtype on params' device.  B * M <= 65535.  With every input on the GPU neither the
           forward nor the backward synchronises with the host.
    """
    warp = _segment_warp_code(warpfunc, "motion_segmentation_objective_torch")
    _check_objective(objective, "parameters and weights")
    xs, ys, ts, ps = _event_tensors(xs, ys, ts, ps, t0, "motion_segmentation_objective_torch", "params and weights")
    weights = _weights_tensor(weights, xs.shape[0])
    M = weights.shape[1]
    params = _models_tensor(params, "params", M, warpfunc, batch_end_indices)
    B = params.shape[0]
    H, W = int(img_size[0]), int(img_size[1])
    _lib.lib()
    dev = E.compute_device(params, weights, xs, ys, ts, ps)
    x, y, t_rel, p, offsets = _batch_events(xs, ys, ts, ps, t0, batch_end_indices, B, dev, "parameter sets")
    from ..autograd import MotionSegmentationObjective
    opts = _model(warp, warpfunc, objective, blur_sigma, obj_param, H, W)
    f = MotionSegmentationObjective.apply(_rows(params, opts[1]), weights, x, y, t_rel, p, offsets, opts)
    return f.to(device=params.device, dtype=params.dtype)


def motion_segmentation_candidates_torch(xs, ys, ts, ps, candidates, weights, warpfunc, t0=None, objective="variance",
                                         blur_sigma=1.0, obj_param=None, img_size=(180, 240), batch_end_indices=None):
    """
    f[b, m, j]: the f[b, m] of motion_segmentation_objective_torch with params[b, m] = candidates[b, m, j] (same weights,
    windows, t0, objective, blur and canvas conventions).  Each pass over the events scores up to 32 // M candidates of
    every model of every window (evk_cmax_motion_segment_candidates_f32); J is split into such passes, and the windows
    into chunks whose workspace stays under SEGMENT_CANDIDATES_WORKSPACE_BYTES and whose images number at most 65535.
    Neither split changes a value's arithmetic.
    @param candidates (B,M,J,K) parameter vectors, any float dtype, any J >= 1
    @returns (B,M,J) f64 tensor of values (no autograd graph) on candidates' device
    """
    warp = _segment_warp_code(warpfunc, "motion_segmentation_candidates_torch")
    _check_objective(objective, "parameters")
    xs, ys, ts, ps = _event_tensors(xs, ys, ts, ps, t0, "motion_segmentation_candidates_torch", "nothing")
    weights = _weights_tensor(weights, xs.shape[0])
    M = weights.shape[1]
    cand = _float_tensor(candidates, "candidates")
    if cand.dim() != 4 or cand.shape[1] != M or cand.shape[2] < 1 or cand.shape[3] != warpfunc.dims:
        raise ValueError("candidates must have shape (B,%d,J,%d) with J >= 1 for %d models of %s, got %s"
                         % (M, warpfunc.dims, M, type(warpfunc).__name__, tuple(cand.shape)))
    B = cand.shape[0]
    H, W = int(img_size[0]), int(img_size[1])
    _lib.lib()
    dev = E.compute_device(cand, weights, xs, ys, ts, ps)
    x, y, t_rel, p, offsets = _batch_events(xs, ys, ts, ps, t0, batch_end_indices, B, dev, "candidate sets")
    with torch.cuda.device(dev):
        w = _device_weights(weights, dev)
        c64 = cand.detach().to(device=dev, dtype=torch.float64)
        f = _segment_candidates(x, y, t_rel, p, w, offsets, c64, _model(warp, warpfunc, objective, blur_sigma, obj_param, H, W))
    return f.to(cand.device)


def motion_segmentation_assign_torch(xs, ys, ts, ps, params, warpfunc, weights, t0=None, blur_sigma=1.0,
                                     img_size=(180, 240), batch_end_indices=None, eps=1e-6):
    """
    The E-step: new memberships (N,M) f32 from the models params and the current memberships weights.  The images of
    motion_segmentation_objective_torch are built with `weights`, blurred (blur_sigma), and then for every event e and
    model m, with k the event's polarity- and weight-free bilinear fractions under params[b, m] and G_bm the blurred
    image (b, m):
        c[e, m] = max(0, sum_taps k G_bm(tap))     (0 when the event is not kept under model m)
        w'[e, m] = (c[e, m] + eps) / (sum_i c[e, i] + M eps)
    A row whose c are all 0 with eps = 0, and a row of an event outside every window, is 1/M; a non-finite c (a
    non-finite image) makes only its own row non-finite.  For users who drive the M-step themselves, e.g. with Adam on
    motion_segmentation_objective_torch.  No autograd graph; the windows run in chunks as in the fit.
    @returns (N,M) f32 tensor on weights' device
    """
    warp = _segment_warp_code(warpfunc, "motion_segmentation_assign_torch")
    xs, ys, ts, ps = _event_tensors(xs, ys, ts, ps, t0, "motion_segmentation_assign_torch", "nothing")
    weights = _weights_tensor(weights, xs.shape[0])
    M = weights.shape[1]
    params = _models_tensor(params, "params", M, warpfunc, batch_end_indices)
    eps = _check_eps(eps)
    B = params.shape[0]
    H, W = int(img_size[0]), int(img_size[1])
    _lib.lib()
    dev = E.compute_device(params, weights, xs, ys, ts, ps)
    x, y, t_rel, p, offsets = _batch_events(xs, ys, ts, ps, t0, batch_end_indices, B, dev, "parameter sets")
    with torch.cuda.device(dev):
        w = _device_weights(weights, dev)
        p64 = params.detach().to(device=dev, dtype=torch.float64).contiguous()
        out = _assign(x, y, t_rel, p, w, offsets, p64, _model(warp, warpfunc, "variance", blur_sigma, None, H, W), eps)
    return out.to(weights.device)


def motion_segmentation_fit_torch(xs, ys, ts, ps, warpfunc, x0, batch_end_indices=None, t0=None, weights0=None,
                                  objective="variance", blur_sigma=1.0, obj_param=None, img_size=(180, 240), em_iters=10,
                                  max_iter=20, line_search_steps=8, eps=1e-6, param_scale=None, ftol=1e-9, gtol=1e-9):
    """
    Segment every window into M independently moving parts: EM on the weighted contrast of
    motion_segmentation_objective_torch, all windows and models at once.
    Start: the models x0 ((B,M,K), or (M,K) for every window) and the memberships weights0 ((N,M)), or uniform 1/M when
    weights0 is None -- the models in x0 must then differ, since the first assignment is all that tells them apart.
    Each of the em_iters rounds is an assignment (motion_segmentation_assign_torch with eps; skipped in round 0 when
    weights0 is given) followed by max_iter iterations of the batched BFGS of motion_contrast_fit_torch over the B*M
    (window, model) rows, the memberships held: f and g from the forward and gradient entries, every line search one
    candidates pass over the events for all models.  The line search, the BFGS update, param_scale (default ones),
    ftol and gtol are motion_contrast_fit_torch's; each round starts the BFGS afresh from diag(param_scale^2).  A final
    assignment follows, and f is each model's objective at the returned params and weights.
    ps is used as given; pass ones or |ps|, as the images of the paper count events.
    The number of iterations is fixed and nothing is read back, so with the events, the window ends and x0 on the GPU
    the fit never synchronises with the host.  Any number of windows: every call of an entry takes a chunk of them
    (fit_window_chunk, at most 65535 // M windows, and 65535 // (M J) for a candidates pass), so the launch sequence
    depends on B only through those numbers of chunks.
    @returns MotionSegmentation(params (B,M,K) f64, weights (N,M) f32, f (B,M) f64, status (B,M) int8 of the last
             round (motion_fit's codes), iterations (B,M) int32 accepted steps summed over the rounds) on the events'
             device
    """
    warp = _segment_warp_code(warpfunc, "motion_segmentation_fit_torch")
    _check_objective(objective, "parameters")
    xs, ys, ts, ps = _event_tensors(xs, ys, ts, ps, t0, "motion_segmentation_fit_torch", "nothing")
    _check_line_search_steps(line_search_steps)
    eps = _check_eps(eps)
    K = warpfunc.dims
    B = _window_count(batch_end_indices)
    x0 = E.as_tensor(x0)
    if x0.dim() not in (2, 3) or tuple(x0.shape[-1:]) != (K,) or not 1 <= x0.shape[-2] <= MAX_MODELS or \
            (x0.dim() == 3 and x0.shape[0] != B):
        raise ValueError("x0 must have shape (B,M,%d) or (M,%d) with 1 <= M <= %d (B = %d windows), got %s"
                         % (K, K, MAX_MODELS, B, tuple(x0.shape)))
    M = x0.shape[-2]
    if weights0 is not None:
        weights0 = _weights_tensor(weights0, xs.shape[0])
        if weights0.shape[1] != M:
            raise ValueError("weights0 has %d models, x0 has %d" % (weights0.shape[1], M))
    H, W = int(img_size[0]), int(img_size[1])
    _lib.lib()
    dev = E.compute_device(*(a for a in (x0, weights0, xs, ys, ts, ps) if isinstance(a, torch.Tensor)))
    x, y, t_rel, p, offsets = _batch_events(xs, ys, ts, ps, t0, batch_end_indices, B, dev, "windows")
    opts = _model(warp, warpfunc, objective, blur_sigma, obj_param, H, W)
    with torch.cuda.device(dev):
        xk = _per_window(x0, B, (M, K), "x0", dev).reshape(B * M, K)
        scale = torch.ones((B * M, K), dtype=torch.float64, device=dev) if param_scale is None else \
            _per_window(param_scale, B * M, (K,), "param_scale", dev)
        w = _device_weights(weights0, dev) if weights0 is not None else \
            torch.full((x.shape[0], M), 1.0 / M, dtype=torch.float32, device=dev)
        iters = torch.zeros(B * M, dtype=torch.int32, device=dev)
        status = torch.zeros(B * M, dtype=torch.int8, device=dev)
        for r in range(int(em_iters)):
            if r or weights0 is None:
                w = _assign(x, y, t_rel, p, w, offsets, xk.reshape(B, M, K), opts, eps)
            fg = _segment_objective_and_gradient(x, y, t_rel, p, w, offsets, M, opts)
            cand = lambda c: _segment_candidates(x, y, t_rel, p, w, offsets, c.reshape(B, M, c.shape[1], K),
                                                 opts).reshape(B * M, c.shape[1])
            xk, _, status, it = _batched_bfgs(fg, cand, xk, scale, max_iter, line_search_steps, ftol, gtol)
            iters += it
        w = _assign(x, y, t_rel, p, w, offsets, xk.reshape(B, M, K), opts, eps)
        f, _ = _segment_objective_and_gradient(x, y, t_rel, p, w, offsets, M, opts, gradient=False)(xk)
    return MotionSegmentation(xk.reshape(B, M, K), w, f.reshape(B, M), status.reshape(B, M), iters.reshape(B, M))


def _check_eps(eps):
    eps = float(eps)
    if not eps >= 0.0 or eps == float("inf"):
        raise ValueError("eps must be finite and >= 0, got %r" % (eps,))
    return eps


def _weights_tensor(weights, n):
    weights = _float_tensor(weights, "weights")
    if weights.dim() != 2 or weights.shape[0] != n or not 1 <= weights.shape[1] <= MAX_MODELS:
        raise ValueError("weights must have shape (N,M) with N = %d events and 1 <= M <= %d, got %s"
                         % (n, MAX_MODELS, tuple(weights.shape)))
    return weights


def _models_tensor(params, name, M, warpfunc, batch_end_indices):
    """params as a (B,M,K) tensor ((M,K) is every window's)"""
    params = _float_tensor(params, name)
    K = warpfunc.dims
    if params.dim() == 2 and tuple(params.shape) == (M, K):
        params = params.unsqueeze(0).expand(_window_count(batch_end_indices), M, K)
    if params.dim() != 3 or tuple(params.shape[1:]) != (M, K):
        raise ValueError("%s must have shape (B,%d,%d) or (%d,%d) for %d models of %s, got %s"
                         % (name, M, K, M, K, M, type(warpfunc).__name__, tuple(params.shape)))
    return params


def _device_weights(weights, dev):
    return weights.detach().to(device=dev, dtype=torch.float32).contiguous()


def _segment_candidates(x, y, t_rel, p, w, offsets, c64, opts):
    """f (B,M,J) f64 of the prepared device events and memberships under the device candidates c64 (B,M,J,K) f64, in
    passes of at most 32 // M candidates over chunks of windows"""
    warp, centre, H, W, objective, sigma, param = opts
    return _chunked_candidates("evk_cmax_motion_segment_candidates", "motion_segment_candidates", (x, y, t_rel, p, w), offsets,
                               c64, (warp, centre, H, W), (sigma, objective, param), SEGMENT_CANDIDATES_WORKSPACE_BYTES,
                               MAX_CANVASES, M=c64.shape[1])


def _segment_chunk(B, M, H, W):
    """windows per call of the forward / gradient / assignment entries"""
    L = _lib.lib()
    per_window = L.evk_cmax_motion_segment_workspace_bytes(1, M, H, W) + 4 * M * (H + 1) * (W + 1)
    return fit_window_chunk(B, per_window, FIT_WORKSPACE_BYTES, MAX_CANVASES // M)


def _segment_objective_and_gradient(x, y, t_rel, p, w, offsets, M, opts, gradient=True):
    """(B*M,K) f64 params -> (f (B*M,) f64, g (B*M,K) f64) at the held memberships w, through
    evk_cmax_motion_segment_f32 / _grad_f32 (grad_f = 1) in chunks of windows (no weight gradient)"""
    warp, centre, H, W, objective, sigma, param = opts
    return _chunked_objective("evk_cmax_motion_segment", "motion_segment", (x, y, t_rel, p, w), offsets, (warp, centre, H, W),
                              (sigma, objective, param), (M,), FIT_WORKSPACE_BYTES, MAX_CANVASES // M, M=M, gradient=gradient)


def _assign(x, y, t_rel, p, w, offsets, p64, opts, eps):
    """the E-step on prepared device inputs: images of the memberships w under the models p64 (B,M,K) f64, then
    evk_cmax_motion_segment_assign_f32, in chunks of windows; rows outside every window are 1/M"""
    warp, centre, H, W, _, sigma, _ = opts
    cx, cy = centre[:2]
    B, M, _ = p64.shape
    L = _lib.lib()
    dev = x.device
    out = torch.full((x.shape[0], M), 1.0 / M, dtype=torch.float32, device=dev)
    if B == 0:
        return out
    prm = _rows(p64, centre).contiguous()
    K = prm.shape[-1]
    wb = _segment_chunk(B, M, H, W)
    iwe = torch.empty((wb * M, H + 1, W + 1), dtype=torch.float32, device=dev)
    f = torch.empty(wb * M, dtype=torch.float64, device=dev)
    ws = _lib.scratch("motion_segment", L.evk_cmax_motion_segment_workspace_bytes(wb, M, H, W), dev)
    for b0 in range(0, B, wb):
        b1 = min(B, b0 + wb)
        pb = _lib.ptr(prm[b0:b1])
        _lib.check(L.evk_cmax_motion_segment_f32(
            _lib.ptr(x), _lib.ptr(y), _lib.ptr(t_rel), _lib.ptr(p), _lib.ptr(w), M, _lib.ptr(offsets[b0:]), b1 - b0, x.shape[0],
            warp, pb, K, cx, cy, H, W, sigma, _lib.OBJ_VARIANCE, 0.0, _lib.ptr(f), _lib.ptr(iwe), _lib.ptr(ws), ws.numel(),
            _lib.stream()))
        _lib.check(L.evk_cmax_motion_segment_assign_f32(
            _lib.ptr(x), _lib.ptr(y), _lib.ptr(t_rel), M, _lib.ptr(offsets[b0:]), b1 - b0, x.shape[0], warp, pb, K, cx, cy,
            H, W, _lib.ptr(iwe), sigma, eps, _lib.ptr(out), _lib.ptr(ws), ws.numel(), _lib.stream()))
    return out
