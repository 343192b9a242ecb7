"""Fit one motion per event window on the GPU: a grid search per window, then batched BFGS on the parametric contrast loss.

The reference fits one window at a time: grid_search_initial / grid_search_optimisation (events_cmax.py:184-311) for a
start, then scipy's BFGS (optimize_contrast, events_cmax.py:313-346), with one full evaluation and one host round trip
per f / f' call.  motion_contrast_fit_torch fits B windows at once: every grid level and every line search is ONE
candidates pass over the events (motion_contrast_candidates_torch), f and its gradient are one call each of the
batched loss's C entries, and the BFGS state is a set of (B,K) / (B,K,K) tensors updated under per-window masks.  The
number of iterations is fixed, so with every input on the GPU the fit never synchronises with the host.  Every call of
an entry takes a chunk of the windows, at most as many as the entry's batch limit and its workspace budget allow.
"""
import collections

import numpy as np
import torch

from .. import _lib
from ..representations import _events as E
from ._batched import fit_window_chunk  # noqa: F401  (a public name of this module)
from ._batched import (_batch_events, _check_objective, _chunked_objective, _depth_entry, _depth_events, _depth_tensor,
                       _event_tensors, _model, _warp_code, _window_count)
from .motion_objective import _candidates

MotionFit = collections.namedtuple("MotionFit", "params f status iterations")
MotionFit.__doc__ = """motion_contrast_fit_torch's result: params (B,K) f64, f (B,) f64, status (B,) int8, iterations (B,) int32"""

# status codes of motion_contrast_fit_torch
CONVERGED, ITERATION_LIMIT, NO_DESCENT, NONFINITE_START = 0, 1, 2, 3
ARMIJO_C1 = 1e-4


def motion_contrast_fit_torch(xs, ys, ts, ps, warpfunc, batch_end_indices=None, t0=None, objective="variance",
                              blur_sigma=1.0, obj_param=None, img_size=(180, 240), x0=None, param_ranges=None,
                              num_samples_per_param=5, grid_levels=1, log_scale=False, param_scale=None, max_iter=50,
                              line_search_steps=8, ftol=1e-9, gtol=1e-9, inv_depth=None):
    """
    Minimise the f_b of motion_contrast_objective_torch over the parameters of every window b on its own, all windows at
    once.  The windows, t0, objective, obj_param and img_size are those of motion_contrast_objective_torch, so any result
    can be checked with it.
    Start point: x0 ((B,K) or (K,)) if given.  Otherwise a grid search per window: level 0 samples the axes that
    grid_search_initial builds from param_ranges ((K,2), or (B,K,2) per window; num_samples_per_param odd, log_scale),
    in the order of its meshgrid, and takes the lowest f (the first of equal ones); each further level (grid_levels in
    all) re-centres every window's axes around its best point with find_new_range's rule (events_cmax.py:160-182,
    including the outermost-spacing quirks).  Each level is one motion_contrast_candidates_torch call.
    Refinement: BFGS per window.  The inverse Hessian starts as diag(param_scale^2) (param_scale defaults to the grid's
    level-0 spacing (hi - lo) / (num_samples_per_param - 1), or ones with x0) and is rescaled by s'y / y'y in the
    coordinates x / param_scale after the first accepted step.  Each iteration scores the step lengths 2^-j,
    j < line_search_steps (<= 32), along d = -H g in ONE candidates pass and takes the largest that meets Armijo
    (c1 = 1e-4), else the best one if it lowers f.  f and g at that point come from the loss's forward and gradient
    entries, and a point whose f is above the current one is not taken (the candidates pass and the forward sum f32
    images in different orders).  When no step is taken, H is reset once, to diag(param_scale^2) times the latest
    s'y / y'Dy (D = diag(param_scale^2); 1 before any update); a second failure without an accepted step between stops
    the window (NO_DESCENT).  The BFGS update is applied when s'y > 1e-10 |s| |y|.  A
    window converges when a full step (alpha = 1) lowers f by less than ftol relative, or when
    max |g * param_scale| <= gtol |f|.  An objective computed from f32 images is known to about 1e-7 relative, and its
    splat makes it only piecewise smooth, so a small gradient or a small decrease can show up well before the
    minimum: the defaults (1e-9) lie below that noise, and a window usually ends where no step lowers f any more
    (NO_DESCENT) rather than CONVERGED -- both are a local minimum to the precision of f.  Stopped windows keep their
    values bit for bit while the others iterate.
    blur_sigma may be a sequence: stage i refines at blur_sigma[i] from stage i-1's result, and the grid search runs
    at blur_sigma[0] only (grid_cmax's grid at blur 2, then refinement at 1, events_cmax.py:28-76).
    camera_motion_warp takes inv_depth, the inverse depth of every event (motion_contrast_objective_torch).  A grid over
    its six parameters costs num_samples_per_param^6 candidates per window, so start it from x0: a camera_rotation_warp
    fit embedded as (w, 0, 0, 0), or an IMU's rates and velocity.
    Every stage runs exactly max_iter iterations on all windows (max_iter = 0 returns the start), so with the events,
    the window ends and x0 (or param_ranges) on the GPU the fit never synchronises with the host.
    Any number of windows B: each candidates call runs the windows in chunks of
    max(1, min(B, CANDIDATES_WORKSPACE_BYTES // its workspace per window, 65535 // min(J, 32))) windows (J the candidates
    of the call: num_samples_per_param^K for a grid level, line_search_steps for a line search), and each forward and
    gradient call in chunks of max(1, min(B, FIT_WORKSPACE_BYTES // (workspace + image per window), 65535)).  The launch
    sequence therefore depends on B only through those numbers of chunks.
    @returns MotionFit(params (B,K) f64, f (B,) f64 at params for the last stage's blur, status (B,) int8, iterations
             (B,) int32 summed over the stages) on the events' device.  status: 0 converged, 1 iteration limit,
             2 no descent, 3 non-finite start, f or g at a stage's start (the window keeps that start).  An empty window,
             or one with no kept event, has g = 0 and returns its start as converged.
    """
    warp = _warp_code(warpfunc, "motion_contrast_fit_torch")
    _check_objective(objective, "parameters")
    xs, ys, ts, ps = _event_tensors(xs, ys, ts, ps, t0, "motion_contrast_fit_torch", "nothing")
    rho = _depth_tensor(inv_depth, warp, xs.shape[0], "motion_contrast_fit_torch")
    sigmas = _fit_arguments("motion_contrast_fit_torch", blur_sigma, line_search_steps, x0, param_ranges)
    H, W = int(img_size[0]), int(img_size[1])
    _lib.lib()
    dev = E.compute_device(*(a for a in (x0, param_ranges, xs, ys, ts, ps) if isinstance(a, torch.Tensor)))
    B = _window_count(batch_end_indices)
    x, y, t_rel, p, offsets = _batch_events(xs, ys, ts, ps, t0, batch_end_indices, B, dev, "windows")
    rho = _depth_events(rho, dev)

    def stage(sigma):
        opts = _model(warp, warpfunc, objective, sigma, obj_param, H, W)
        return (_objective_and_gradient(x, y, t_rel, p, offsets, opts, rho),
                lambda c: _candidates(x, y, t_rel, p, offsets, c, opts, rho))
    with torch.cuda.device(dev):
        return _fit_stages(stage, sigmas, B, warpfunc.dims, dev, x0, param_ranges, num_samples_per_param, grid_levels,
                           log_scale, param_scale, max_iter, line_search_steps, ftol, gtol)


def _fit_arguments(who, blur_sigma, line_search_steps, x0, param_ranges):
    """the argument checks the fits share, before any CUDA call; returns the blur sigmas of the stages"""
    sigmas = [float(s) for s in (blur_sigma if isinstance(blur_sigma, (list, tuple)) else [blur_sigma])]
    if not sigmas:
        raise ValueError("blur_sigma must be a number or a non-empty sequence")
    _check_line_search_steps(line_search_steps)
    if x0 is None and param_ranges is None:
        raise ValueError("%s needs x0 or param_ranges" % who)
    return sigmas


def _check_line_search_steps(line_search_steps):
    if not 1 <= int(line_search_steps) <= 32:
        raise ValueError("line_search_steps must be in 1..32, got %r" % (line_search_steps,))


def _fit_stages(stage, sigmas, B, K, dev, x0, param_ranges, num_samples_per_param, grid_levels, log_scale, param_scale,
                max_iter, line_search_steps, ftol, gtol, bounds=None, bound_to_ranges=False, unit_first_step=False):
    """The start point and the BFGS stages the fits share.  stage(sigma) -> (fg, candidates) of the objective at that
    blur.  bounds ((K,2) or (B,K,2)) confines the line searches; without it, bound_to_ranges confines a grid-started fit
    to param_ranges widened by one level-0 grid step on each side, and further to take in the grid's best point (a
    later grid level may lie beyond the ranges).
    unit_first_step is _batched_bfgs'."""
    if bounds is not None:
        bounds = _per_window(bounds, B, (K, 2), "bounds", dev)
    if x0 is None:
        ranges = _per_window(param_ranges, B, (K, 2), "param_ranges", dev)
        start = _grid_search(stage(sigmas[0])[1], ranges, num_samples_per_param, grid_levels, log_scale)
        scale = (ranges[..., 1] - ranges[..., 0]) / (num_samples_per_param - 1)
        if bounds is None and bound_to_ranges:
            # one grid step beyond the ranges: a start on the ranges' edge must be free to step outwards
            bounds = torch.stack((torch.minimum(ranges[..., 0] - scale, start), torch.maximum(ranges[..., 1] + scale, start)),
                                 dim=-1)
    else:
        start = _per_window(x0, B, (K,), "x0", dev)
        scale = torch.ones((B, K), dtype=torch.float64, device=dev)
    if param_scale is not None:
        scale = _per_window(param_scale, B, (K,), "param_scale", dev)
    xk = start
    iters = torch.zeros(B, dtype=torch.int32, device=dev)
    status = f = None
    for sigma in sigmas:
        fg, candidates = stage(sigma)
        xk, f, status, it = _batched_bfgs(fg, candidates, xk, scale, max_iter, line_search_steps, ftol, gtol, bounds,
                                          unit_first_step)
        iters += it
    return MotionFit(xk, f, status, iters)


def _per_window(v, B, shape, name, dev):
    """v of `shape` or (B,)+shape as a (B,)+shape f64 tensor on dev (a host value is copied without a host wait)"""
    t = v if isinstance(v, torch.Tensor) else torch.from_numpy(np.array(v, dtype=np.float64))
    _check_per_window(t, B, shape, name)
    if tuple(t.shape) == tuple(shape):
        t = t.unsqueeze(0).expand((B,) + tuple(shape))
    return _to_device(t.to(torch.float64), dev).contiguous()


def _check_per_window(v, B, shape, name):
    got = tuple(v.shape) if isinstance(v, torch.Tensor) else np.shape(v)
    if got != tuple(shape) and got != (B,) + tuple(shape):
        raise ValueError("%s must have shape %s or %s, got %s" % (name, tuple(shape), (B,) + tuple(shape), got))


def _to_device(t, dev):
    """a copy of t on dev; a host tensor goes through pinned memory, so the copy does not wait for the host"""
    if t.device == dev:
        return t.clone()
    if t.device.type == "cpu" and dev.type == "cuda":
        return t.contiguous().pin_memory().to(dev, non_blocking=True)
    return t.to(dev)


# One forward + gradient call of motion_contrast_fit_torch takes at most this many windows (the entries' batch limit)
# and at most as many as fit FIT_WORKSPACE_BYTES of workspace and images; larger batches run in chunks of windows.
FIT_MAX_WINDOWS = 65535
FIT_WORKSPACE_BYTES = 4 << 30


def _objective_and_gradient(x, y, t_rel, p, offsets, opts, rho=None):
    """(B,K) f64 params -> (f (B,) f64, g (B,K) f64) through evk_cmax_motion_objective_f32 / _grad_f32 (grad_f = 1), or
    their depth twins with camera_motion_warp's device inverse depth rho, in chunks of windows (fit_window_chunk); the
    windows are independent, so a chunk changes no value's arithmetic"""
    warp, centre, H, W, objective, sigma, param = opts
    stem, events = _depth_entry("evk_cmax_motion_objective", (x, y, t_rel, p), rho)
    return _chunked_objective(stem, "motion_objective", events, offsets, (warp, centre, H, W), (sigma, objective, param), (1,),
                              FIT_WORKSPACE_BYTES, FIT_MAX_WINDOWS)


def _grid_axes(ranges, num_samples_per_param, log_scale):
    """(B,K,2) f64 ranges -> (B,K,S) axes, each exactly as grid_search_initial builds it (events_cmax.py:241-311)"""
    assert num_samples_per_param % 2 == 1
    half = int(num_samples_per_param / 2.0) + 1
    if log_scale:
        scale = np.logspace(0, 2.0, half)[1:]
        scale /= scale[-1]
    else:
        scale = np.linspace(0, 1.0, half)[1:]
    s = _to_device(torch.from_numpy(scale), ranges.device)
    lo, hi = ranges[..., 0], ranges[..., 1]
    span = hi - lo
    mid = (lo + span / 2.0).unsqueeze(-1)
    half_span = (span / 2.0).unsqueeze(-1)
    return torch.cat(((mid - s * half_span).flip(-1), mid, mid + s * half_span), dim=-1)


def _grid_points(axes):
    """(B,K,S) axes -> (B,S^K,K) points in the order of grid_search_initial's np.meshgrid (first two axes swapped)"""
    B, K, S = axes.shape
    idx = np.vstack([np.ravel(g) for g in np.meshgrid(*([np.arange(S)] * K))])            # (K, S^K)
    idx = _to_device(torch.from_numpy(idx), axes.device)
    return torch.gather(axes, 2, idx.unsqueeze(0).expand(B, K, idx.shape[1])).transpose(1, 2)


def _new_ranges(axes, best):
    """find_new_range (events_cmax.py:160-182) of every axis: (B,K,S) axes and (B,K) best samples -> (B,K,2) ranges"""
    S = axes.shape[-1]
    k = torch.searchsorted(axes.contiguous(), best.unsqueeze(-1).contiguous()).squeeze(-1)
    at = lambda i: torch.gather(axes, 2, i.clamp(0, S - 1).unsqueeze(-1)).squeeze(-1)
    end = (axes[..., -1] - axes[..., -2]).abs()
    below = torch.where(k >= S - 1, end, torch.where(k == 0, (axes[..., 0] - axes[..., -1]).abs(), (at(k) - at(k - 1)).abs()))
    above = torch.where(k >= S - 1, end, (at(k) - at(k + 1)).abs())
    return torch.stack((best - below, best + above), dim=-1)


def _grid_search(evaluate, ranges, num_samples_per_param=5, levels=1, log_scale=False, bounds=None):
    """Coarse-to-fine grid search of every window: `levels` levels of grid_search_initial's grid, each re-centred with
    find_new_range.  evaluate((B,P,K) points) -> (B,P) f.  Returns the (B,K) best point of the last level (the first of
    equal values; a NaN counts as +inf).  bounds: None, or (B,K,2) [lo, hi] that every re-centred range is clamped to
    (find_new_range can step beyond the first level's ranges)."""
    best = None
    for level in range(levels):
        if level:
            ranges = _new_ranges(axes, best)
            if bounds is not None:
                ranges = torch.minimum(torch.maximum(ranges, bounds[..., :1]), bounds[..., 1:])
        axes = _grid_axes(ranges, num_samples_per_param, log_scale)
        pts = _grid_points(axes)
        f = evaluate(pts)
        j = torch.nan_to_num(f, nan=float("inf")).argmin(dim=1)
        best = torch.gather(pts, 1, j.view(-1, 1, 1).expand(-1, 1, pts.shape[2])).squeeze(1)
    return best


def _batched_bfgs(fg, candidates, x0, scale, max_iter=50, line_search_steps=8, ftol=1e-9, gtol=1e-9, bounds=None,
                  unit_first_step=False):
    """
    The BFGS core of motion_contrast_fit_torch, on any batched objective: fg((B,K) x) -> (f (B,), g (B,K)) and
    candidates((B,J,K) points) -> (B,J) f, all f64.  Runs exactly max_iter iterations over every window, under masks.
    bounds: None, or (B,K,2) [lo, hi] per window: a line-search point outside its window's box scores +inf, so no step
    leaves the box.
    unit_first_step: start from H = D / |g * scale| instead of D = diag(scale^2), so that the first step is one unit of
    scale long whatever the size of g (scipy's BFGS likewise makes its first step about one unit long).
    @returns (x (B,K), f (B,), status (B,) int8, iterations (B,) int32)
    """
    x = x0.to(torch.float64).clone()
    B, K = x.shape
    dev = x.device
    scale = scale.to(device=dev, dtype=torch.float64).expand(B, K)
    D = torch.diag_embed(scale * scale)
    Hinv = D.clone()
    f, g = fg(x)
    finite = torch.isfinite(f) & torch.isfinite(g).all(1) & torch.isfinite(x).all(1)
    status = torch.where(finite, torch.full_like(f, ITERATION_LIMIT, dtype=torch.int8),
                         torch.full_like(f, NONFINITE_START, dtype=torch.int8))
    active = finite & ~_small_gradient(g, scale, f, gtol)
    status = torch.where(finite & ~active, torch.zeros_like(status), status)
    iters = torch.zeros(B, dtype=torch.int32, device=dev)
    scaled = torch.zeros(B, dtype=torch.bool, device=dev)     # H rescaled after the first accepted step
    gam = torch.ones(B, dtype=torch.float64, device=dev)      # the latest s'y / y'Dy: a reset starts from gam D
    if unit_first_step:
        gn = (g * scale).norm(dim=1)
        gam = torch.where(finite & (gn > 0), 1.0 / torch.where(gn > 0, gn, torch.ones_like(gn)), gam)
        Hinv = gam.view(-1, 1, 1) * D
    reset = torch.zeros(B, dtype=torch.bool, device=dev)      # H reset since the last accepted step
    alphas = torch.pow(2.0, -torch.arange(line_search_steps, dtype=torch.float64, device=dev))
    for _ in range(max_iter):
        d = -(Hinv @ g.unsqueeze(-1)).squeeze(-1)
        slope = (g * d).sum(1)
        pts = x.unsqueeze(1) + alphas.view(1, -1, 1) * d.unsqueeze(1)
        fc = torch.nan_to_num(candidates(pts), nan=float("inf"))
        if bounds is not None:
            inside = ((pts >= bounds[:, None, :, 0]) & (pts <= bounds[:, None, :, 1])).all(2)
            fc = torch.where(inside, fc, float("inf"))
        armijo = fc <= f.unsqueeze(1) + ARMIJO_C1 * alphas.unsqueeze(0) * slope.unsqueeze(1)
        j_best = fc.argmin(1)
        j = torch.where(armijo.any(1), armijo.to(torch.int8).argmax(1), j_best)
        step = active & (slope < 0) & (armijo.any(1) | (fc.gather(1, j_best.unsqueeze(1)).squeeze(1) < f))
        x_try = torch.where(step.unsqueeze(1), pts.gather(1, j.view(-1, 1, 1).expand(-1, 1, K)).squeeze(1), x)
        f_try, g_try = fg(x_try)
        ok = torch.isfinite(f_try) & torch.isfinite(g_try).all(1)
        # a step the forward does not confirm (the candidates pass and the forward sum f32 images in different orders)
        # is not taken
        accept = step & ok & (f_try <= f)
        # only a full step (alpha = 1) judges convergence by the decrease: a short one says little about the distance left
        converged = accept & (j == 0) & ((f - f_try) < ftol * f.abs())
        converged |= accept & _small_gradient(g_try, scale, f_try, gtol)
        # no accepted step: reset H once, then stop
        failed = active & ~accept
        stop_nd = failed & reset
        do_reset = failed & ~reset
        s = x_try - x
        yv = g_try - g
        sy = (s * yv).sum(1)
        upd = accept & (sy > 1e-10 * s.norm(dim=1) * yv.norm(dim=1)) & (sy > 0)
        # first accepted step: H = (s'y / y'Dy) D, the s'y / y'y rescaling in the coordinates x / scale
        yDy = (yv * scale * scale * yv).sum(1)
        gam = torch.where(upd & (yDy > 0), sy / torch.where(yDy > 0, yDy, torch.ones_like(yDy)), gam)
        first = upd & ~scaled
        Hs = torch.where(first.view(-1, 1, 1), gam.view(-1, 1, 1) * D, Hinv)
        Hnew = _bfgs_update(Hs, s, yv, torch.where(upd, sy, torch.ones_like(sy)))
        Hinv = torch.where(upd.view(-1, 1, 1), Hnew, torch.where(do_reset.view(-1, 1, 1), gam.view(-1, 1, 1) * D, Hinv))
        scaled |= upd
        reset = torch.where(accept, torch.zeros_like(reset), reset | do_reset)
        x = torch.where(accept.unsqueeze(1), x_try, x)
        f = torch.where(accept, f_try, f)
        g = torch.where(accept.unsqueeze(1), g_try, g)
        iters += accept.to(torch.int32)
        status = torch.where(active & converged, torch.zeros_like(status), status)
        status = torch.where(stop_nd, torch.full_like(status, NO_DESCENT), status)
        active = active & ~converged & ~stop_nd
    return x, f, status, iters


def _small_gradient(g, scale, f, gtol):
    return (g * scale).abs().amax(1) <= gtol * f.abs()


def _bfgs_update(Hm, s, y, sy):
    """H+ = (I - rho s y') H (I - rho y s') + rho s s', rho = 1 / s'y, for every window"""
    rho = (1.0 / sy).view(-1, 1, 1)
    K = s.shape[1]
    I = torch.eye(K, dtype=Hm.dtype, device=Hm.device).expand_as(Hm)
    V = I - rho * s.unsqueeze(2) * y.unsqueeze(1)
    return V @ Hm @ V.transpose(1, 2) + rho * s.unsqueeze(2) * s.unsqueeze(1)
