"""Fit one motion per event window to the average-timestamp loss of Zhu et al. (CVPR'19) on the GPU: a grid search per
window, then batched BFGS, as motion_contrast_fit_torch fits the contrast loss.

The reference's only fit of this loss is optimize_contrast(..., zhu_timestamp_objective()) (events_cmax.py:313-346): one
window per call, a warp on the host and numeric gradients.  motion_timestamp_fit_torch fits B windows at once: every grid
level and every line search is ONE candidates pass over the events (motion_timestamp_candidates_torch), and f and its
gradient are one call each of the batched loss's C entries.
"""
import torch

from .. import _lib
from ..representations import _events as E
from ._batched import (_chunked_objective, _depth_entry, _depth_events, _depth_tensor, _event_tensors, _timestamp_events,
                       _ts_model, _warp_code, _window_count)
from .motion_fit import FIT_WORKSPACE_BYTES, _check_per_window, _fit_arguments, _fit_stages
from .motion_timestamp_objective import _ts_candidates

# One forward + gradient call of motion_timestamp_fit_torch takes at most this many windows (the entries' batch limit:
# two tail images per window) and at most as many as fit motion_fit.FIT_WORKSPACE_BYTES
TIMESTAMP_FIT_MAX_WINDOWS = 32767


def motion_timestamp_fit_torch(xs, ys, ts, ps, warpfunc, batch_end_indices=None, t0=None, blur_sigma=2.0,
                               timestamp_reverse=False, img_size=(180, 240), x0=None, param_ranges=None, bounds=None,
                               num_samples_per_param=5, grid_levels=1, log_scale=False, param_scale=None, max_iter=50,
                               line_search_steps=8, ftol=1e-9, gtol=1e-9, inv_depth=None):
    """
    Minimise the f_b of motion_timestamp_objective_torch over the parameters of every window b on its own, all windows at
    once.  The windows, t0, stamps (timestamp_reverse), blur and img_size are those of motion_timestamp_objective_torch,
    so any result can be checked with it.
    Direction: this MINIMISES Zhu's loss, f = sum G(T_+)^2 + sum G(T_-)^2, which is smallest at the true motion.  The
    reference's optimize_contrast(..., zhu_timestamp_objective()) minimises -f (objectives.py:550), i.e. maximises the
    loss, which drives its fit away from the motion; no option here reproduces that direction.
    Start point, refinement, stages (blur_sigma may be a sequence), tolerances, statuses and the absence of host
    synchronisation are those of motion_contrast_fit_torch, with f and g from evk_motion_timestamp_objective_f32 /
    _grad_f32 and every grid level and line search one evk_motion_timestamp_candidates_f32 pass.
    Any number of windows B: each candidates call runs the windows in chunks of
    max(1, min(B, TIMESTAMP_CANDIDATES_WORKSPACE_BYTES // its workspace per window, 32767 // min(J, 32))) windows (J the
    candidates of the call: num_samples_per_param^K for a grid level, line_search_steps for a line search), and each
    forward and gradient call in chunks of max(1, min(B, FIT_WORKSPACE_BYTES // (workspace + images per window), 32767)).
    The launch sequence depends on B only through those numbers of chunks.
    One difference: the inverse Hessian starts as diag(param_scale^2) / |g * param_scale|, so that the first step is one
    unit of param_scale long.  This loss's gradient is large against its scale (f is a sum over the canvas, not a
    mean), and a first step of H g with H = diag(param_scale^2) overshoots by far more than the 2^-(line_search_steps-1)
    the line search can shorten it by.
    camera_motion_warp takes inv_depth, the inverse depth of every event, and starts from x0 as in
    motion_contrast_fit_torch.
    Bounds: an event warped off the canvas adds nothing to f, so a motion that sends every event off the canvas has
    f = 0, the loss's global minimum, and a long step can reach it.  bounds ((K,2) or (B,K,2), [lo, hi] per parameter)
    confines every line search to a box: a point outside scores +inf and is never taken.  With param_ranges and no
    bounds, the box is param_ranges widened by one level-0 grid step on each side (grid points lie on the ranges' edges,
    and a start on the box's edge could not step outwards), and further where the grid's best point lies beyond it.  With x0 and no bounds the fit is UNBOUNDED and a window may end on such a degenerate minimum: pass bounds.
    @returns MotionFit(params (B,K) f64, f (B,) f64 at params for the last stage's blur, status (B,) int8, iterations
             (B,) int32) on the events' device, as motion_contrast_fit_torch.  An empty window, or one whose start keeps
             no event, has g = 0 and returns its start as converged.
    """
    warp = _warp_code(warpfunc, "motion_timestamp_fit_torch")
    xs, ys, ts, ps = _event_tensors(xs, ys, ts, ps, t0, "motion_timestamp_fit_torch", "nothing")
    rho = _depth_tensor(inv_depth, warp, xs.shape[0], "motion_timestamp_fit_torch")
    sigmas = _fit_arguments("motion_timestamp_fit_torch", blur_sigma, line_search_steps, x0, param_ranges)
    K = warpfunc.dims
    B = _window_count(batch_end_indices)
    if bounds is not None:
        _check_per_window(bounds, B, (K, 2), "bounds")
    H, W = int(img_size[0]), int(img_size[1])
    _lib.lib()
    dev = E.compute_device(*(a for a in (x0, param_ranges, bounds, xs, ys, ts, ps) if isinstance(a, torch.Tensor)))
    x, y, t_rel, tau, p, offsets = _timestamp_events(xs, ys, ts, ps, t0, batch_end_indices, B, dev, "windows", timestamp_reverse)
    rho = _depth_events(rho, dev)
    with torch.cuda.device(dev):

        def stage(sigma):
            opts = _ts_model(warp, warpfunc, sigma, H, W)
            return (_objective_and_gradient(x, y, t_rel, tau, p, offsets, opts, rho),
                    lambda c: _ts_candidates(x, y, t_rel, tau, p, offsets, c, opts, rho))
        return _fit_stages(stage, sigmas, B, K, dev, x0, param_ranges, num_samples_per_param, grid_levels, log_scale,
                           param_scale, max_iter, line_search_steps, ftol, gtol, bounds, bound_to_ranges=True,
                           unit_first_step=True)


def _objective_and_gradient(x, y, t_rel, tau, p, offsets, opts, rho=None):
    """(B,K) f64 params -> (f (B,) f64, g (B,K) f64) through evk_motion_timestamp_objective_f32 / _grad_f32 (grad_f = 1),
    or their depth twins with camera_motion_warp's device inverse depth rho, in chunks of at most
    TIMESTAMP_FIT_MAX_WINDOWS windows whose workspace and images fit FIT_WORKSPACE_BYTES; the windows are independent, so
    a chunk changes no value's arithmetic"""
    warp, centre, H, W, sigma = opts
    stem, events = _depth_entry("evk_motion_timestamp_objective", (x, y, t_rel, tau, p), rho)
    return _chunked_objective(stem, "motion_timestamp_objective", events, offsets, (warp, centre, H, W), (sigma,), (2, 2),
                              FIT_WORKSPACE_BYTES, TIMESTAMP_FIT_MAX_WINDOWS)
