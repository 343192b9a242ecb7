"""Depth from a known camera motion: an inverse-depth field per event window, given on a coarse grid of nodes, as a
batched, differentiable contrast loss, its candidates pass and a coarse-to-fine fit.

camera_motion_warp explains events with the camera's velocity (w, v) and the inverse depth rho of every event, which
its callers had to know.  Depth from a known motion is the third canonical contrast-maximisation problem next to
optical flow and rotation (Gallego, Rebecq, Scaramuzza, CVPR 2018): with (w, v) known, from an IMU, odometry or a
camera_motion_warp fit, the events are sharpest at the scene's depth.  Here rho is a smooth field over the sensor on a
gh x gw grid of nodes, interpolated bilinearly at every event as the grid-flow loss interpolates its flow, and the
loss is the camera-motion contrast loss at that rho, computed without forming a per-event rho array: each event's node
cell, weights and rotation are computed once per pass, and the backward sums the node gradient of a CTA in shared
memory (evk_cmax_depth_grid_objective_f32 / _grad_f32, evk_cmax_depth_grid_candidates_f32).
"""
import collections

import torch

from .. import _lib
from ..representations import _events as E
from ._batched import (_batch_events, _centre, _check_objective, _chunked_candidates, _chunked_objective, _event_tensors,
                       _float_tensor, _rows, _window_count)
from .grid_flow import MAX_FIT_PARAMETERS, MAX_GRID_NODES, _check_grid_shape, _scalars, _stages
from .motion_fit import (FIT_MAX_WINDOWS, FIT_WORKSPACE_BYTES, _check_line_search_steps, _check_per_window, _grid_search,
                         _per_window)
from .motion_objective import CANDIDATES_WORKSPACE_BYTES
from .warps import camera_motion_warp

DepthGridFit = collections.namedtuple("DepthGridFit", "inv_depth f contrast status iterations")
DepthGridFit.__doc__ = """depth_grid_fit_torch's result: inv_depth (B,gh,gw) f64 on the last grid, f (B,) f64 = contrast
+ smoothness R (the fitted objective), contrast (B,) f64, status (B,) int8, iterations (B,) int32"""


def _check_warp(warpfunc, who):
    if type(warpfunc) is not camera_motion_warp:
        raise ValueError("%s takes the camera's intrinsics from a camera_motion_warp, got %s" % (who, type(warpfunc).__name__))


def _depth_grid_tensor(grid, H, W, name="inv_depth_grid", lead=1):
    """grid as a (B,gh,gw) (lead 1) or (B,J,gh,gw) (lead 2) float tensor, checked against the node limits"""
    g = _float_tensor(grid, name)
    if lead == 1 and g.dim() == 2:
        g = g.unsqueeze(0)
    if g.dim() != 2 + lead or (lead == 2 and g.shape[1] < 1):
        raise ValueError("%s must have shape %s, got %s" % (name, "(B,gh,gw) or (gh,gw)" if lead == 1 else
                                                            "(B,J,gh,gw) with J >= 1", tuple(g.shape)))
    _check_grid_shape(g.shape[-2], g.shape[-1], H, W, MAX_GRID_NODES)
    return g


def _model(motion, warpfunc, B, dev, grid, H, W):
    """the layout of the depth-grid entries (_batched._model_layout): the motion (6,) or (B,6) as device rows
    (wx, wy, wz, vx, vy, vz, fx, fy) f64 of every window, copied without a host wait, and the principal point"""
    centre = _centre(_lib.WARP_CAMERA_MOTION, warpfunc)
    rows = _rows(_per_window(motion, B, (6,), "motion", dev), centre).contiguous()
    return ("grid", grid, H, W, (rows, centre[0], centre[1]))


def _candidates(ev, c, model, scalars):
    """f (B,J) f64 of the prepared device events ev under the device candidates c (B,J,gh gw) f32"""
    return _chunked_candidates("evk_cmax_depth_grid_candidates", "depth_grid_candidates", ev[:4], ev[4], c, model, scalars,
                               CANDIDATES_WORKSPACE_BYTES, 65535)


def depth_grid_contrast_objective_torch(xs, ys, ts, ps, inv_depth_grid, motion, warpfunc, img_size, t0=None,
                                        objective="variance", blur_sigma=1.0, obj_param=None, batch_end_indices=None):
    """
    Contrast objective f_b of every sample b of a batch of event windows, seen by a camera with the known motion
    motion[b] = (wx, wy, wz, vx, vy, vz) (camera_motion_warp's parameters and units, with warpfunc's intrinsics), through
    a scene whose inverse depth is given on a grid of nodes.  inv_depth_grid[b] is (gh, gw) with 2 <= gh <= H,
    2 <= gw <= W and gh gw <= 4096, (H, W) = img_size.  Node (i, j) sits at pixel (j (W-1)/(gw-1), i (H-1)/(gh-1))
    (align_corners), and an event at (x, y) takes rho interpolated bilinearly from the nodes at
    (x (gw-1)/(W-1), y (gh-1)/(H-1)), with the node cell, weights and zero outside taps of
    grid_flow_contrast_objective_torch.  Everything after that is motion_contrast_objective_torch with
    camera_motion_warp and inv_depth = that rho: the keep rules (a negative or non-finite rho is dropped, and so is
    Pz <= 0), the bounds mask, the (H+1, W+1) canvas, the blur and the objectives variance / sos / soe / sosa.
    The field is the inverse depth seen at each sensor pixel, taken as static over the window: the approximation the
    per-event inverse depth of camera_motion_warp already makes when one depth map is sampled at the events.  At
    gh = H, gw = W with events at integer pixels rho is the node at the event's pixel; for a constant grid c, f is the
    loss at inv_depth = c to f32 rounding; at v = 0 f is camera_rotation_warp's and the gradient is zero.
    @param inv_depth_grid (B,gh,gw) or (gh,gw), in 1 / (the depth unit of v); the only differentiable input
    @param motion (B,6) or (6,) camera motions (data: no gradient; depth and translation share one scale factor)
    @param warpfunc a camera_motion_warp, whose intrinsics are used
    @returns (B,) tensor of f in inv_depth_grid's dtype, on its device.  With every input on the GPU neither the forward
           nor the backward synchronises with the host.  The backward is accurate to f32 rounding.
    """
    who = "depth_grid_contrast_objective_torch"
    _check_warp(warpfunc, who)
    _check_objective(objective, "inverse depth")
    xs, ys, ts, ps = _event_tensors(xs, ys, ts, ps, t0, who, "the inverse-depth grid")
    H, W = int(img_size[0]), int(img_size[1])
    g = _depth_grid_tensor(inv_depth_grid, H, W)
    B, gh, gw = g.shape
    _check_per_window(motion, B, (6,), "motion")
    _lib.lib()
    dev = E.compute_device(g, xs, ys, ts, ps)
    x, y, t_rel, p, offsets = _batch_events(xs, ys, ts, ps, t0, batch_end_indices, B, dev, "inverse-depth grids")
    from ..autograd import DepthGridObjective
    with torch.cuda.device(dev):
        model = _model(motion, warpfunc, B, dev, (gh, gw), H, W)
    f = DepthGridObjective.apply(g, x, y, t_rel, p, offsets, model[4] + (H, W) + _scalars(objective, blur_sigma, obj_param))
    return f.to(device=g.device, dtype=g.dtype)


def depth_grid_contrast_candidates_torch(xs, ys, ts, ps, candidates, motion, warpfunc, img_size, t0=None,
                                         objective="variance", blur_sigma=1.0, obj_param=None, batch_end_indices=None):
    """
    The depth-grid contrast objective of every window b under each of its J candidate grids candidates[b, j]: f[b, j] is
    the f_b that depth_grid_contrast_objective_torch returns with inv_depth_grid[b] = candidates[b, j].  Each pass over
    the events scores up to min(32, 12288 // (gh gw)) candidates of every window (evk_cmax_depth_grid_candidates_f32),
    and the windows run in chunks whose workspace stays under CANDIDATES_WORKSPACE_BYTES; neither split changes a value.
    @param candidates (B,J,gh,gw) inverse-depth grids, any float dtype (rounded to f32), any J >= 1
    @returns (B,J) f64 tensor of values (no autograd graph) on candidates' device
    """
    who = "depth_grid_contrast_candidates_torch"
    _check_warp(warpfunc, who)
    _check_objective(objective, "inverse depth")
    xs, ys, ts, ps = _event_tensors(xs, ys, ts, ps, t0, who, "nothing")
    H, W = int(img_size[0]), int(img_size[1])
    cand = _depth_grid_tensor(candidates, H, W, "candidates", lead=2)
    B, J, gh, gw = cand.shape
    _check_per_window(motion, B, (6,), "motion")
    _lib.lib()
    dev = E.compute_device(cand, xs, ys, ts, ps)
    ev = _batch_events(xs, ys, ts, ps, t0, batch_end_indices, B, dev, "candidate sets")
    with torch.cuda.device(dev):
        c = cand.detach().to(device=dev, dtype=torch.float32).reshape(B, J, gh * gw)
        f = _candidates(ev, c, _model(motion, warpfunc, B, dev, (gh, gw), H, W),
                        _scalars(objective, blur_sigma, obj_param))
    return f.to(cand.device)


def depth_grid_fit_torch(xs, ys, ts, ps, motion, warpfunc, img_size, inv_depth_range,
                         grid_shapes=((3, 4), (6, 8), (12, 16)), smoothness=1e-2, charbonnier_eps=0.05,
                         batch_end_indices=None, t0=None, objective="variance", blur_sigma=1.0, obj_param=None, x0=None,
                         num_samples=15, grid_levels=2, max_iter=50, line_search_steps=8, ftol=1e-9, gtol=1e-9):
    """
    Fit an inverse-depth grid to every event window on its own, all windows at once, coarse to fine, with the camera
    motion known: minimise
        F_b(D) = f_b(D) + smoothness R(D)
    over the nodes D, with f_b the loss of depth_grid_contrast_objective_torch (same windows, motion, warpfunc, t0,
    objective, blur_sigma, obj_param and img_size, so any result can be checked with it) and R
    charbonnier_smoothness(D, charbonnier_eps) over neighbouring nodes (not normalised by the grid size).
    Every node is boxed to inv_depth_range ((2,) or (B,2): [lo, hi] with 0 <= lo < hi, in 1 / the depth unit of v),
    which is required: contrast maximisation collapses the events when depth is free -- with a forward component of v a
    large rho sends every event towards the focus of expansion, and the contrast keeps growing.
    Start: x0 ((gh0,gw0) or (B,gh0,gw0) on the first grid) if given; otherwise a constant inverse depth per window from
    a grid search over inv_depth_range (motion_contrast_fit_torch's grid: num_samples odd points, grid_levels levels,
    each refined range clamped to the box), each level one candidates pass over constant grids.
    Stages: for each (gh, gw) of grid_shapes, the previous result is upsampled to the new grid (bilinear,
    align_corners=True, in f64) and clamped to the box, then for each blur of blur_sigma (a number or a sequence)
    motion_contrast_fit_torch's BFGS runs on F over the K = gh gw nodes (K <= 512: the inverse Hessians are dense),
    its first step one grid spacing (hi - lo) / (num_samples - 1) long, its line searches one candidates pass each.
    Every stage runs exactly max_iter iterations on all windows, so with the events, window ends, motion and
    inv_depth_range on the GPU the fit never synchronises with the host.
    The defaults of smoothness, charbonnier_eps, num_samples and grid_levels were chosen on the slanted-plane and
    two-plane windows of the tests (rho 0.2-1 per m, 1 m/s): see DESIGN.md section 6.
    @returns DepthGridFit(inv_depth (B,gh,gw) f64 on the last grid, f (B,) f64 = F for the last blur, contrast (B,) f64 =
             f - smoothness R, status (B,) int8 of the last stage, iterations (B,) int32 summed over the stages), on the
             events' device.
    """
    who = "depth_grid_fit_torch"
    _check_warp(warpfunc, who)
    _check_objective(objective, "inverse depth")
    xs, ys, ts, ps = _event_tensors(xs, ys, ts, ps, t0, who, "nothing")

    def events(B, dev):
        return _batch_events(xs, ys, ts, ps, t0, batch_end_indices, B, dev, "windows")

    def loss(ev, model, sigma):
        return _chunked_objective("evk_cmax_depth_grid_objective", "depth_grid_objective", ev[:4], ev[4], model,
                                  _scalars(objective, sigma, obj_param), (1,), FIT_WORKSPACE_BYTES, FIT_MAX_WINDOWS)

    def candidates(ev, c, model, sigma):
        return _candidates(ev, c, model, _scalars(objective, sigma, obj_param))
    return DepthGridFit(*_depth_grid_fit(who, (xs, ys, ts, ps), motion, warpfunc, img_size, inv_depth_range, grid_shapes,
                                         smoothness, charbonnier_eps, batch_end_indices, blur_sigma, x0, num_samples,
                                         grid_levels, max_iter, line_search_steps, ftol, gtol, events, loss, candidates))


def _depth_grid_fit(who, tensors, motion, warpfunc, img_size, inv_depth_range, grid_shapes, smoothness, charbonnier_eps,
                    batch_end_indices, blur_sigma, x0, num_samples, grid_levels, max_iter, line_search_steps, ftol, gtol,
                    events, loss, candidates):
    """The coarse-to-fine, boxed fit of F = f + smoothness R that depth_grid_fit_torch and depth_grid_timestamp_fit_torch
    share: the argument checks (before any CUDA call), the constant start and the BFGS stages per grid shape and blur.
    tensors: the events, which with x0, inv_depth_range and motion choose the device;  events(B, dev) -> the prepared
    device events;  loss(events, model, sigma) -> fg of f on the nodes (_chunked_objective);  candidates(events, c,
    model, sigma) -> f (B,J) f64 of the f32 node grids c (B,J,gh gw), with model = _model's layout for the grid (gh, gw).
    Returns (inv_depth (B,gh,gw), F, f, status, iterations)."""
    H, W = int(img_size[0]), int(img_size[1])
    shapes = [(int(a), int(b)) for a, b in grid_shapes]
    if not shapes:
        raise ValueError("grid_shapes must name at least one (gh, gw)")
    for gh, gw in shapes:
        _check_grid_shape(gh, gw, H, W, MAX_GRID_NODES)
        if gh * gw > MAX_FIT_PARAMETERS:
            raise ValueError("%s keeps a dense inverse Hessian of K = gh gw <= %d parameters per window; a %d x %d grid "
                             "has K = %d" % (who, MAX_FIT_PARAMETERS, gh, gw, gh * gw))
    sigmas = [float(s) for s in (blur_sigma if isinstance(blur_sigma, (list, tuple)) else [blur_sigma])]
    if not sigmas:
        raise ValueError("blur_sigma must be a number or a non-empty sequence")
    _check_line_search_steps(line_search_steps)
    if float(smoothness) < 0 or not float(charbonnier_eps) > 0:
        raise ValueError("smoothness must be >= 0 and charbonnier_eps > 0")
    if inv_depth_range is None:
        raise ValueError("%s needs inv_depth_range, the [lo, hi] box of every node" % who)
    B = _window_count(batch_end_indices)
    _check_per_window(inv_depth_range, B, (2,), "inv_depth_range")
    if not isinstance(inv_depth_range, torch.Tensor) or inv_depth_range.device.type == "cpu":
        r = torch.as_tensor(inv_depth_range, dtype=torch.float64)
        if not bool(((r[..., 0] >= 0) & (r[..., 0] < r[..., 1])).all()):
            raise ValueError("inv_depth_range must have 0 <= lo < hi, got %s" % (r.tolist(),))
    _check_per_window(motion, B, (6,), "motion")
    gh0, gw0 = shapes[0]
    if x0 is not None:
        _check_per_window(x0, B, (gh0, gw0), "x0")
    elif int(num_samples) < 1 or int(num_samples) % 2 != 1 or int(grid_levels) < 1:
        raise ValueError("num_samples must be odd and grid_levels >= 1, got %r and %r" % (num_samples, grid_levels))
    lam, eps = float(smoothness), float(charbonnier_eps)
    _lib.lib()
    dev = E.compute_device(*(a for a in (x0, inv_depth_range, motion) + tuple(tensors) if isinstance(a, torch.Tensor)))
    ev = events(B, dev)
    with torch.cuda.device(dev):
        box = _per_window(inv_depth_range, B, (2,), "inv_depth_range", dev).unsqueeze(1)     # (B,1,2)
        scale = (box[:, 0, 1] - box[:, 0, 0]) / (max(int(num_samples), 2) - 1)
        motion_model = _model(motion, warpfunc, B, dev, None, H, W)[4]

        def stage_loss(ev, grid, sigma):
            model = ("grid", grid, H, W, motion_model)
            return loss(ev, model, sigma), lambda c: candidates(ev, c, model, sigma)
        if x0 is None:
            start = _constant_start(ev, box, (gh0, gw0), H, W, motion_model, sigmas[0], int(num_samples), int(grid_levels),
                                    candidates)
            grid = start.view(B, 1, 1, 1).expand(B, 1, gh0, gw0).contiguous()
        else:
            grid = _per_window(x0, B, (gh0, gw0), "x0", dev).unsqueeze(1)
        D, f, rest, status, iters = _stages(grid, shapes, sigmas, box, scale, ev, stage_loss, lam, eps, max_iter,
                                            line_search_steps, ftol, gtol)
    return D[:, 0], f, rest, status, iters


def _constant_start(ev, box, grid, H, W, motion_model, sigma, num_samples, levels, candidates):
    """(B,) f64: the best constant inverse depth of every window, grid-searched inside the box (B,1,2) with the
    candidates function of _depth_grid_fit"""
    gh, gw = grid
    model = ("grid", grid, H, W, motion_model)

    def evaluate(pts):
        B, P, _ = pts.shape
        return candidates(ev, pts.to(torch.float32).expand(B, P, gh * gw).contiguous(), model, sigma)
    return _grid_search(evaluate, box, num_samples, levels, bounds=box)[:, 0]
