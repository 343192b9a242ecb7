"""Depth from a known camera motion with the average-timestamp loss of Zhu et al. (CVPR'19): an inverse-depth field per
event window, given on a coarse grid of nodes, as a batched, differentiable loss, its candidates pass and a boxed
coarse-to-fine fit.

The loss is the camera-motion timestamp loss of motion_timestamp_objective.py (camera_motion_warp with a per-event
inverse depth) at the rho that depth_grid.py interpolates from the nodes, computed without forming a per-event rho
array: each event's node cell, weights and rotation are computed once per pass, and the backward sums the node gradient
of a CTA in shared memory (evk_depth_grid_timestamp_objective_f32 / _grad_f32, evk_depth_grid_timestamp_candidates_f32).
The fit is depth_grid.py's, with this loss.
"""
import collections

import torch

from .. import _lib
from ..representations import _events as E
from ._batched import _chunked_candidates, _chunked_objective, _event_tensors, _timestamp_events
from .depth_grid import _check_warp, _depth_grid_fit, _depth_grid_tensor, _model
from .grid_flow_timestamp import _blur_sigma
from .motion_fit import FIT_WORKSPACE_BYTES, _check_per_window
from .motion_timestamp_fit import TIMESTAMP_FIT_MAX_WINDOWS
from .motion_timestamp_objective import TIMESTAMP_CANDIDATES_WORKSPACE_BYTES

DepthGridTimestampFit = collections.namedtuple("DepthGridTimestampFit", "inv_depth f loss status iterations")
DepthGridTimestampFit.__doc__ = """depth_grid_timestamp_fit_torch's result: inv_depth (B,gh,gw) f64 on the last grid, f (B,)
f64 = loss + smoothness R (the fitted objective), loss (B,) f64 (Zhu's loss), status (B,) int8, iterations (B,) int32"""


def depth_grid_timestamp_objective_torch(xs, ys, ts, ps, inv_depth_grid, motion, warpfunc, img_size, t0=None,
                                         blur_sigma=2.0, timestamp_reverse=False, batch_end_indices=None):
    """
    Average-timestamp loss f_b of every sample b of a batch of event windows, seen by a camera with the known motion
    motion[b] = (wx, wy, wz, vx, vy, vz) (camera_motion_warp's parameters and units, with warpfunc's intrinsics), through
    a scene whose inverse depth is given on a grid of nodes.  inv_depth_grid[b] is (gh, gw) with 2 <= gh <= H,
    2 <= gw <= W and gh gw <= 4096, (H, W) = img_size, and an event takes rho interpolated from the nodes exactly as in
    depth_grid_contrast_objective_torch (align_corners, f32 ratios and products, zero outside taps).  Everything after
    that is motion_timestamp_objective_torch with camera_motion_warp and inv_depth = that rho: samples, t0, the
    normalised stamps and timestamp_reverse, the keep rules (a negative or non-finite rho, Pz <= 0 or a non-finite Pz,
    the bounds mask: not kept, and a non-finite warp never makes f NaN), weight 1, a NaN p dropped, the per-polarity
    images T = S / C on the (H+1, W+1) canvas, the blur and f_b = sum(G_+^2) + sum(G_-^2).  At gh = H, gw = W with
    events at integer pixels rho is the node at the event's pixel; for a constant grid c, f is the loss at
    inv_depth = c to f32 rounding; at v = 0 f is camera_rotation_warp's and the gradient is zero.
    @param inv_depth_grid (B,gh,gw) or (gh,gw), in 1 / (the depth unit of v); the only differentiable input
    @param motion (B,6) or (6,) camera motions (data: no gradient; depth and translation share one scale factor)
    @param warpfunc a camera_motion_warp, whose intrinsics are used
    @returns (B,) tensor of f in inv_depth_grid's dtype, on its device, 0 <= B <= 32767.  With every input on the GPU
           neither the forward nor the backward synchronises with the host.  The backward is accurate to f32 rounding.
    """
    who = "depth_grid_timestamp_objective_torch"
    _check_warp(warpfunc, who)
    xs, ys, ts, ps = _event_tensors(xs, ys, ts, ps, t0, who, "the inverse-depth grid")
    H, W = int(img_size[0]), int(img_size[1])
    g = _depth_grid_tensor(inv_depth_grid, H, W)
    B, gh, gw = g.shape
    _check_per_window(motion, B, (6,), "motion")
    sigma = _blur_sigma(blur_sigma)
    _lib.lib()
    dev = E.compute_device(g, xs, ys, ts, ps)
    ev = _timestamp_events(xs, ys, ts, ps, t0, batch_end_indices, B, dev, "inverse-depth grids", timestamp_reverse)
    from ..autograd import DepthGridTimestampObjective
    with torch.cuda.device(dev):
        model = _model(motion, warpfunc, B, dev, (gh, gw), H, W)
    f = DepthGridTimestampObjective.apply(g, *ev, model[4] + (H, W, sigma))
    return f.to(device=g.device, dtype=g.dtype)


def depth_grid_timestamp_candidates_torch(xs, ys, ts, ps, candidates, motion, warpfunc, img_size, t0=None, blur_sigma=2.0,
                                          timestamp_reverse=False, batch_end_indices=None):
    """
    The depth-grid average-timestamp loss of every window b under each of its J candidate grids candidates[b, j]:
    f[b, j] is the f_b that depth_grid_timestamp_objective_torch returns with inv_depth_grid[b] = candidates[b, j].  Each
    pass over the events scores up to min(32, 12288 // (gh gw)) candidates of every window
    (evk_depth_grid_timestamp_candidates_f32), and the windows run in chunks of at most 32767 // (candidates per pass)
    whose workspace stays under TIMESTAMP_CANDIDATES_WORKSPACE_BYTES; neither split changes a value.
    @param candidates (B,J,gh,gw) inverse-depth grids, any float dtype (rounded to f32), any J >= 1
    @returns (B,J) f64 tensor of values (no autograd graph) on candidates' device
    """
    who = "depth_grid_timestamp_candidates_torch"
    _check_warp(warpfunc, who)
    xs, ys, ts, ps = _event_tensors(xs, ys, ts, ps, t0, who, "nothing")
    H, W = int(img_size[0]), int(img_size[1])
    cand = _depth_grid_tensor(candidates, H, W, "candidates", lead=2)
    B, J, gh, gw = cand.shape
    _check_per_window(motion, B, (6,), "motion")
    sigma = _blur_sigma(blur_sigma)
    _lib.lib()
    dev = E.compute_device(cand, xs, ys, ts, ps)
    ev = _timestamp_events(xs, ys, ts, ps, t0, batch_end_indices, B, dev, "candidate sets", timestamp_reverse)
    with torch.cuda.device(dev):
        c = cand.detach().to(device=dev, dtype=torch.float32).reshape(B, J, gh * gw)
        f = _candidates(ev, c, _model(motion, warpfunc, B, dev, (gh, gw), H, W), sigma)
    return f.to(cand.device)


def _candidates(ev, c, model, sigma):
    """f (B,J) f64 of the prepared device events ev (_timestamp_events) under the device candidates c (B,J,gh gw) f32"""
    return _chunked_candidates("evk_depth_grid_timestamp_candidates", "depth_grid_timestamp_candidates", ev[:5], ev[5], c,
                               model, (sigma,), TIMESTAMP_CANDIDATES_WORKSPACE_BYTES, 32767)


def depth_grid_timestamp_fit_torch(xs, ys, ts, ps, motion, warpfunc, img_size, inv_depth_range,
                                   grid_shapes=((3, 4), (6, 8), (12, 16)), smoothness=1.0, charbonnier_eps=0.05,
                                   batch_end_indices=None, t0=None, blur_sigma=2.0, timestamp_reverse=False, x0=None,
                                   num_samples=15, grid_levels=2, max_iter=50, line_search_steps=8, ftol=1e-9, gtol=1e-9):
    """
    Fit an inverse-depth grid to every event window on its own, all windows at once, coarse to fine, with the camera
    motion known: minimise
        F_b(D) = f_b(D) + smoothness R(D)
    over the nodes D, with f_b the loss of depth_grid_timestamp_objective_torch (same windows, motion, warpfunc, t0,
    stamps, blur_sigma and img_size, so any result can be checked with it) and R charbonnier_smoothness(D,
    charbonnier_eps).  Direction: this MINIMISES Zhu's loss, as motion_timestamp_fit_torch does.  The start (a constant
    inverse depth per window from a grid search of num_samples points and grid_levels levels over the box, or x0), the
    stages, the upsampling and clamping between grids, the BFGS over K = gh gw <= 512 nodes, the statuses and the
    absence of host synchronisation are depth_grid_fit_torch's; each forward and gradient call takes a chunk of
    max(1, min(B, FIT_WORKSPACE_BYTES // (workspace + images per window), 32767)) windows and each candidates call a
    chunk as depth_grid_timestamp_candidates_torch's.
    The box inv_depth_range ((2,) or (B,2): [lo, hi] with 0 <= lo < hi) is required, and it matters more here than for
    the contrast fit: an event warped off the canvas adds nothing to Zhu's loss, so a node pushed to a large rho can
    lower f by sending the edge events near it off the sensor, the degenerate minimum grid_flow_timestamp_fit_torch's
    bounds guard against.  The line search scores a point outside the box +inf and rejects it rather than projecting it
    onto the box, so such a node stops at its last accepted point inside the box, near hi, not necessarily on the face.
    tools/bench_depth_grid_timestamp.py reports, per window, the share of nodes within 1 % of (hi - lo) of a face, the
    error of the border nodes and the share of events the fitted grid warps off the canvas.
    smoothness and charbonnier_eps: the defaults were chosen on the windows of tests/test_gpu_depth_grid.py's recovery
    test (a slanted plane, a step between two planes, a slanted plane with a forward component of v; rho 0.2-1 per m),
    see DESIGN.md section 6.  Zhu's loss sums squared timestamp images over the canvas, so its scale, and the
    smoothness that balances it, is not the contrast loss's.
    @returns DepthGridTimestampFit(inv_depth (B,gh,gw) f64 on the last grid, f (B,) f64 = F for the last blur, loss (B,)
             f64 = f - smoothness R, status (B,) int8 of the last stage, iterations (B,) int32 summed over the stages),
             on the events' device.
    """
    who = "depth_grid_timestamp_fit_torch"
    _check_warp(warpfunc, who)
    xs, ys, ts, ps = _event_tensors(xs, ys, ts, ps, t0, who, "nothing")
    for s in (blur_sigma if isinstance(blur_sigma, (list, tuple)) else [blur_sigma]):
        _blur_sigma(s)
    H, W = int(img_size[0]), int(img_size[1])

    def events(B, dev):
        return _timestamp_events(xs, ys, ts, ps, t0, batch_end_indices, B, dev, "windows", timestamp_reverse)

    def loss(ev, model, sigma):
        return _chunked_objective("evk_depth_grid_timestamp_objective", "depth_grid_timestamp_objective", ev[:5], ev[5],
                                  model, (sigma,), (2, 2), FIT_WORKSPACE_BYTES, TIMESTAMP_FIT_MAX_WINDOWS)
    return DepthGridTimestampFit(*_depth_grid_fit(who, (xs, ys, ts, ps), motion, warpfunc, (H, W), inv_depth_range,
                                                  grid_shapes, smoothness, charbonnier_eps, batch_end_indices, blur_sigma,
                                                  x0, num_samples, grid_levels, max_iter, line_search_steps, ftol, gtol,
                                                  events, loss, _candidates))
