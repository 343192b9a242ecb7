"""Dense optical flow per event window from a coarse grid of flow nodes, fitted to the average-timestamp loss of Zhu et
al. (CVPR'19): a batched, differentiable loss, its candidates pass and a coarse-to-fine fit.

The loss is the dense-flow timestamp loss of flow_timestamp_objective.py (the warp of optic_flow.py:37-44, the
timestamp images of image.py:286-353 and the sum of squares of objectives.py:524-551) at the flow that grid_flow.py
interpolates from the nodes, computed without forming the dense flow: each event's node cell and weights are computed
once per pass, and the backward sums the node gradient of a CTA in shared memory (evk_grid_flow_timestamp_objective_f32
/ _grad_f32, evk_grid_flow_timestamp_candidates_f32).  The fit is grid_flow.py's, started from a global
motion_timestamp_fit_torch and confined to a box.
"""
import collections

import torch

from .. import _lib
from ..representations import _events as E
from ._batched import _chunked_candidates, _chunked_objective, _event_tensors, _timestamp_events
from .grid_flow import _grid_fit, _grid_tensor
from .motion_fit import FIT_WORKSPACE_BYTES
from .motion_timestamp_fit import TIMESTAMP_FIT_MAX_WINDOWS, motion_timestamp_fit_torch
from .motion_timestamp_objective import TIMESTAMP_CANDIDATES_WORKSPACE_BYTES
from .warps import linvel_warp

GridFlowTimestampFit = collections.namedtuple("GridFlowTimestampFit", "flow f loss status iterations")
GridFlowTimestampFit.__doc__ = """grid_flow_timestamp_fit_torch's result: flow (B,2,gh,gw) f64 on the last grid, f (B,) f64
= loss + smoothness R (the fitted objective), loss (B,) f64 (Zhu's loss), status (B,) int8, iterations (B,) int32"""


def grid_flow_timestamp_objective_torch(xs, ys, ts, ps, grid_flow, img_size, t0=None, blur_sigma=2.0,
                                        timestamp_reverse=False, batch_end_indices=None):
    """
    Average-timestamp loss f_b of every sample b of a batch of event windows, warped by a dense flow given on a grid of
    nodes.  grid_flow[b] is (2, gh, gw) with 2 <= gh <= H, 2 <= gw <= W and gh gw <= 4096, (H, W) = img_size, and an
    event takes the flow interpolated from the nodes exactly as in grid_flow_contrast_objective_torch (align_corners,
    the two ratios rounded to f32, the products in f32, a node tap outside the grid contributing 0).  Everything after
    that is flow_timestamp_objective_torch (samples, t0, the warp in f32, the normalised stamps and timestamp_reverse,
    the keep rule 0 <= x' < W, 0 <= y' < H, a NaN f for a sample with a non-finite warped position, a NaN p dropped, the
    per-polarity images T = S / C on the (H+1, W+1) canvas, the blur and f_b = sum(G_+^2) + sum(G_-^2)).  For events
    at integer pixels inside the sensor, f equals
        flow_timestamp_objective_torch(..., F.interpolate(grid_flow, (H, W), mode="bilinear", align_corners=True))
    to f32 rounding, and the gradient equals autograd through that composition; at gh = H, gw = W the grid is the dense
    flow.  Computed without forming the dense flow (evk_grid_flow_timestamp_objective_f32 / _grad_f32).
    @param grid_flow (B,2,gh,gw) or (2,gh,gw); the only differentiable input (expanded views work)
    @param img_size (H, W) of the sensor
    @returns (B,) tensor of f in grid_flow's dtype, on grid_flow's device, 0 <= B <= 32767.  With every input on the GPU
           neither the forward nor the backward synchronises with the host.  The backward is accurate to f32 rounding
           (as the dense-flow loss's).
    """
    xs, ys, ts, ps = _event_tensors(xs, ys, ts, ps, t0, "grid_flow_timestamp_objective_torch", "the node grid")
    H, W = int(img_size[0]), int(img_size[1])
    g = _grid_tensor(grid_flow, H, W)
    B = g.shape[0]
    sigma = _blur_sigma(blur_sigma)
    _lib.lib()
    dev = E.compute_device(g, xs, ys, ts, ps)
    x, y, t_rel, tau, p, offsets = _timestamp_events(xs, ys, ts, ps, t0, batch_end_indices, B, dev, "node grids",
                                                     timestamp_reverse)
    from ..autograd import GridFlowTimestampObjective
    f = GridFlowTimestampObjective.apply(g, x, y, t_rel, tau, p, offsets, (H, W, sigma))
    return f.to(device=g.device, dtype=g.dtype)


def grid_flow_timestamp_candidates_torch(xs, ys, ts, ps, candidates, img_size, t0=None, blur_sigma=2.0,
                                         timestamp_reverse=False, batch_end_indices=None):
    """
    The grid-flow average-timestamp loss of every window b under each of its J candidate node grids candidates[b, j]:
    f[b, j] is the f_b that grid_flow_timestamp_objective_torch returns with grid_flow[b] = candidates[b, j].  Each pass
    over the events scores up to min(32, 12288 // (gh gw)) candidates of every window
    (evk_grid_flow_timestamp_candidates_f32), and the windows run in chunks of at most 32767 // (candidates per pass)
    whose workspace stays under TIMESTAMP_CANDIDATES_WORKSPACE_BYTES; neither split changes a value.
    @param candidates (B,J,2,gh,gw) node grids, any float dtype (rounded to f32), any J >= 1
    @returns (B,J) f64 tensor of values (no autograd graph) on candidates' device
    """
    xs, ys, ts, ps = _event_tensors(xs, ys, ts, ps, t0, "grid_flow_timestamp_candidates_torch", "nothing")
    H, W = int(img_size[0]), int(img_size[1])
    cand = _grid_tensor(candidates, H, W, "candidates", lead=2)
    B, J, _, gh, gw = cand.shape
    sigma = _blur_sigma(blur_sigma)
    _lib.lib()
    dev = E.compute_device(cand, xs, ys, ts, ps)
    ev = _timestamp_events(xs, ys, ts, ps, t0, batch_end_indices, B, dev, "candidate sets", timestamp_reverse)
    with torch.cuda.device(dev):
        c = cand.detach().to(device=dev, dtype=torch.float32).reshape(B, J, 2 * gh * gw)
        f = _candidates(ev, c, (gh, gw), H, W, sigma)
    return f.to(cand.device)


def _blur_sigma(blur_sigma):
    """blur_sigma as a float; NaN is rejected here, before any CUDA call (the entries reject it too)"""
    s = float(blur_sigma)
    if s != s:
        raise ValueError("blur_sigma must be a number, got NaN")
    return s


def _candidates(ev, c, grid, H, W, sigma):
    """f (B,J) f64 of the prepared device events ev (_timestamp_events) under the device candidates c (B,J,2 gh gw) f32"""
    return _chunked_candidates("evk_grid_flow_timestamp_candidates", "grid_flow_timestamp_candidates", ev[:5], ev[5], c,
                               ("grid", grid, H, W), (sigma,), TIMESTAMP_CANDIDATES_WORKSPACE_BYTES, 32767)


def grid_flow_timestamp_fit_torch(xs, ys, ts, ps, img_size, grid_shapes=((3, 4), (6, 8), (12, 16)), smoothness=1e-2,
                                  charbonnier_eps=1.0, batch_end_indices=None, t0=None, blur_sigma=2.0,
                                  timestamp_reverse=False, x0=None, param_ranges=None, bounds=None, num_samples_per_param=5,
                                  grid_levels=1, log_scale=False, param_scale=None, max_iter=50, line_search_steps=8,
                                  ftol=1e-9, gtol=1e-9):
    """
    Fit a node-grid flow to every event window on its own, all windows at once, coarse to fine: minimise
        F_b(g) = f_b(g) + smoothness R(g)
    with f_b the loss of grid_flow_timestamp_objective_torch (same windows, t0, stamps, blur_sigma and img_size, so any
    result can be checked with it) and R charbonnier_smoothness(g, charbonnier_eps).  The stages, the upsampling between
    grids, the BFGS with unit_first_step, param_scale, the statuses, K = 2 gh gw <= 512 and the absence of host
    synchronisation are those of grid_flow_fit_torch; each forward and gradient call takes a chunk of
    max(1, min(B, FIT_WORKSPACE_BYTES // (workspace + images per window), 32767)) windows and each candidates call a
    chunk as grid_flow_timestamp_candidates_torch's.
    Direction: this MINIMISES Zhu's loss, as motion_timestamp_fit_torch does.
    Start point: x0 ((B,2,gh0,gw0) or (2,gh0,gw0) on the first grid of grid_shapes) if given; otherwise a global flow from
    motion_timestamp_fit_torch with linvel_warp() on param_ranges ((2,2) or (B,2,2) ranges of (vx, vy), and that fit's
    num_samples_per_param, grid_levels, log_scale, max_iter, line_search_steps, ftol, gtol and first blur), as u = -vx,
    v = -vy at every node.
    Bounds: an event warped off the canvas adds nothing to f, so a flow that sends every event off the canvas has f = 0,
    the loss's global minimum, and a long step can reach it.  bounds ((2,2) or (B,2,2): [lo, hi] of u and of v) confines
    every node of every line search to a box: a point outside scores +inf and is never taken.  With param_ranges and no
    bounds, the box is the flow range that -param_ranges implies (u in [-hi_vx, -lo_vx], v in [-hi_vy, -lo_vy]) widened
    by one level-0 grid step on each side, and further where the global start lies beyond it.  Bilinear upsampling with
    align_corners keeps every node inside the per-component range of the coarser grid, so a start inside the box stays
    inside it at every stage; a start outside it (x0, or a global start outside bounds) is clamped onto it.  With x0 and no bounds the fit is UNBOUNDED and a window may end on such a degenerate
    minimum: pass bounds.
    smoothness: the default 1e-2 was chosen on the affine-flow windows of tests/test_gpu_grid_flow_timestamp.py (90 x 120
    sensor, 30 k events per window over 0.1 s, 3 x 4 then 6 x 8 nodes, blur 1).  Of 1e-2, 1e-1, 1, 10 and 100 it
    recovered the flows best, to an RMS node error of 0.14-0.54 px over the window (1: 0.51-1.07 px; 10 and above
    flatten the flow), and every value recovered all 8 windows within 1.5 px.  The loss sums squared timestamp images over
    the canvas (about 650 there), so its scale, and the smoothness that balances it, is not the contrast loss's.
    @returns GridFlowTimestampFit(flow (B,2,gh,gw) f64 on the last grid, f (B,) f64 = F at flow for the last blur, loss
             (B,) f64 = f - smoothness R, status (B,) int8 of the last stage, iterations (B,) int32 summed over the
             stages), on the events' device.
    """
    xs, ys, ts, ps = _event_tensors(xs, ys, ts, ps, t0, "grid_flow_timestamp_fit_torch", "nothing")
    H, W = int(img_size[0]), int(img_size[1])
    for s in (blur_sigma if isinstance(blur_sigma, (list, tuple)) else [blur_sigma]):
        _blur_sigma(s)

    def global_fit(sigma):
        return motion_timestamp_fit_torch(xs, ys, ts, ps, linvel_warp(), batch_end_indices, t0, sigma, timestamp_reverse,
                                          (H, W), param_ranges=param_ranges, num_samples_per_param=num_samples_per_param,
                                          grid_levels=grid_levels,
                                          log_scale=log_scale, max_iter=max_iter, line_search_steps=line_search_steps,
                                          ftol=ftol, gtol=gtol).params

    def events(B, dev):
        return _timestamp_events(xs, ys, ts, ps, t0, batch_end_indices, B, dev, "windows", timestamp_reverse)

    def loss(ev, grid, sigma):
        return (_chunked_objective("evk_grid_flow_timestamp_objective", "grid_flow_timestamp_objective", ev[:5], ev[5],
                                   ("grid", grid, H, W), (sigma,), (2, 2), FIT_WORKSPACE_BYTES, TIMESTAMP_FIT_MAX_WINDOWS),
                lambda c: _candidates(ev, c, grid, H, W, sigma))
    return GridFlowTimestampFit(*_grid_fit("grid_flow_timestamp_fit_torch", (xs, ys, ts, ps), (H, W), grid_shapes,
                                           smoothness, charbonnier_eps, batch_end_indices, blur_sigma, x0, param_ranges,
                                           bounds, num_samples_per_param, param_scale, max_iter, line_search_steps, ftol,
                                           gtol, global_fit, events, loss, bound_to_ranges=True))

