"""Dense optical flow per event window from a coarse grid of flow nodes: a batched, differentiable contrast loss, its
candidates pass and a coarse-to-fine fit.

The reference estimates optic flow with contrast maximisation one ROI at a time (grid_cmax, events_cmax.py:28-76: a
scipy fit of a linear velocity per patch).  The usual model-based answer is a flow given on a coarse grid of nodes and
interpolated bilinearly to the pixels (tile-based flow, Shiba et al., ECCV 2022), with a smoothness term: a smooth dense
field with a few hundred unknowns per window.  The loss is the dense-flow contrast loss of flow_objective.py (the warp
of optic_flow.py:37-44 and the image of draw_flow.py:15-26) at the interpolated flow, computed without forming the dense
flow: each event's node cell and weights are computed once per pass, and the backward sums the node gradient of a CTA in
shared memory (evk_cmax_grid_flow_objective_f32 / _grad_f32, evk_cmax_grid_flow_candidates_f32).
"""
import collections

import torch

from .. import _lib
from ..representations import _events as E
from ._batched import MAX_GRID_CANDIDATE_NODES  # noqa: F401  (a public name of this module)
from ._batched import (DEFAULT_PARAM, OBJECTIVES, _batch_events, _check_objective, _chunked_candidates, _chunked_objective,
                       _event_tensors, _float_tensor, _window_count)
from .motion_fit import (FIT_MAX_WINDOWS, FIT_WORKSPACE_BYTES, _batched_bfgs, _check_line_search_steps, _check_per_window,
                         _per_window, motion_contrast_fit_torch)
from .motion_objective import CANDIDATES_WORKSPACE_BYTES
from .warps import linvel_warp

GridFlowFit = collections.namedtuple("GridFlowFit", "flow f contrast status iterations")
GridFlowFit.__doc__ = """grid_flow_fit_torch's result: flow (B,2,gh,gw) f64 on the last grid, f (B,) f64 = contrast +
smoothness R (the fitted objective), contrast (B,) f64, status (B,) int8, iterations (B,) int32"""

MAX_GRID_NODES = 4096             # gh gw of the loss
MAX_FIT_PARAMETERS = 512          # 2 gh gw of a fit: its dense (B,K,K) inverse Hessians take 2 MB per window


def _grid_tensor(grid_flow, H, W, name="grid_flow", lead=1):
    """grid_flow as a (B,2,gh,gw) (lead 1) or (B,J,2,gh,gw) (lead 2) float tensor, checked against the node limits"""
    g = _float_tensor(grid_flow, name)
    if lead == 1 and g.dim() == 3:
        g = g.unsqueeze(0)
    if g.dim() != 3 + lead or g.shape[lead] != 2 or (lead == 2 and g.shape[1] < 1):
        raise ValueError("%s must have shape %s, got %s" % (name, "(B,2,gh,gw) or (2,gh,gw)" if lead == 1 else
                                                            "(B,J,2,gh,gw) with J >= 1", tuple(g.shape)))
    gh, gw = g.shape[-2:]
    _check_grid_shape(gh, gw, H, W, MAX_GRID_NODES)
    return g


def _check_grid_shape(gh, gw, H, W, max_nodes):
    if not (2 <= gh <= H and 2 <= gw <= W) or gh * gw > max_nodes:
        raise ValueError("a node grid must have 2 <= gh <= H = %d, 2 <= gw <= W = %d and gh * gw <= %d, got %d x %d"
                         % (H, W, max_nodes, gh, gw))


def _scalars(objective, blur_sigma, obj_param):
    return float(blur_sigma), OBJECTIVES[objective], float(obj_param if obj_param is not None else
                                                           DEFAULT_PARAM.get(objective, 0.0))


def grid_flow_contrast_objective_torch(xs, ys, ts, ps, grid_flow, img_size, t0=None, objective="variance", blur_sigma=1.0,
                                       obj_param=None, batch_end_indices=None):
    """
    Contrast objective f_b of every sample b of a batch of event windows, warped by a dense flow given on a grid of nodes.
    grid_flow[b] is (2, gh, gw) with 2 <= gh <= H, 2 <= gw <= W and gh gw <= 4096, (H, W) = img_size.  Node (i, j) sits at
    pixel (j (W-1)/(gw-1), i (H-1)/(gh-1)) (align_corners), and an event at (x, y) takes the flow (u, v) interpolated
    bilinearly from the nodes at (x (gw-1)/(W-1), y (gh-1)/(H-1)) (the two ratios rounded to f32, the products in f32); a
    node tap outside the grid contributes 0, as with zero padding.  Everything after that is flow_contrast_objective_torch
    (samples, t0, the warp x' = x + u (t - t0_b), y' = y + v (t - t0_b) in f32, the keep rule 0 <= x' < W, 0 <= y' < H,
    the (H+1, W+1) canvas, the blur, the objectives variance / sos / soe / sosa, and a NaN f for a sample with a non-finite
    warped position).  For events at integer pixels inside the sensor, f equals
        flow_contrast_objective_torch(..., F.interpolate(grid_flow, (H, W), mode="bilinear", align_corners=True))
    to f32 rounding, and the gradient equals autograd through that composition; at gh = H, gw = W the grid is the dense
    flow.  Computed without forming the dense flow (evk_cmax_grid_flow_objective_f32 / _grad_f32).
    @param grid_flow (B,2,gh,gw) or (2,gh,gw); the only differentiable input (expanded views work)
    @param img_size (H, W) of the sensor
    @returns (B,) tensor of f in grid_flow's dtype, on grid_flow's device.  With every input on the GPU neither the
           forward nor the backward synchronises with the host.  The backward is accurate to f32 rounding (as the dense
           flow loss's).
    """
    _check_objective(objective, "flow")
    xs, ys, ts, ps = _event_tensors(xs, ys, ts, ps, t0, "grid_flow_contrast_objective_torch", "the node grid")
    H, W = int(img_size[0]), int(img_size[1])
    g = _grid_tensor(grid_flow, H, W)
    B = g.shape[0]
    _lib.lib()
    dev = E.compute_device(g, xs, ys, ts, ps)
    x, y, t_rel, p, offsets = _batch_events(xs, ys, ts, ps, t0, batch_end_indices, B, dev, "node grids")
    from ..autograd import GridFlowObjective
    sigma, obj, param = _scalars(objective, blur_sigma, obj_param)
    f = GridFlowObjective.apply(g, x, y, t_rel, p, offsets, (H, W, obj, sigma, param))
    return f.to(device=g.device, dtype=g.dtype)


def grid_flow_contrast_candidates_torch(xs, ys, ts, ps, candidates, img_size, t0=None, objective="variance", blur_sigma=1.0,
                                        obj_param=None, batch_end_indices=None):
    """
    The grid-flow contrast objective of every window b under each of its J candidate node grids candidates[b, j]: f[b, j]
    is the f_b that grid_flow_contrast_objective_torch returns with grid_flow[b] = candidates[b, j].  Each pass over the
    events scores up to min(32, 12288 // (gh gw)) candidates of every window (evk_cmax_grid_flow_candidates_f32), and the
    windows run in chunks whose workspace stays under CANDIDATES_WORKSPACE_BYTES; neither split changes a value.
    @param candidates (B,J,2,gh,gw) node grids, any float dtype (rounded to f32), any J >= 1
    @returns (B,J) f64 tensor of values (no autograd graph) on candidates' device
    """
    _check_objective(objective, "flow")
    xs, ys, ts, ps = _event_tensors(xs, ys, ts, ps, t0, "grid_flow_contrast_candidates_torch", "nothing")
    H, W = int(img_size[0]), int(img_size[1])
    cand = _grid_tensor(candidates, H, W, "candidates", lead=2)
    B, J, _, gh, gw = cand.shape
    _lib.lib()
    dev = E.compute_device(cand, xs, ys, ts, ps)
    x, y, t_rel, p, offsets = _batch_events(xs, ys, ts, ps, t0, batch_end_indices, B, dev, "candidate sets")
    with torch.cuda.device(dev):
        c = cand.detach().to(device=dev, dtype=torch.float32).reshape(B, J, 2 * gh * gw)
        f = _candidates(x, y, t_rel, p, offsets, c, (gh, gw), H, W, _scalars(objective, blur_sigma, obj_param))
    return f.to(cand.device)


def _candidates(x, y, t_rel, p, offsets, c, grid, H, W, scalars):
    """f (B,J) f64 of the prepared device events under the device candidates c (B,J,2 gh gw) f32"""
    return _chunked_candidates("evk_cmax_grid_flow_candidates", "grid_flow_candidates", (x, y, t_rel, p), offsets, c,
                               ("grid", grid, H, W), scalars, CANDIDATES_WORKSPACE_BYTES, 65535)


def charbonnier_smoothness(grid_flow, eps):
    """
    R of every window and its gradient: with rho(d) = sqrt(d^2 + eps^2) - eps (the Charbonnier penalty, 0 at d = 0),
        R = sum_c [ sum_{i, j < gw-1} rho(g[c,i,j+1] - g[c,i,j]) + sum_{i < gh-1, j} rho(g[c,i+1,j] - g[c,i,j]) ]
    over both flow components c (every channel c of any (..., C, gh, gw) grid), every horizontally and every vertically
    neighbouring pair of nodes.
    @param grid_flow (..., 2, gh, gw) float tensor
    @returns (R (...), dR/dgrid_flow (..., 2, gh, gw)) in grid_flow's dtype
    """
    e2 = float(eps) ** 2
    dh = grid_flow[..., :, 1:] - grid_flow[..., :, :-1]
    dv = grid_flow[..., 1:, :] - grid_flow[..., :-1, :]
    sh, sv = torch.sqrt(dh * dh + e2), torch.sqrt(dv * dv + e2)
    R = (sh - float(eps)).sum((-3, -2, -1)) + (sv - float(eps)).sum((-3, -2, -1))
    gh_, gv_ = dh / sh, dv / sv
    g = torch.zeros_like(grid_flow)
    g[..., :, 1:] += gh_
    g[..., :, :-1] -= gh_
    g[..., 1:, :] += gv_
    g[..., :-1, :] -= gv_
    return R, g


def grid_flow_fit_torch(xs, ys, ts, ps, img_size, grid_shapes=((3, 4), (6, 8), (12, 16)), smoothness=1e-3,
                        charbonnier_eps=1.0, batch_end_indices=None, t0=None, objective="variance", blur_sigma=1.0,
                        obj_param=None, x0=None, param_ranges=None, num_samples_per_param=5, grid_levels=1,
                        log_scale=False, param_scale=None, max_iter=50, line_search_steps=8, ftol=1e-9, gtol=1e-9):
    """
    Fit a node-grid flow to every event window on its own, all windows at once, coarse to fine: minimise
        F_b(g) = f_b(g) + smoothness R(g)
    with f_b the contrast objective of grid_flow_contrast_objective_torch (same windows, t0, objective, blur_sigma,
    obj_param and img_size, so any result can be checked with it) and R charbonnier_smoothness(g, charbonnier_eps).
    R is not normalised by the grid size: on a grid twice as fine a smooth flow has half the neighbour differences and
    four times the pairs.
    Start point: x0 ((B,2,gh0,gw0) or (2,gh0,gw0) on the first grid of grid_shapes) if given; otherwise a global flow from
    motion_contrast_fit_torch with linvel_warp() on param_ranges ((2,2) or (B,2,2) ranges of (vx, vy), and that fit's
    num_samples_per_param, grid_levels, log_scale, max_iter, line_search_steps, ftol, gtol, first blur), as u = -vx,
    v = -vy at every node.
    Stages: for each (gh, gw) of grid_shapes, the previous result is upsampled to the new grid (bilinear,
    align_corners=True, in f64), then, for each blur of blur_sigma (a number or a sequence), motion_contrast_fit_torch's
    BFGS runs on F with the same line search, step rule and status codes, over the K = 2 gh gw node values (K <= 512:
    the inverse Hessians are dense (B,K,K) f64).  Its line searches score all step lengths in one candidates pass
    (grid_flow_contrast_candidates_torch) plus R.  The inverse Hessian starts as diag(param_scale^2) / |g param_scale|,
    so the first step is one unit of param_scale long; param_scale (a number) defaults to the linvel grid's level-0
    spacing, max over (vx, vy) of (hi - lo) / (num_samples_per_param - 1), or 1 with x0.
    Every stage runs exactly max_iter iterations on all windows, so with the events, the window ends and x0 (or
    param_ranges) on the GPU the fit never synchronises with the host.  Each forward and gradient call takes a chunk of
    max(1, min(B, FIT_WORKSPACE_BYTES // (workspace + image per window), 65535)) windows and each candidates call a chunk
    as grid_flow_contrast_candidates_torch's.
    @returns GridFlowFit(flow (B,2,gh,gw) f64 on the last grid, f (B,) f64 = F at flow for the last blur, contrast (B,)
             f64 = f - smoothness R, status (B,) int8 of the last stage, iterations (B,) int32 summed over the stages),
             on the events' device.  Larger grids need a limited-memory method and are rejected.
    """
    _check_objective(objective, "flow")
    xs, ys, ts, ps = _event_tensors(xs, ys, ts, ps, t0, "grid_flow_fit_torch", "nothing")
    H, W = int(img_size[0]), int(img_size[1])

    def global_fit(sigma):
        return motion_contrast_fit_torch(xs, ys, ts, ps, linvel_warp(), batch_end_indices, t0, objective, sigma, obj_param,
                                         (H, W), param_ranges=param_ranges, num_samples_per_param=num_samples_per_param,
                                         grid_levels=grid_levels, log_scale=log_scale, max_iter=max_iter,
                                         line_search_steps=line_search_steps, ftol=ftol, gtol=gtol).params

    def events(B, dev):
        return _batch_events(xs, ys, ts, ps, t0, batch_end_indices, B, dev, "windows")

    def loss(ev, grid, sigma):
        x, y, t_rel, p, offsets = ev
        scalars = _scalars(objective, sigma, obj_param)
        return (_chunked_objective("evk_cmax_grid_flow_objective", "grid_flow_objective", ev[:4], offsets, ("grid", grid, H, W),
                                   scalars, (1,), FIT_WORKSPACE_BYTES, FIT_MAX_WINDOWS),
                lambda c: _candidates(x, y, t_rel, p, offsets, c, grid, H, W, scalars))
    return GridFlowFit(*_grid_fit("grid_flow_fit_torch", (xs, ys, ts, ps), (H, W), grid_shapes, smoothness, charbonnier_eps,
                                  batch_end_indices, blur_sigma, x0, param_ranges, None, num_samples_per_param, param_scale,
                                  max_iter, line_search_steps, ftol, gtol, global_fit, events, loss))


def _grid_fit(who, tensors, size, grid_shapes, smoothness, charbonnier_eps, batch_end_indices, blur_sigma, x0, param_ranges,
              bounds, num_samples_per_param, param_scale, max_iter, line_search_steps, ftol, gtol, global_fit, events, loss,
              bound_to_ranges=False):
    """The coarse-to-fine fit of F = f + smoothness R that grid_flow_fit_torch and grid_flow_timestamp_fit_torch share:
    the argument checks (before any CUDA call), the start, and the BFGS stages per grid shape and blur.
    tensors: the inputs that choose the device;  global_fit(sigma) -> (B,2) linvel params (vx, vy) of the global fit at
    the first blur, the start without x0;  events(B, dev) -> the prepared device events;  loss(events, (gh, gw), sigma)
    -> (fg of f, candidates of f on f32 node grids).  bounds ((2,2) or (B,2,2)): [lo, hi] of u and of v at every node;
    without it, bound_to_ranges confines a fit started from the global fit to the flow range -param_ranges implies,
    widened by one level-0 grid step and stretched to contain the start.  Returns (flow, F, f, status, iterations)."""
    H, W = size
    shapes = [(int(a), int(b)) for a, b in grid_shapes]
    if not shapes:
        raise ValueError("grid_shapes must name at least one (gh, gw)")
    for gh, gw in shapes:
        _check_grid_shape(gh, gw, H, W, MAX_GRID_NODES)
        if 2 * gh * gw > MAX_FIT_PARAMETERS:
            raise ValueError("%s keeps a dense inverse Hessian of K = 2 gh gw <= %d parameters per window; "
                             "a %d x %d grid has K = %d" % (who, MAX_FIT_PARAMETERS, gh, gw, 2 * gh * gw))
    sigmas = [float(s) for s in (blur_sigma if isinstance(blur_sigma, (list, tuple)) else [blur_sigma])]
    if not sigmas:
        raise ValueError("blur_sigma must be a number or a non-empty sequence")
    _check_line_search_steps(line_search_steps)
    if x0 is None and param_ranges is None:
        raise ValueError("%s needs x0 or param_ranges" % who)
    if float(smoothness) < 0 or not float(charbonnier_eps) > 0:
        raise ValueError("smoothness must be >= 0 and charbonnier_eps > 0")
    B = _window_count(batch_end_indices)
    gh0, gw0 = shapes[0]
    if x0 is not None:
        got = tuple(x0.shape) if isinstance(x0, torch.Tensor) else tuple(torch.as_tensor(x0).shape)
        if got not in ((2, gh0, gw0), (B, 2, gh0, gw0)):
            raise ValueError("x0 must have shape %s or %s, got %s" % ((2, gh0, gw0), (B, 2, gh0, gw0), got))
    if bounds is not None:
        _check_per_window(bounds, B, (2, 2), "bounds")
    lam, eps = float(smoothness), float(charbonnier_eps)
    _lib.lib()
    dev = E.compute_device(*(a for a in (x0, param_ranges, bounds) + tuple(tensors) if isinstance(a, torch.Tensor)))
    box = None
    if x0 is None:
        params = global_fit(sigmas[0])
        with torch.cuda.device(dev):
            flow = (-params).view(B, 2, 1, 1).expand(B, 2, gh0, gw0).contiguous()
            r = _per_window(param_ranges, B, (2, 2), "param_ranges", dev)
            step = (r[..., 1] - r[..., 0]) / (num_samples_per_param - 1)
            if param_scale is None:
                param_scale = step.amax(1)
            if bounds is None and bound_to_ranges:
                # u = -vx, v = -vy: the ranges' edges swap; one grid step beyond them, and the start inside
                box = torch.stack((torch.minimum(-r[..., 1] - step, -params), torch.maximum(-r[..., 0] + step, -params)), -1)
    else:
        flow = _per_window(x0, B, (2, gh0, gw0), "x0", dev)
    if bounds is not None:
        box = _per_window(bounds, B, (2, 2), "bounds", dev)
    ev = events(B, dev)
    with torch.cuda.device(dev):
        scale = torch.as_tensor(1.0 if param_scale is None else param_scale, dtype=torch.float64, device=dev)
        return _stages(flow, shapes, sigmas, box, scale, ev, loss, lam, eps, max_iter, line_search_steps, ftol, gtol)


def _stages(grid, shapes, sigmas, box, scale, ev, loss, lam, eps, max_iter, line_search_steps, ftol, gtol):
    """The BFGS stages of the coarse-to-fine node-grid fits (grid flow, depth grid): grid (B,C,gh0,gw0) f64 is the start
    on the first of the (gh, gw) shapes, with C channels per node; box None or (B,C,2) [lo, hi] of every node of
    channel c; scale a number or (B,) tensor, the BFGS param_scale of every node; loss(ev, (gh, gw), sigma) -> (fg of f,
    candidates of f on f32 node grids).  Returns (grid, F, f, status, iterations) on the last shape."""
    B, C = grid.shape[:2]
    iters = torch.zeros(B, dtype=torch.int32, device=grid.device)
    status = f = None
    for gh, gw in shapes:
        if tuple(grid.shape[2:]) != (gh, gw):
            grid = torch.nn.functional.interpolate(grid, (gh, gw), mode="bilinear", align_corners=True)
        K = C * gh * gw
        sc = scale.reshape(-1, 1).expand(B, K)
        lim = None
        if box is not None:
            # every node of channel c in [lo_c, hi_c]: the clamp moves a start outside the box onto it, and undoes the
            # rounding of the upsampling
            lim = box.unsqueeze(2).expand(B, C, gh * gw, 2).reshape(B, K, 2)
            grid = torch.minimum(torch.maximum(grid, box[..., 0, None, None]), box[..., 1, None, None])
        xk = grid.reshape(B, K)
        for sigma in sigmas:
            fg, candidates = _stage(*loss(ev, (gh, gw), sigma), (C, gh, gw), lam, eps)
            xk, f, status, it = _batched_bfgs(fg, candidates, xk, sc, max_iter, line_search_steps, ftol, gtol, lim,
                                              unit_first_step=True)
            iters += it
        grid = xk.reshape(B, C, gh, gw)
    rest = f - lam * charbonnier_smoothness(grid, eps)[0]
    return grid, f, rest, status, iters


def _stage(obj, cand, grid, lam, eps):
    """fg and candidates of F = f + lam R on the grid (C, gh, gw) of C channels, for _batched_bfgs: obj (B,K) nodes ->
    (f, g) of the loss, cand (B,J,K) f32 node grids -> (B,J) f"""
    C, gh, gw = grid

    def fg(xk):
        f, g = obj(xk)
        R, gR = charbonnier_smoothness(xk.view(-1, C, gh, gw), eps)
        return f + lam * R, g + lam * gR.reshape(g.shape)

    def candidates(pts):
        B, J, K = pts.shape
        f = cand(pts.to(torch.float32))
        R = charbonnier_smoothness(pts.reshape(B, J, C, gh, gw), eps)[0]
        return f + lam * R

    return fg, candidates
