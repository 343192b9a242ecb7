"""Camera motion and depth together: the depth-grid contrast loss of depth_grid.py made differentiable in the camera
motion as well as in the inverse-depth nodes, its joint candidates pass, and a coarse-to-fine fit of both per window.

With an event camera and nothing else neither the motion nor the depth is known, and the monocular use of contrast
maximisation fits both (Gallego, Rebecq, Scaramuzza, CVPR 2018; the joint ego-motion and depth of Shiba et al., TPAMI
2024).  The loss's f is depth_grid_contrast_objective_torch's bit for bit (evk_cmax_depth_grid_objective_f32); its
backward is one event pass that contracts df/dx', df/dy' with both dx'/drho (into the nodes) and the camera motion's
Jacobian rows at each event's rho (into (w, v): evk_cmax_depth_grid_joint_grad_f32); the candidates pass scores
(motion, grid) pairs (evk_cmax_depth_grid_joint_candidates_f32), so one line search moves both.  Depth and translation
share one scale, which the fit holds fixed at |v| = |x0[3:]|: it moves w, the direction of v and the nodes.
"""
import collections

import numpy as np
import torch

from .. import _lib
from ..representations import _events as E
from ._batched import (MAX_CANDIDATES, MAX_GRID_CANDIDATE_NODES, _batch_events, _centre, _check_objective,
                       _event_tensors, _float_tensor, _pointers, _rows, _window_count, fit_window_chunk)
from .depth_grid import _candidates as _depth_grid_candidates
from .depth_grid import _check_warp, _constant_start, _depth_grid_tensor, _model
from .grid_flow import MAX_FIT_PARAMETERS, MAX_GRID_NODES, _check_grid_shape, _scalars, charbonnier_smoothness
from .motion_fit import (FIT_MAX_WINDOWS, FIT_WORKSPACE_BYTES, _batched_bfgs, _check_line_search_steps, _check_per_window,
                         _per_window)
from .motion_objective import CANDIDATES_WORKSPACE_BYTES

MotionAndDepthFit = collections.namedtuple("MotionAndDepthFit", "motion inv_depth f contrast status iterations")
MotionAndDepthFit.__doc__ = """motion_and_depth_fit_torch's result: motion (B,6) f64 (wx, wy, wz, vx, vy, vz),
inv_depth (B,gh,gw) f64 on the last grid, f (B,) f64 = contrast + smoothness R (the fitted objective), contrast (B,)
f64, status (B,) int8 of the last stage, iterations (B,) int32 summed over the stages"""

MOTION_PARAMETERS = 5    # w and the two chart coordinates of the direction of v, in front of the nodes
CHART_BOX = 1.0          # |a|, |b| of the direction chart: at most 54.7 degrees from the chart's centre


def _motion_tensor(motion, B, lead, name):
    """motion as a float tensor of shape (B,6) (lead 1; (6,) is every window's) or (B,J,6) (lead 2)"""
    m = _float_tensor(motion, name)
    if lead == 1 and tuple(m.shape) == (6,):
        m = m.unsqueeze(0).expand(B, 6)
    want = (B, 6) if lead == 1 else (B, m.shape[1] if m.dim() == 3 else -1, 6)
    if tuple(m.shape) != want or (lead == 2 and m.shape[1] < 1):
        raise ValueError("%s must have shape %s, got %s" % (name, "(B,6) or (6,) with B = %d" % B if lead == 1 else
                                                            "(B,J,6) with B = %d, J >= 1" % B, tuple(m.shape)))
    return m


def motion_and_depth_contrast_objective_torch(xs, ys, ts, ps, inv_depth_grid, motion, warpfunc, img_size, t0=None,
                                              objective="variance", blur_sigma=1.0, obj_param=None, batch_end_indices=None):
    """
    The contrast objective f_b of depth_grid_contrast_objective_torch (same arguments, keep rules, objectives and value,
    bit for bit), differentiable in the camera motion as well as in the inverse-depth nodes.
    @param inv_depth_grid (B,gh,gw) or (gh,gw) inverse-depth nodes
    @param motion (B,6) or (6,) camera motions (wx, wy, wz, vx, vy, vz) in camera_motion_warp's units; differentiable
           (the focal lengths and the principal point of warpfunc are constants)
    @returns (B,) tensor of f in inv_depth_grid's dtype, on its device.  With every input on the GPU neither the forward
           nor the backward synchronises with the host.  The backward is one pass over the events: the node gradient of
           depth_grid_contrast_objective_torch and the motion gradient, accurate to f32 rounding.
    """
    who = "motion_and_depth_contrast_objective_torch"
    _check_warp(warpfunc, who)
    _check_objective(objective, "inverse depth and the motion")
    xs, ys, ts, ps = _event_tensors(xs, ys, ts, ps, t0, who, "the inverse-depth grid and the motion")
    H, W = int(img_size[0]), int(img_size[1])
    g = _depth_grid_tensor(inv_depth_grid, H, W)
    B = g.shape[0]
    m = _motion_tensor(motion, B, 1, "motion")
    _lib.lib()
    dev = E.compute_device(g, xs, ys, ts, ps)
    x, y, t_rel, p, offsets = _batch_events(xs, ys, ts, ps, t0, batch_end_indices, B, dev, "inverse-depth grids")
    from ..autograd import MotionAndDepthObjective
    f = MotionAndDepthObjective.apply(g, m, x, y, t_rel, p, offsets,
                                      (_centre(_lib.WARP_CAMERA_MOTION, warpfunc), H, W) +
                                      _scalars(objective, blur_sigma, obj_param))
    return f.to(device=g.device, dtype=g.dtype)


def motion_and_depth_contrast_candidates_torch(xs, ys, ts, ps, motion_candidates, grid_candidates, warpfunc, img_size,
                                               t0=None, objective="variance", blur_sigma=1.0, obj_param=None,
                                               batch_end_indices=None):
    """
    The contrast objective of every window b under each of its J (motion, inverse-depth grid) pairs: f[b, j] is the f_b
    that depth_grid_contrast_objective_torch returns with motion[b] = motion_candidates[b, j] and inv_depth_grid[b] =
    grid_candidates[b, j].  Each pass over the events scores up to min(32, 12288 // (gh gw)) pairs of every window
    (evk_cmax_depth_grid_joint_candidates_f32), and the windows run in chunks whose workspace stays under
    CANDIDATES_WORKSPACE_BYTES; neither split changes a value.
    @param motion_candidates (B,J,6) camera motions, any float dtype (the entry reads them as f64 and rounds to f32)
    @param grid_candidates (B,J,gh,gw) inverse-depth grids, any float dtype (rounded to f32), any J >= 1
    @returns (B,J) f64 tensor of values (no autograd graph) on grid_candidates' device
    """
    who = "motion_and_depth_contrast_candidates_torch"
    _check_warp(warpfunc, who)
    _check_objective(objective, "inverse depth and the motion")
    xs, ys, ts, ps = _event_tensors(xs, ys, ts, ps, t0, who, "nothing")
    H, W = int(img_size[0]), int(img_size[1])
    cand = _depth_grid_tensor(grid_candidates, H, W, "grid_candidates", lead=2)
    B, J, gh, gw = cand.shape
    mc = _motion_tensor(motion_candidates, B, 2, "motion_candidates")
    if mc.shape[1] != J:
        raise ValueError("motion_candidates has %d candidates per window and grid_candidates %d" % (mc.shape[1], J))
    _lib.lib()
    dev = E.compute_device(cand, mc, xs, ys, ts, ps)
    ev = _batch_events(xs, ys, ts, ps, t0, batch_end_indices, B, dev, "candidate sets")
    with torch.cuda.device(dev):
        c = cand.detach().to(device=dev, dtype=torch.float32).reshape(B, J, gh * gw)
        m = E.to_device(mc.detach(), dev).to(torch.float64)
        f = _joint_candidates(ev, m, c, (gh, gw), H, W, _centre(_lib.WARP_CAMERA_MOTION, warpfunc),
                              _scalars(objective, blur_sigma, obj_param))
    return f.to(cand.device)


def _joint_candidates(ev, motion, c, grid, H, W, centre, scalars):
    """f (B,J) f64 of the prepared device events under the device pairs motion (B,J,6) f64, c (B,J,gh gw) f32, in
    passes of at most min(MAX_CANDIDATES, MAX_GRID_CANDIDATE_NODES // (gh gw)) pairs over chunks of windows whose
    workspace fits CANDIDATES_WORKSPACE_BYTES (the windows and the pairs are independent: no split changes a value)"""
    L = _lib.lib()
    B, J, G = c.shape
    gh, gw = grid
    dev = c.device
    f = torch.empty((B, J), dtype=torch.float64, device=dev)
    if B == 0:
        return f
    jc = max(1, min(J, MAX_CANDIDATES, MAX_GRID_CANDIDATE_NODES // G))
    query = L.evk_cmax_depth_grid_joint_candidates_workspace_bytes
    wb = fit_window_chunk(B, query(1, jc, gh, gw, H, W), CANDIDATES_WORKSPACE_BYTES, 65535 // jc)
    ws = _lib.scratch("depth_grid_candidates", query(wb, jc, gh, gw, H, W), dev)
    x, y, t_rel, p, offsets = ev
    front = _pointers((x, y, t_rel, p))
    for b0 in range(0, B, wb):
        b1 = min(B, b0 + wb)
        for j0 in range(0, J, jc):
            j1 = min(J, j0 + jc)
            rows = _rows(motion[b0:b1, j0:j1], centre).contiguous()
            cc = c[b0:b1, j0:j1].contiguous()
            out = torch.empty((b1 - b0, j1 - j0), dtype=torch.float64, device=dev)
            _lib.check(L.evk_cmax_depth_grid_joint_candidates_f32(
                *front, _lib.ptr(offsets[b0:]), b1 - b0, x.shape[0], _lib.ptr(rows), centre[0], centre[1], _lib.ptr(cc),
                j1 - j0, gh, gw, H, W, *scalars, _lib.ptr(out), _lib.ptr(ws), ws.numel(), _lib.stream()))
            f[b0:b1, j0:j1] = out
    return f


def _joint_objective(ev, grid, H, W, centre, scalars):
    """fg: (motion (B,6) f64, nodes (B,gh gw) f64) -> (f (B,) f64, g_motion (B,6) f64, g_nodes (B,gh gw) f64) through
    evk_cmax_depth_grid_objective_f32 and evk_cmax_depth_grid_joint_grad_f32 (grad_f = 1), in chunks of at most
    FIT_MAX_WINDOWS windows whose workspace and images fit FIT_WORKSPACE_BYTES"""
    L = _lib.lib()
    gh, gw = grid
    x, y, t_rel, p, offsets = ev
    dev = x.device
    front = _pointers((x, y, t_rel, p))
    query = L.evk_cmax_depth_grid_joint_grad_workspace_bytes

    def fg(motion, nodes):
        B = nodes.shape[0]
        rows = _rows(motion, centre).contiguous()
        d = nodes.to(torch.float32).contiguous()
        f = torch.empty(B, dtype=torch.float64, device=dev)
        gm = torch.empty((B, 6), dtype=torch.float64, device=dev)
        gd = torch.empty((B, gh * gw), dtype=torch.float32, device=dev)
        wb = fit_window_chunk(B, query(1, gh, gw, H, W) + 4 * (H + 1) * (W + 1), FIT_WORKSPACE_BYTES, FIT_MAX_WINDOWS)
        iwe = torch.empty((wb, H + 1, W + 1), dtype=torch.float32, device=dev)
        ones = torch.ones(wb, dtype=torch.float32, device=dev)
        ws = _lib.scratch("depth_grid_objective", query(wb, gh, gw, H, W), dev)
        for b0 in range(0, B, wb):
            b1 = min(B, b0 + wb)
            lead = front + (_lib.ptr(offsets[b0:]), b1 - b0, x.shape[0], _lib.ptr(rows[b0:]), centre[0], centre[1],
                            _lib.ptr(d[b0:]), gh, gw, H, W, *scalars)
            _lib.check(L.evk_cmax_depth_grid_objective_f32(*lead, _lib.ptr(f[b0:]), _lib.ptr(iwe), _lib.ptr(ws), ws.numel(),
                                                           _lib.stream()))
            _lib.check(L.evk_cmax_depth_grid_joint_grad_f32(*lead, _lib.ptr(iwe), _lib.ptr(ones), _lib.ptr(gd[b0:]),
                                                            _lib.ptr(gm[b0:]), _lib.ptr(ws), ws.numel(), _lib.stream()))
        return f, gm, gd.to(torch.float64)
    return fg


# ---- the direction chart of the fit ------------------------------------------------------------------------------
def _chart_frame(v):
    """(B,3) velocities -> the chart around their directions: (vhat, e1, e2, speed), with e1, e2 an orthonormal basis
    of the plane normal to vhat (built from the coordinate axis least aligned with vhat), all device tensor ops"""
    speed = v.norm(dim=1, keepdim=True)
    vh = v / speed
    axis = (torch.arange(3, device=v.device) == vh.abs().argmin(1, keepdim=True)).to(v.dtype)
    e1 = torch.linalg.cross(vh, axis)
    e1 = e1 / e1.norm(dim=1, keepdim=True)
    e2 = torch.linalg.cross(vh, e1)
    return vh, e1, e2, speed


def _chart_velocity(ab, frame):
    """the gnomonic chart v = speed normalise(vhat + a e1 + b e2) of the (B,2) coordinates ab"""
    vh, e1, e2, speed = frame
    u = vh + ab[:, :1] * e1 + ab[:, 1:] * e2
    return speed * u / u.norm(dim=1, keepdim=True)


def _chart_gradient(ab, frame, gv):
    """(B,2) dF/d(a, b) from dF/dv (B,3): dv/da = speed (e1 - (u.e1) u / |u|^2) / |u|, likewise for b"""
    vh, e1, e2, speed = frame
    u = vh + ab[:, :1] * e1 + ab[:, 1:] * e2
    n2 = (u * u).sum(1, keepdim=True)
    n = n2.sqrt()
    gu = speed / n * (gv - (gv * u).sum(1, keepdim=True) * u / n2)     # dF/du
    return torch.cat(((gu * e1).sum(1, keepdim=True), (gu * e2).sum(1, keepdim=True)), dim=1)


def motion_and_depth_fit_torch(xs, ys, ts, ps, warpfunc, img_size, x0, inv_depth_range,
                               grid_shapes=((3, 4), (6, 8), (12, 16)), smoothness=1e-2, charbonnier_eps=0.05,
                               rotation_scale=0.05, direction_scale=0.05, batch_end_indices=None, t0=None,
                               objective="variance", blur_sigma=1.0, obj_param=None, inv_depth0=None, num_samples=15,
                               grid_levels=2, max_iter=50, line_search_steps=8, ftol=1e-9, gtol=1e-9):
    """
    Fit the camera motion and an inverse-depth grid to every event window on its own, all windows at once, coarse to
    fine: minimise
        F_b(w, v, D) = f_b(w, v, D) + smoothness R(D)
    with f_b the loss of motion_and_depth_contrast_objective_torch (so any result can be checked with it or with
    depth_grid_contrast_objective_torch) and R charbonnier_smoothness(D, charbonnier_eps), as depth_grid_fit_torch.
    Depth and translation share one scale, so the fit keeps |v_b| = |x0_b[3:]| and moves w, the direction of v and the
    nodes D: pass the speed from odometry for metric depth, or speed 1 for depth up to scale.
    x0 ((6,) or (B,6), required; a zero speed is an error): the start motion, such as an IMU's rates and velocity, or an
    embedded camera_rotation_warp fit with a guessed heading.
    The direction of v is v = |v| normalise(vhat + a e1 + b e2), a gnomonic chart around the direction vhat at the start
    of every BFGS run (e1, e2 orthonormal, normal to vhat), with |a|, |b| <= CHART_BOX, so every fit runs over the
    K = 3 + 2 + gh gw unknowns (w, a, b, D) (K <= 512: the inverse Hessians are dense), the nodes boxed to
    inv_depth_range ((2,) or (B,2): [lo, hi] with 0 <= lo < hi) as in depth_grid_fit_torch.
    Start: the nodes are inv_depth0 ((gh0,gw0) or (B,gh0,gw0) on the first grid) if given, otherwise the best constant
    inverse depth at x0's motion from depth_grid_fit_torch's grid search (num_samples, grid_levels).
    Stages: for each (gh, gw) of grid_shapes the previous nodes are upsampled (bilinear, align_corners=True, f64) and
    clamped to the box, the motion carried forward; for each blur of blur_sigma (a number or a sequence)
    motion_contrast_fit_torch's BFGS runs on F, its scales rotation_scale for w, direction_scale for (a, b) and the grid
    spacing (hi - lo) / (num_samples - 1) for the nodes, its first step one unit of those scales long, its gradient one
    joint backward and its line searches one joint candidates pass each.
    Every stage runs exactly max_iter iterations on all windows, so with the events, window ends, x0 and inv_depth_range
    on the GPU the fit never synchronises with the host.  The defaults of the scales were chosen on the scenes of the
    tests (rho 0.2-1 per m, |v| about 1 m/s): see DESIGN.md section 6.
    @returns MotionAndDepthFit(motion (B,6) f64, inv_depth (B,gh,gw) f64 on the last grid, f (B,) f64 = F for the last
             blur, contrast (B,) f64 = f - smoothness R, status (B,) int8 of the last stage, iterations (B,) int32 summed
             over the stages), on the events' device.  A window whose speed is zero on the GPU (not checked there) ends
             with a non-finite start status.
    """
    who = "motion_and_depth_fit_torch"
    _check_warp(warpfunc, who)
    _check_objective(objective, "inverse depth and the motion")
    xs, ys, ts, ps = _event_tensors(xs, ys, ts, ps, t0, who, "nothing")
    H, W = int(img_size[0]), int(img_size[1])
    shapes = [(int(a), int(b)) for a, b in grid_shapes]
    if not shapes:
        raise ValueError("grid_shapes must name at least one (gh, gw)")
    for gh, gw in shapes:
        _check_grid_shape(gh, gw, H, W, MAX_GRID_NODES)
        if MOTION_PARAMETERS + gh * gw > MAX_FIT_PARAMETERS:
            raise ValueError("%s keeps a dense inverse Hessian of K = 5 + gh gw <= %d parameters per window; a %d x %d "
                             "grid has K = %d" % (who, MAX_FIT_PARAMETERS, gh, gw, MOTION_PARAMETERS + gh * gw))
    sigmas = [float(s) for s in (blur_sigma if isinstance(blur_sigma, (list, tuple)) else [blur_sigma])]
    if not sigmas:
        raise ValueError("blur_sigma must be a number or a non-empty sequence")
    _check_line_search_steps(line_search_steps)
    if float(smoothness) < 0 or not float(charbonnier_eps) > 0:
        raise ValueError("smoothness must be >= 0 and charbonnier_eps > 0")
    if not (float(rotation_scale) > 0 and float(direction_scale) > 0):
        raise ValueError("rotation_scale and direction_scale must be > 0")
    if x0 is None:
        raise ValueError("%s needs x0, the start motion (wx, wy, wz, vx, vy, vz) whose speed |v| it keeps" % who)
    if inv_depth_range is None:
        raise ValueError("%s needs inv_depth_range, the [lo, hi] box of every node" % who)
    B = _window_count(batch_end_indices)
    _check_per_window(x0, B, (6,), "x0")
    _check_per_window(inv_depth_range, B, (2,), "inv_depth_range")
    if not isinstance(x0, torch.Tensor) or x0.device.type == "cpu":
        v0 = torch.as_tensor(np.asarray(x0, dtype=np.float64) if not isinstance(x0, torch.Tensor) else x0,
                             dtype=torch.float64).reshape(-1, 6)[:, 3:]
        if not bool((v0.norm(dim=1) > 0).all()):
            raise ValueError("x0 has a zero speed |v|: depth and translation share one scale, which the fit keeps at "
                             "|x0[3:]|; pass speed 1 for depth up to scale")
    if not isinstance(inv_depth_range, torch.Tensor) or inv_depth_range.device.type == "cpu":
        r = torch.as_tensor(inv_depth_range, dtype=torch.float64)
        if not bool(((r[..., 0] >= 0) & (r[..., 0] < r[..., 1])).all()):
            raise ValueError("inv_depth_range must have 0 <= lo < hi, got %s" % (r.tolist(),))
    gh0, gw0 = shapes[0]
    if inv_depth0 is not None:
        _check_per_window(inv_depth0, B, (gh0, gw0), "inv_depth0")
    elif int(num_samples) < 1 or int(num_samples) % 2 != 1 or int(grid_levels) < 1:
        raise ValueError("num_samples must be odd and grid_levels >= 1, got %r and %r" % (num_samples, grid_levels))
    lam, eps = float(smoothness), float(charbonnier_eps)
    _lib.lib()
    dev = E.compute_device(*(a for a in (x0, inv_depth_range, inv_depth0, xs, ys, ts, ps) if isinstance(a, torch.Tensor)))
    ev = _batch_events(xs, ys, ts, ps, t0, batch_end_indices, B, dev, "windows")
    centre = _centre(_lib.WARP_CAMERA_MOTION, warpfunc)
    with torch.cuda.device(dev):
        motion = _per_window(x0, B, (6,), "x0", dev)
        box = _per_window(inv_depth_range, B, (2,), "inv_depth_range", dev).unsqueeze(1)     # (B,1,2)
        spacing = (box[:, 0, 1] - box[:, 0, 0]) / (max(int(num_samples), 2) - 1)
        if inv_depth0 is None:
            def candidates(ev, c, model, sigma):
                return _depth_grid_candidates(ev, c, model, _scalars(objective, sigma, obj_param))
            start = _constant_start(ev, box, (gh0, gw0), H, W, _model(motion, warpfunc, B, dev, None, H, W)[4], sigmas[0],
                                    int(num_samples), int(grid_levels), candidates)
            grid = start.view(B, 1, 1, 1).expand(B, 1, gh0, gw0).contiguous()
        else:
            grid = _per_window(inv_depth0, B, (gh0, gw0), "inv_depth0", dev).unsqueeze(1)
        iters = torch.zeros(B, dtype=torch.int32, device=dev)
        inf = torch.full((B, 3), float("inf"), dtype=torch.float64, device=dev)
        inf = torch.stack((-inf, inf), dim=-1)                                   # w is free
        chart = torch.full((B, 2), CHART_BOX, dtype=torch.float64, device=dev)
        chart = torch.stack((-chart, chart), dim=-1)
        status = F = None
        for gh, gw in shapes:
            if tuple(grid.shape[2:]) != (gh, gw):
                grid = torch.nn.functional.interpolate(grid, (gh, gw), mode="bilinear", align_corners=True)
            grid = torch.minimum(torch.maximum(grid, box[..., 0, None, None]), box[..., 1, None, None])
            G = gh * gw
            bounds = torch.cat((inf, chart, box.expand(B, G, 2)), dim=1)
            scale = torch.cat((torch.full((B, 3), float(rotation_scale), dtype=torch.float64, device=dev),
                               torch.full((B, 2), float(direction_scale), dtype=torch.float64, device=dev),
                               spacing.view(B, 1).expand(B, G)), dim=1)
            for sigma in sigmas:
                scalars = _scalars(objective, sigma, obj_param)
                frame = _chart_frame(motion[:, 3:])
                fg, cand = _joint_stage(_joint_objective(ev, (gh, gw), H, W, centre, scalars), ev, frame, (gh, gw), H, W,
                                        centre, scalars, lam, eps)
                xk = torch.cat((motion[:, :3], torch.zeros((B, 2), dtype=torch.float64, device=dev), grid.reshape(B, G)), 1)
                xk, F, status, it = _batched_bfgs(fg, cand, xk, scale, max_iter, line_search_steps, ftol, gtol, bounds,
                                                  unit_first_step=True)
                iters += it
                motion = torch.cat((xk[:, :3], _chart_velocity(xk[:, 3:5], frame)), dim=1)
                grid = xk[:, MOTION_PARAMETERS:].reshape(B, 1, gh, gw)
        rest = F - lam * charbonnier_smoothness(grid, eps)[0]
    return MotionAndDepthFit(motion, grid[:, 0], F, rest, status, iters)


def _joint_stage(fg_joint, ev, frame, grid, H, W, centre, scalars, lam, eps):
    """fg and candidates of F = f + lam R over x = (w, a, b, D) (B, 5 + gh gw) for _batched_bfgs, with v on the chart
    `frame`"""
    gh, gw = grid

    def motion_of(x):
        return torch.cat((x[..., :3], _chart_velocity(x[..., 3:5].reshape(-1, 2), frame_of(x)).reshape(x.shape[:-1] + (3,))),
                         dim=-1)

    def frame_of(x):
        if x.dim() == 2:
            return frame
        J = x.shape[1]
        return tuple(t.repeat_interleave(J, dim=0) for t in frame)

    def fg(x):
        ab, D = x[:, 3:5], x[:, MOTION_PARAMETERS:]
        f, gm, gd = fg_joint(motion_of(x), D)
        R, gR = charbonnier_smoothness(D.view(-1, 1, gh, gw), eps)
        g = torch.cat((gm[:, :3], _chart_gradient(ab, frame, gm[:, 3:]), gd + lam * gR.reshape(gd.shape)), dim=1)
        return f + lam * R, g

    def candidates(pts):
        B, J, _ = pts.shape
        D = pts[..., MOTION_PARAMETERS:]
        f = _joint_candidates(ev, motion_of(pts), D.to(torch.float32).contiguous(), grid, H, W, centre, scalars)
        return f + lam * charbonnier_smoothness(D.reshape(B, J, 1, gh, gw), eps)[0]
    return fg, candidates
