"""The plumbing the batched losses share (flow_objective, flow_timestamp_objective, motion_objective,
motion_timestamp_objective, motion_fit, motion_timestamp_fit, motion_segmentation): the events of a batch as the kernels
take them, the checks of the arguments the public functions have in common, and the two loops that run an entry over
chunks of windows -- the candidates passes (_chunked_candidates) and a fit's forward and gradient (_chunked_objective).
The chunk rule itself is fit_window_chunk.
"""
import torch

from .. import _lib
from ..representations import _events as E
from .warps import (affine_warp, camera_motion_warp, camera_rotation_warp, homography_warp, linvel_warp, pure_rotation_warp,
                    xyztheta_warp)

OBJECTIVES = {"variance": _lib.OBJ_VARIANCE, "sos": _lib.OBJ_SOS, "soe": _lib.OBJ_SOE, "sosa": _lib.OBJ_SOSA}
DEFAULT_PARAM = {"sosa": 3.0}   # sosa_objective(p=3)
_WARPS = ((linvel_warp, _lib.WARP_LINVEL), (pure_rotation_warp, _lib.WARP_ROTATION), (xyztheta_warp, _lib.WARP_XYZTHETA),
          (affine_warp, _lib.WARP_AFFINE), (homography_warp, _lib.WARP_HOMOGRAPHY),
          (camera_rotation_warp, _lib.WARP_CAMERA_ROTATION), (camera_motion_warp, _lib.WARP_CAMERA_MOTION))
# the models about a fixed centre (cx, cy), the camera models' principal point
_CENTRED = (_lib.WARP_XYZTHETA, _lib.WARP_AFFINE, _lib.WARP_HOMOGRAPHY, _lib.WARP_CAMERA_ROTATION, _lib.WARP_CAMERA_MOTION)
# the camera models, whose rows carry their focal lengths (_rows)
_FOCAL = (_lib.WARP_CAMERA_ROTATION, _lib.WARP_CAMERA_MOTION)
MAX_CANDIDATES = 32   # parameter vectors per window and pass over the events
MAX_GRID_CANDIDATE_NODES = 12288   # candidates times nodes of a grid-flow candidates pass (the grids a CTA holds)


def _check_objective(objective, wrt):
    if objective not in OBJECTIVES:
        if objective in ("moa", "isoa"):
            raise ValueError("objective %r is piecewise constant in the %s and has no gradient; use one of %s"
                             % (objective, wrt, sorted(OBJECTIVES)))
        raise ValueError("unknown objective %r (one of %s)" % (objective, sorted(OBJECTIVES)))


def _warp_code(warpfunc, who):
    warp = next((code for cls, code in _WARPS if type(warpfunc) is cls), None)
    if warp is None:
        raise ValueError("%s supports the models linvel_warp, pure_rotation_warp and xyztheta_warp, the planar models "
                         "affine_warp and homography_warp, and camera_rotation_warp and camera_motion_warp, got %s"
                         % (who, type(warpfunc).__name__))
    return warp


def _depth_tensor(inv_depth, warp, n, who):
    """The checks of inv_depth, before any CUDA call: the camera_motion_warp's inverse depth of every event is required
    with that model and rejected with any other; an (N,) float array aligned with the concatenated events, data (no
    grad).  Returns it flat, or None."""
    if warp != _lib.WARP_CAMERA_MOTION:
        if inv_depth is not None:
            raise ValueError("%s: inv_depth is the per-event inverse depth of camera_motion_warp; the other models take "
                             "none" % who)
        return None
    if inv_depth is None:
        raise ValueError("%s: camera_motion_warp needs inv_depth, the inverse depth of every event (an (N,) array aligned "
                         "with the events)" % who)
    rho = _float_tensor(inv_depth, "inv_depth")
    if rho.requires_grad:
        raise ValueError("%s: inv_depth is data and must not require grad (detach it)" % who)
    if rho.dim() != 1 or rho.shape[0] != n:
        raise ValueError("%s: inv_depth must have shape (%d,), one value per event, got %s" % (who, n, tuple(rho.shape)))
    return rho


def _depth_events(rho, dev):
    """the checked inverse depth as the depth entries take it, f32 on dev (None stays None)"""
    if rho is None:
        return None
    with torch.cuda.device(dev):
        return E.to_device(rho, dev).to(torch.float32).contiguous()


def _depth_entry(stem, events, rho):
    """the entry stem and event arrays of a motion loss: the depth twin of `stem` (evk_cmax_motion_objective ->
    evk_cmax_motion_depth_objective), which takes the inverse depth right after the other event arrays, when rho is given"""
    if rho is None:
        return stem, events
    head, tail = stem.rsplit("_", 1)
    return "%s_depth_%s" % (head, tail), tuple(events) + (rho,)


def _centre(warp, warpfunc):
    """the model's constants: (cx, cy), which the entries take behind K, followed for camera_rotation_warp and
    camera_motion_warp by their focal lengths (fx, fy), which _rows appends to every parameter row"""
    centre = tuple(float(c) for c in warpfunc.center) if warp in _CENTRED else (0.0, 0.0)
    if warp in _FOCAL:
        centre += tuple(float(f) for f in warpfunc.focal)
    return centre


def _rows(params, centre):
    """params (..., K) as the rows of the motion entries: for camera_rotation_warp (centre (cx, cy, fx, fy)) each row
    (wx, wy, wz) becomes (wx, wy, wz, fx, fy), in f64, and camera_motion_warp's (wx, wy, wz, vx, vy, vz) likewise.  Differentiable in params, so the focal-length columns of the
    entries' gradient drop out through autograd; the two columns are fills on params' device, with no host round trip.
    Any other model's params come back as they are."""
    if len(centre) == 2:
        return params
    params = params.to(torch.float64)
    return torch.cat([params] + [params.new_full(params.shape[:-1] + (1,), f) for f in centre[2:]], dim=-1)


def _model(warp, warpfunc, objective, blur_sigma, obj_param, H, W):
    """the scalar arguments the motion entries share: (warp code, _centre, H, W, objective code, sigma, obj_param)"""
    centre = _centre(warp, warpfunc)
    param = float(obj_param if obj_param is not None else DEFAULT_PARAM.get(objective, 0.0))
    return warp, centre, H, W, OBJECTIVES[objective], float(blur_sigma), param


def _ts_model(warp, warpfunc, blur_sigma, H, W):
    """the scalar arguments the motion timestamp entries share: (warp code, _centre, H, W, sigma)"""
    return warp, _centre(warp, warpfunc), H, W, float(blur_sigma)


def _float_tensor(v, name):
    v = E.as_tensor(v)
    if not v.is_floating_point():
        raise ValueError("%s must be a floating-point tensor, got %s" % (name, v.dtype))
    return v


def _params_tensor(params, warpfunc):
    """params as a (B,K) float tensor ((K,) is one sample)"""
    params = _float_tensor(params, "params")
    if params.dim() == 1:
        params = params.unsqueeze(0)
    if params.dim() != 2 or params.shape[1] != warpfunc.dims:
        raise ValueError("params must have shape (B,%d) or (%d,) for %s, got %s"
                         % (warpfunc.dims, warpfunc.dims, type(warpfunc).__name__, tuple(params.shape)))
    return params


def _candidates_tensor(candidates, warpfunc):
    """candidates as a (B,J,K) float tensor"""
    cand = _float_tensor(candidates, "candidates")
    if cand.dim() != 3 or cand.shape[2] != warpfunc.dims or cand.shape[1] < 1:
        raise ValueError("candidates must have shape (B,J,%d) with J >= 1 for %s, got %s"
                         % (warpfunc.dims, type(warpfunc).__name__, tuple(cand.shape)))
    return cand


def _window_count(batch_end_indices):
    if batch_end_indices is None:
        return 1
    if isinstance(batch_end_indices, torch.Tensor):
        return batch_end_indices.reshape(-1).shape[0]
    return len(batch_end_indices)


def _check_window_count(batch_end_indices, B, what):
    """_batch_events' check of the sample count, for the functions that make it before any CUDA call"""
    if batch_end_indices is not None and _window_count(batch_end_indices) != B:
        raise ValueError("%d samples of events for a batch of %d %s" % (_window_count(batch_end_indices), B, what))


def _event_tensors(xs, ys, ts, ps, t0, who, wrt):
    """the events as flat tensors; they and t0 are data and must not require grad"""
    xs, ys, ts, ps = (E.as_tensor(a).reshape(-1) for a in (xs, ys, ts, ps))
    if any(a.requires_grad for a in (xs, ys, ts, ps)) or (isinstance(t0, torch.Tensor) and t0.requires_grad):
        raise ValueError("%s differentiates with respect to %s only; the events and t0 must not require grad (detach them)"
                         % (who, wrt))
    n = xs.shape[0]
    if not (ys.shape[0] == ts.shape[0] == ps.shape[0] == n):
        raise ValueError("xs, ys, ts, ps must have the same length")
    return xs, ys, ts, ps


def _batch_events(xs, ys, ts, ps, t0, batch_end_indices, B, dev, what, stamps=False):
    """The events of a batch of B samples on `dev` as the batched kernels take them: x, y, p f32, t_rel = t - t0_b
    formed in ts' dtype then cast to f32 (t0 None: each sample's last stamp), and the B+1 int64 sample offsets.
    With `stamps`, also the stamps on `dev` in that dtype and the sample index of every event."""
    n = xs.shape[0]
    with torch.cuda.device(dev):
        if batch_end_indices is None:
            ends = torch.full((1,), n, dtype=torch.int64, device=dev)
        elif isinstance(batch_end_indices, torch.Tensor):
            ends = batch_end_indices.reshape(-1).to(device=dev, dtype=torch.int64)
        else:
            ends = torch.tensor([int(e) for e in batch_end_indices], dtype=torch.int64).to(dev)
        if ends.shape[0] != B:
            raise ValueError("%d samples of events for a batch of %d %s" % (ends.shape[0], B, what))
        offsets = torch.cat((torch.zeros(1, dtype=torch.int64, device=dev), ends))
        x, y, p = (E.to_device(a, dev).to(torch.float32).contiguous() for a in (xs, ys, ps))
        t = E.to_device(ts, dev)
        rt = torch.result_type(t, 1.0)
        t = t.to(rt)
        if n == 0:
            t_rel = torch.empty(0, dtype=torch.float32, device=dev)
            sample = torch.empty(0, dtype=torch.int64, device=dev)
        else:
            if t0 is None:
                t0b = t[(ends - 1).clamp(0, n - 1)]                     # each sample's last event (as warp_events_flow_torch)
            else:
                t0b = torch.as_tensor(t0, dtype=rt).to(dev).reshape(-1).expand(B)
            # the sample of each event: windows are contiguous, [ends[b-1], ends[b])
            sample = torch.searchsorted(ends, torch.arange(n, device=dev), right=True).clamp_(max=B - 1)
            t_rel = (t - t0b.to(rt)[sample]).to(torch.float32).contiguous()
    if stamps:
        return x, y, t_rel, p, offsets, t, sample
    return x, y, t_rel, p, offsets


def _normalised_stamps(t, sample, offsets, reverse):
    """tau of every event as f32: (t - t_first_b) / (t_last_b - t_first_b + 1e-6) of its sample b, or
    (-t + t_last_b) / (...) (image.py:324-327), in t's dtype, as device tensor ops (no host read-back).  t: the stamps
    in a float dtype, sample: each event's sample index, offsets: the B+1 sample offsets."""
    n = t.shape[0]
    if n == 0:
        return torch.empty(0, dtype=torch.float32, device=t.device)
    t_first = t[offsets[:-1].clamp(0, n - 1)]
    t_last = t[(offsets[1:] - 1).clamp(0, n - 1)]
    den = ((t_last - t_first) + 1e-6)[sample]
    num = (-t + t_last[sample]) if reverse else (t - t_first[sample])
    return (num / den).to(torch.float32).contiguous()


def _timestamp_events(xs, ys, ts, ps, t0, batch_end_indices, B, dev, what, reverse):
    """_batch_events for the average-timestamp losses: x, y, t_rel, tau (_normalised_stamps), p, offsets"""
    x, y, t_rel, p, offsets, t, sample = _batch_events(xs, ys, ts, ps, t0, batch_end_indices, B, dev, what, stamps=True)
    with torch.cuda.device(dev):
        tau = _normalised_stamps(t, sample, offsets, reverse)
    return x, y, t_rel, tau, p, offsets


def fit_window_chunk(B, per_window_bytes, budget, cap):
    """Windows per call of a fit's forward and gradient entries: at most `cap` (the entries' batch limit) and at most
    as many as fit `budget` bytes of workspace and images, but at least one"""
    return max(1, min(B, budget // per_window_bytes, cap))


def _pointers(tensors):
    return tuple(_lib.ptr(a) for a in tensors)


def _model_layout(model, K):
    """the arguments of a motion entry in front of its parameter pointer, between the parameter count and (H, W), and
    those its workspace query takes in front of (H, W): model = (warp, _centre, H, W); K is the parameters per row
    before _rows.  A grid-flow entry takes model = ("grid", (gh, gw), H, W): its grids of K = 2 gh gw floats are
    followed by gh, gw, which its query takes too.  A depth-grid entry takes model = ("grid", (gh, gw), H, W,
    (rows, cx, cy)): the device motion rows (B,8) f64 of the windows and the principal point go in front of its grids
    of K = gh gw floats (_lead passes the rows of a chunk's windows)."""
    kind, extra, H, W = model[:4]
    if kind == "grid":
        return tuple(model[4]) if len(model) > 4 else (), (), extra, extra, H, W
    return (kind,), (K + len(extra) - 2, extra[0], extra[1]), (), (), H, W


def _lead(pre, b0):
    """_model_layout's arguments in front of the parameter pointer for the chunk from window b0: a tensor of per-window
    rows goes as the pointer to row b0"""
    return tuple(_lib.ptr(a[b0:]) if isinstance(a, torch.Tensor) else a for a in pre)


def _chunked_candidates(stem, key, events, offsets, c64, model, scalars, budget, cap, M=None):
    """f (B,J) f64 of the prepared device events under the device candidates c64 (B,J,K) through the entry `stem`_f32,
    in passes of at most MAX_CANDIDATES candidate images per window over chunks of windows whose workspace
    (`stem`_workspace_bytes) fits `budget` and whose images number at most `cap`.  `events` are the arrays in front of
    the offsets and `scalars` the arguments behind W; model is _model_layout's.  With M, the entry scores M models per
    window: the last of `events` is the memberships, c64 is (B,M,J,K) and f (B,M,J).  The camera models' candidates
    reach the entry with their focal lengths (_rows); camera_motion_warp's `events` end with the inverse depth
    (_depth_entry)."""
    J, K = c64.shape[-2:]
    pre, mid, grid, query, H, W = _model_layout(model, K)
    B = c64.shape[0]
    ms = () if M is None else (M,)
    L = _lib.lib()
    entry, workspace_bytes = getattr(L, stem + "_f32"), getattr(L, stem + "_workspace_bytes")
    dev = events[0].device
    f = torch.empty(c64.shape[:-1], dtype=torch.float64, device=dev)
    if B == 0:
        return f
    jc = min(J, MAX_CANDIDATES // (M or 1))
    if grid:
        jc = max(1, min(jc, MAX_GRID_CANDIDATE_NODES // (grid[0] * grid[1])))
    wb = fit_window_chunk(B, workspace_bytes(1, *ms, jc, *query, H, W), budget, cap // ((M or 1) * jc))
    ws = _lib.scratch(key, workspace_bytes(wb, *ms, jc, *query, H, W), dev)
    front = _pointers(events) + ms
    for b0 in range(0, B, wb):
        b1 = min(B, b0 + wb)
        for j0 in range(0, J, jc):
            j1 = min(J, j0 + jc)
            c = _rows(c64[b0:b1, ..., j0:j1, :], model[1]).contiguous()
            out = torch.empty(c.shape[:-1], dtype=torch.float64, device=dev)
            _lib.check(entry(*front, _lib.ptr(offsets[b0:]), b1 - b0, events[0].shape[0], *_lead(pre, b0), _lib.ptr(c),
                             j1 - j0, *mid, *grid, H, W, *scalars, _lib.ptr(out), _lib.ptr(ws), ws.numel(), _lib.stream()))
            f[b0:b1, ..., j0:j1] = out
    return f


def _chunked_objective(stem, key, events, offsets, model, scalars, images, budget, cap, M=None, gradient=True):
    """fg: (B,K) f64 params -> (f (B,) f64, g (B,K) f64) of the prepared device events through the entries `stem`_f32 /
    `stem`_grad_f32 (grad_f = 1), in chunks of at most `cap` windows whose workspace (`stem`_workspace_bytes) and images
    fit `budget` (fit_window_chunk); the windows are independent, so a chunk changes no value's arithmetic.  `events`
    are the arrays in front of the offsets, `scalars` the arguments behind W, model is _model_layout's and `images` the
    canvases per window of each image the forward hands to the gradient.  With M, the entries score M models per window:
    the last of `events` is the memberships (they get no gradient), params is (B*M,K), f (B*M,) and g (B*M,K).  Without
    `gradient`, g is None and the gradient entry is not called.  A grid-flow entry takes the parameters (the nodes) and
    returns their gradient in f32.  The camera models' rows reach the entries with their focal lengths (_rows), and
    g leaves out the entries' two focal-length columns."""
    ms, no_weight_gradient = ((), ()) if M is None else ((M,), (None,))
    rows = M or 1
    L = _lib.lib()
    forward, grad, workspace_bytes = (getattr(L, stem + s) for s in ("_f32", "_grad_f32", "_workspace_bytes"))
    dev = events[0].device
    front = _pointers(events) + ms

    def fg(params):
        K = params.shape[1]
        B = params.shape[0] // rows
        pre, mid, grid, query, H, W = _model_layout(model, K)
        dtype = torch.float32 if grid else torch.float64
        prm = _rows(params.to(dtype), model[1]).contiguous()
        f = torch.empty(B * rows, dtype=torch.float64, device=dev)
        g = torch.empty((B * rows, prm.shape[1]), dtype=dtype, device=dev) if gradient else None
        wb = fit_window_chunk(B, workspace_bytes(1, *ms, *query, H, W) + 4 * sum(images) * (H + 1) * (W + 1), budget, cap)
        kept = [torch.empty((wb * c, H + 1, W + 1), dtype=torch.float32, device=dev) for c in images]
        imgs = _pointers(kept)
        ones = torch.ones(wb * rows, dtype=torch.float32, device=dev)
        ws = _lib.scratch(key, workspace_bytes(wb, *ms, *query, H, W), dev)
        for b0 in range(0, B, wb):
            b1 = min(B, b0 + wb)
            r0, r1 = b0 * rows, b1 * rows
            ev = front + (_lib.ptr(offsets[b0:]), b1 - b0, events[0].shape[0], *_lead(pre, b0), _lib.ptr(prm[r0:r1]), *mid,
                          *grid, H, W, *scalars)
            _lib.check(forward(*ev, _lib.ptr(f[r0:r1]), *imgs, _lib.ptr(ws), ws.numel(), _lib.stream()))
            if gradient:
                _lib.check(grad(*ev, *imgs, _lib.ptr(ones), _lib.ptr(g[r0:r1]), *no_weight_gradient, _lib.ptr(ws),
                                ws.numel(), _lib.stream()))
        return f, (g[:, :K].to(torch.float64) if g is not None else None)
    return fg
