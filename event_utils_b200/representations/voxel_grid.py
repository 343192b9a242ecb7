"""Voxel-grid builders -- drop-in for the reference's lib/representations/voxel_grid.py.

Same signatures and return types; the work is one CUDA pass over the events
(csrc/evk_voxel.cu) instead of B passes of ~15 temporaries each.
"""
import ctypes

import numpy as np
import torch

from .. import _lib, config
from . import _events as E
from .image import events_to_image, events_to_image_torch  # noqa: F401  (re-exported like the reference)


def _voxel_device(x, y, t, p, t0, dt, B, H, W, flags=0, aos=None, out=None):
    """Launch the voxel kernels on device-resident f32 arrays; returns (B,H,W) f32 on that device."""
    L = _lib.lib()
    dev = (aos if aos is not None else x).device
    with torch.cuda.device(dev):
        if out is None:
            out = torch.empty((B, H, W), dtype=torch.float32, device=dev)
        flags |= E.variant_flag()
        ws_bytes = L.evk_voxel_workspace_bytes(B, H, W, flags)
        ws = _lib.scratch("voxel_ws", ws_bytes, dev)
        oob = _lib.oob_counter(dev)
        if aos is not None:
            _lib.check(L.evk_voxel_aos_f32(_lib.ptr(aos), aos.shape[0], t0, dt, B, H, W, flags, _lib.ptr(out),
                                           _lib.ptr(ws), ws.numel(), _lib.ptr(oob), _lib.stream()))
        else:
            _lib.check(L.evk_voxel_f32(_lib.ptr(x), _lib.ptr(y), _lib.ptr(t), _lib.ptr(p), x.shape[0], t0, dt,
                                       B, H, W, flags, _lib.ptr(out), _lib.ptr(ws), ws.numel(), _lib.ptr(oob),
                                       _lib.stream()))
        E.raise_if_oob(oob, "voxel grid", (B, H, W))
    return out


def _times_f32(ts, dev):
    """Timestamps as f32 + the two scalars voxel_grid.py:133-134 derives from them.
    Integer timestamps are made relative first (exact), like the reference's int arithmetic."""
    loader_arrays = isinstance(ts, np.ndarray)
    ts = E.as_tensor(ts).reshape(-1)
    if ts.dtype == torch.float64 and loader_arrays:
        # numpy float64 stamps, as the data loaders hold them (hdf5_dataset.py:18-23): the reference
        # cannot take numpy at all (quirk B4), so this is our extension -- made relative to the first
        # stamp in float64 BEFORE the cast, because absolute stamps (1.6e9 s + us) do not fit float32
        t64 = E.to_device(ts, dev)
        rel = (t64 - t64[0])
        dt = np.float32(float(rel[-1].item()))
        return rel.to(torch.float32).contiguous(), 0.0, float(dt)
    if ts.dtype == torch.float32:
        t = E.to_device(ts, dev).contiguous()
        first, last = (float(v) for v in torch.stack((ts[0], ts[-1])).tolist())
        t0 = np.float32(first)
        dt = np.float32(last) - np.float32(first)
        return t, float(t0), float(dt)
    if ts.dtype == torch.float64:
        # the reference fails here: index_put_ f64 weights into an f32 image (image.py:95)
        raise RuntimeError("Index put requires the source and destination dtypes match, "
                           "got Float for the destination and Double for the source.")
    ts = E.to_device(ts, dev)
    if not ts.dtype.is_floating_point:
        rel = (ts - ts[0])
        dt = np.float32(float(rel[-1].item()))
        return rel.to(torch.float32).contiguous(), 0.0, float(dt)
    t = ts.to(torch.float32).contiguous()
    return t, float(t[0].item()), float((t[-1] - t[0]).item())


def _device_events(xs, ys, ts, ps, dev, aos_ok=True):
    """The events as the voxel kernels take them on `dev`: (aos, x, y, t, p, t0, dt, flags).  aos is the (N,4) view when
    the four arrays are the columns of one CUDA tensor (x, y, t, p are then None).  t0 / dt are read on the device
    (EVK_AUTO_SPAN in flags) when the stamps are f32 on the device already."""
    aos = E.aos_base(xs, ys, ts, ps) if aos_ok and isinstance(xs, torch.Tensor) and xs.is_cuda else None
    if aos is not None:
        # t0 / dt are read on the device (EVK_AUTO_SPAN): no host round trip before the launch
        return aos, None, None, None, None, 0.0, 1.0, _lib.AUTO_SPAN
    ts_t = E.as_tensor(ts)
    if ts_t.is_cuda and ts_t.dtype == torch.float32 and ts_t.dim() == 1:
        t, t0, dt, flags = ts_t.contiguous(), 0.0, 1.0, _lib.AUTO_SPAN
    else:
        t, t0, dt = _times_f32(ts, dev)
        flags = 0
    return None, E.coords_f32(xs, dev), E.coords_f32(ys, dev), t, E.weights_f32(ps, dev), t0, dt, flags


def events_to_voxel_torch(xs, ys, ts, ps, B, device=None, sensor_size=(180, 240), temporal_bilinear=True):
    """
    Turn a set of events into a (B,H,W) float32 voxel grid with temporal bilinear interpolation.
    Drop-in for lib/representations/voxel_grid.py:114-153.
    @param xs, ys, ts, ps event components (tensors on any device, or numpy arrays)
    @param B number of bins
    @param device device of the returned grid (default: the device of xs)
    @param sensor_size (H, W)
    @param temporal_bilinear only True is defined (the reference's False branch raises NameError)
    @returns voxel grid tensor
    Differentiable like the reference w.r.t. ps and ts (event_utils_b200.autograd).
    """
    assert(len(xs) == len(ys) and len(ys) == len(ts) and len(ts) == len(ps))
    if not temporal_bilinear:
        raise NotImplementedError("temporal_bilinear=False is undefined in the reference "
                                  "(voxel_grid.py:144-147 raises NameError)")
    if len(xs) == 0:
        raise IndexError("index -1 is out of bounds for dimension 0 with size 0")
    xs_t = E.as_tensor(xs)
    if device is None:
        device = xs_t.device
    device = torch.device(device)
    H, W = int(sensor_size[0]), int(sensor_size[1])
    B = int(B)
    ps_t = E.as_tensor(ps)
    if ps_t.dtype == torch.float64 and not isinstance(ps, np.ndarray):
        raise RuntimeError("Index put requires the source and destination dtypes match, "
                           "got Float for the destination and Double for the source.")
    dev = E.compute_device(xs, ys, ts, ps)
    if E.needs_grad(ps, ts):
        from ..autograd import VoxelGrid
        return VoxelGrid.apply(xs, ys, ts, ps, (device, B, H, W, False, None))

    host_f32 = all(isinstance(a, torch.Tensor) and not a.is_cuda and a.dtype == torch.float32
                   and a.dim() == 1 and a.is_contiguous() for a in (xs, ys, ts, ps))
    if host_f32:
        # host arrays: chunked, double-buffered H2D copy overlapped with the scatter (evk_host.cu)
        L = _lib.lib()
        with torch.cuda.device(dev):
            t0 = np.float32(ts[0].item())
            dt = np.float32(ts[-1].item()) - t0
            out = torch.empty((B, H, W), dtype=torch.float32, pin_memory=True)
            bad = ctypes.c_ulonglong(0)
            _lib.check(L.evk_voxel_host_f32(_lib.pipeline(), _lib.ptr(xs), _lib.ptr(ys), _lib.ptr(ts), _lib.ptr(ps),
                                            xs.shape[0], float(t0), float(dt), B, H, W, 0, _lib.ptr(out),
                                            ctypes.byref(bad)))
        if bad.value and config.check_index_errors:
            raise IndexError("%d events index outside the voxel grid of shape %s" % (bad.value, (B, H, W)))
        return out if device.type == "cpu" else out.to(device)

    aos, x, y, t, p, t0, dt, flags = _device_events(xs, ys, ts, ps, dev)
    grid = _voxel_device(x, y, t, p, t0, dt, B, H, W, flags=flags, aos=aos)
    return grid if grid.device == device else grid.to(device)


def events_to_voxel_packed(xs, ys, ts, ps, B, device=None, sensor_size=(180, 240)):
    """
    Voxel grid straight from the reference's STORAGE layout (extension, row f4 of the scope table):
    xs, ys int16, ts float64, ps bool / uint8 in {0,1} -- what DynamicH5Dataset / MemMapDataset read
    from disk (hdf5_dataset.py:18-23, memmap_dataset.py) before they cast.  Polarity is mapped p*2-1
    and the stamps are made relative in float64 on the device; numpy or torch inputs, host or CUDA.
    Equals events_to_voxel_torch(xs.float(), ys.float(), (ts-ts[0]).float(), ps*2-1, B, ...).
    """
    assert(len(xs) == len(ys) and len(ys) == len(ts) and len(ts) == len(ps))
    if len(xs) == 0:
        raise IndexError("index -1 is out of bounds for dimension 0 with size 0")
    L = _lib.lib()
    xt, yt, tt, pt = (E.as_tensor(a).reshape(-1) for a in (xs, ys, ts, ps))
    if device is None:
        device = xt.device
    device = torch.device(device)
    dev = E.compute_device(xt, yt, tt, pt)
    H, W, B = int(sensor_size[0]), int(sensor_size[1]), int(B)
    pb = pt.view(torch.uint8) if pt.dtype == torch.bool else pt
    if (not xt.is_cuda and xt.dtype == torch.int16 and yt.dtype == torch.int16 and tt.dtype == torch.float64
            and pb.dtype == torch.uint8 and all(a.is_contiguous() for a in (xt, yt, tt, pb))):
        # host arrays in the storage dtypes: chunked, double-buffered H2D of the RAW 13 B/event
        with torch.cuda.device(dev):
            out = torch.empty((B, H, W), dtype=torch.float32, pin_memory=True)
            bad = ctypes.c_ulonglong(0)
            _lib.check(L.evk_voxel_host_packed_f32(_lib.pipeline(), _lib.ptr(xt), _lib.ptr(yt), _lib.ptr(tt), _lib.ptr(pb),
                                                   xt.shape[0], float(tt[0]), float(tt[-1]), B, H, W, 0, _lib.ptr(out),
                                                   ctypes.byref(bad)))
        if bad.value and config.check_index_errors:
            raise IndexError("%d events index outside the voxel grid of shape %s" % (bad.value, (B, H, W)))
        return out if device.type == "cpu" else out.to(device)
    with torch.cuda.device(dev):
        x = E.to_device(xt, dev).to(torch.int16).contiguous()
        y = E.to_device(yt, dev).to(torch.int16).contiguous()
        t = E.to_device(tt, dev).to(torch.float64).contiguous()
        p = E.to_device(pt, dev).to(torch.uint8).contiguous()
        out = torch.empty((B, H, W), dtype=torch.float32, device=dev)
        flags = E.variant_flag() | _lib.AUTO_SPAN
        ws = _lib.scratch("voxel_ws", L.evk_voxel_workspace_bytes(B, H, W, flags), dev)
        oob = _lib.oob_counter(dev)
        _lib.check(L.evk_voxel_packed_f32(_lib.ptr(x), _lib.ptr(y), _lib.ptr(t), _lib.ptr(p), x.shape[0], 0.0, 1.0, B, H, W,
                                          flags, _lib.ptr(out), _lib.ptr(ws), ws.numel(), _lib.ptr(oob), _lib.stream()))
        E.raise_if_oob(oob, "voxel grid", (B, H, W))
    return out if out.device == device else out.to(device)


def events_to_neg_pos_voxel_torch(xs, ys, ts, ps, B, device=None, sensor_size=(180, 240), temporal_bilinear=True):
    """
    Positive and negative events in separate voxel grids; drop-in for voxel_grid.py:155-182
    (weights [p>0] and [p<=0]).  The reference runs the whole voxel build twice; here both grids
    come out of ONE pass over the events (evk_voxel_negpos_f32).  Differentiable like the reference
    w.r.t. ts (event_utils_b200.autograd).
    @returns (voxel_pos, voxel_neg)
    """
    assert(len(xs) == len(ys) and len(ys) == len(ts) and len(ts) == len(ps))
    if not temporal_bilinear:
        raise NotImplementedError("temporal_bilinear=False is undefined in the reference "
                                  "(voxel_grid.py:144-147 raises NameError)")
    if len(xs) == 0:
        raise IndexError("index -1 is out of bounds for dimension 0 with size 0")
    _lib.lib()
    if device is None:
        device = E.as_tensor(xs).device
    device = torch.device(device)
    dev = E.compute_device(xs, ys, ts, ps)
    H, W, B = int(sensor_size[0]), int(sensor_size[1]), int(B)
    if E.needs_grad(ts):
        from ..autograd import VoxelGrid
        out = VoxelGrid.apply(xs, ys, ts, ps, (device, B, H, W, True, None))
        return out[0], out[1]
    with torch.cuda.device(dev):
        _, x, y, t, p, t0, dt, flags = _device_events(xs, ys, ts, ps, dev, aos_ok=False)
        out = _negpos_device(x, y, t, p, t0, dt, B, H, W, flags)
    if out.device != device:
        out = out.to(device)
    return out[0], out[1]


def _negpos_device(x, y, t, p, t0, dt, B, H, W, flags):
    """Both grids of events_to_neg_pos_voxel_torch from device-resident f32 arrays: (2,B,H,W) f32."""
    L = _lib.lib()
    dev = x.device
    with torch.cuda.device(dev):
        flags |= E.variant_flag()
        out = torch.empty((2, B, H, W), dtype=torch.float32, device=dev)
        ws = _lib.scratch("voxel_ws", 2 * L.evk_voxel_workspace_bytes(B, H, W, flags), dev)
        oob = _lib.oob_counter(dev)
        _lib.check(L.evk_voxel_negpos_f32(_lib.ptr(x), _lib.ptr(y), _lib.ptr(t), _lib.ptr(p), x.shape[0], t0, dt, B, H, W,
                                          flags, _lib.ptr(out), _lib.ptr(ws), ws.numel(), _lib.ptr(oob), _lib.stream()))
        E.raise_if_oob(oob, "voxel grid", (B, H, W))
    return out


def events_to_voxel(xs, ys, ts, ps, B, sensor_size=(180, 240), temporal_bilinear=True):
    """
    numpy flavour; drop-in for voxel_grid.py:184-217: integer xs/ys, float64 (B,H,W) result.
    Coordinates equal to H or W fall on the (H+1,W+1) canvas' pad row/column and are dropped
    (image.py:17,44); anything negative or larger raises ValueError like ravel_multi_index.
    The accumulation itself runs in f32 on the GPU (<= 1e-6 relative of the f64 reference).
    """
    assert(len(xs) == len(ys) and len(ys) == len(ts) and len(ts) == len(ps))
    if not temporal_bilinear:
        raise NotImplementedError("temporal_bilinear=False is undefined in the reference "
                                  "(voxel_grid.py:210-214 raises UnboundLocalError)")
    xs, ys = np.asarray(xs).squeeze(), np.asarray(ys).squeeze()
    if not (np.issubdtype(xs.dtype, np.integer) and np.issubdtype(ys.dtype, np.integer)):
        raise TypeError("only int indices permitted")
    ts, ps = np.asarray(ts, dtype=np.float64).reshape(-1), np.asarray(ps, dtype=np.float64).reshape(-1)
    H, W = int(sensor_size[0]), int(sensor_size[1])
    dev = E.compute_device()
    with torch.cuda.device(dev):
        x = torch.from_numpy(np.ascontiguousarray(xs).reshape(-1)).to(dev)
        y = torch.from_numpy(np.ascontiguousarray(ys).reshape(-1)).to(dev)
        lo = min(int(x.min()), int(y.min()))
        if lo < 0 or int(x.max()) > W or int(y.max()) > H:
            print("Issue with input arrays! minx={}, maxx={}, miny={}, maxy={}, sensor_size={}".format(
                int(x.min()), int(x.max()), int(y.min()), int(y.max()), (H + 1, W + 1)))
            raise ValueError
        # timestamps relative to the first one in f64, THEN f32: absolute stamps do not fit f32
        trel = torch.from_numpy(ts - ts[0]).to(dev).to(torch.float32)
        dt = float(np.float32(ts[-1] - ts[0]))
        p = torch.from_numpy(ps).to(dev).to(torch.float32)
        grid = _voxel_device(x.to(torch.float32), y.to(torch.float32), trel, p, 0.0, dt, int(B), H + 1, W + 1)
        return grid[:, :H, :W].double().cpu().numpy()


def events_to_neg_pos_voxel(xs, ys, ts, ps, B, sensor_size=(180, 240), temporal_bilinear=True):
    """Drop-in for voxel_grid.py:219-243 (weights np.where(ps,1,0) / np.where(ps,0,1))."""
    ps = np.asarray(ps)
    pos_weights = np.where(ps, 1, 0)
    neg_weights = np.where(ps, 0, 1)
    voxel_pos = events_to_voxel(xs, ys, ts, pos_weights, B, sensor_size=sensor_size, temporal_bilinear=temporal_bilinear)
    voxel_neg = events_to_voxel(xs, ys, ts, neg_weights, B, sensor_size=sensor_size, temporal_bilinear=temporal_bilinear)
    return voxel_pos, voxel_neg


def events_to_voxel_timesync_torch(xs, ys, ts, ps, B, t0, t1, device=None, np_ts=None,
        sensor_size=(180, 240), temporal_bilinear=True):
    """Voxel grid of the events between t0 and t1; drop-in for voxel_grid.py:82-112."""
    assert(t1 > t0)
    if np_ts is None:
        np_ts = ts.detach().cpu().numpy()   # the window bounds only: ts may require grad
    if device is None:
        device = xs.device
    start_idx = np.searchsorted(np_ts, t0)
    end_idx = np.searchsorted(np_ts, t1)
    assert(start_idx < end_idx)
    return events_to_voxel_torch(xs[start_idx:end_idx], ys[start_idx:end_idx], ts[start_idx:end_idx],
                                 ps[start_idx:end_idx], B, device, sensor_size=sensor_size,
                                 temporal_bilinear=temporal_bilinear)


def _batched_windows(xs, ys, ts, ps, starts, ends, B, sensor_size):
    """All windows [starts[w], ends[w]) in ONE launch (evk_voxel_windows_f32); None if the inputs are
    not contiguous float32 CUDA tensors (callers then fall back to one call per window)."""
    if not all(isinstance(a, torch.Tensor) and a.is_cuda and a.dtype == torch.float32 and a.dim() == 1
               and a.is_contiguous() for a in (xs, ys, ts, ps)):
        return None
    H, W, B = int(sensor_size[0]), int(sensor_size[1]), int(B)
    if len(starts) == 0:
        return []
    if E.needs_grad(ps, ts):
        from ..autograd import VoxelGrid
        return list(VoxelGrid.apply(xs, ys, ts, ps, (xs.device, B, H, W, False, (starts, ends))).unbind(0))
    return list(_windows_device(xs, ys, ts, ps, starts, ends, B, H, W)[0].unbind(0))


def _windows_device(xs, ys, ts, ps, starts, ends, B, H, W):
    """The (nw,B,H,W) grids of the windows [starts[w], ends[w]) of contiguous f32 CUDA arrays, and the device
    (start, end) pairs."""
    nw = len(starts)
    L = _lib.lib()
    dev = xs.device
    with torch.cuda.device(dev):
        pairs = torch.tensor(np.stack((np.asarray(starts, dtype=np.int64), np.asarray(ends, dtype=np.int64)), 1).reshape(-1),
                             dtype=torch.int64, device=dev)
        out = torch.empty((nw, B, H, W), dtype=torch.float32, device=dev)
        oob = _lib.oob_counter(dev)
        total = int(np.sum(np.asarray(ends) - np.asarray(starts)))
        _lib.check(L.evk_voxel_windows_f32(_lib.ptr(xs), _lib.ptr(ys), _lib.ptr(ts), _lib.ptr(ps), _lib.ptr(pairs), nw, total,
                                           B, H, W, _lib.WINDOW_PAIRS, _lib.ptr(out), _lib.ptr(oob), _lib.stream()))
        E.raise_if_oob(oob, "voxel grid", (B, H, W))
    return out, pairs


def voxel_grids_fixed_n_torch(xs, ys, ts, ps, B, n, sensor_size=(180, 240), temporal_bilinear=True):
    """List of voxel grids of n events each; drop-in for voxel_grid.py:37-57 (windows
    range(0, len(xs)-n, n)).  CUDA float32 inputs: every window in one kernel launch."""
    starts = list(range(0, len(xs) - n, n))
    if temporal_bilinear:
        grids = _batched_windows(xs, ys, ts, ps, starts, [i + n for i in starts], B, sensor_size)
        if grids is not None:
            return grids
    return [events_to_voxel_torch(xs[i:i + n], ys[i:i + n], ts[i:i + n], ps[i:i + n], B,
                                  sensor_size=sensor_size, temporal_bilinear=temporal_bilinear)
            for i in starts]


def voxel_grids_fixed_t_torch(xs, ys, ts, ps, B, t, sensor_size=(180, 240), temporal_bilinear=True):
    """List of voxel grids of temporal width t; drop-in for voxel_grid.py:59-80.  CUDA float32
    inputs: every window in one kernel launch."""
    np_ts = ts.detach().cpu().numpy()
    t_starts = np.arange(ts[0].item(), ts[-1].item() - t, t)
    if temporal_bilinear:
        starts = [int(np.searchsorted(np_ts, t0)) for t0 in t_starts]
        ends = [int(np.searchsorted(np_ts, t0 + t)) for t0 in t_starts]
        assert(all(s < e for s, e in zip(starts, ends)))       # voxel_grid.py:108
        grids = _batched_windows(xs, ys, ts, ps, starts, ends, B, sensor_size)
        if grids is not None:
            return grids
    return [events_to_voxel_timesync_torch(xs, ys, ts, ps, B, t_start, t_start + t, np_ts=np_ts,
                                           sensor_size=sensor_size, temporal_bilinear=temporal_bilinear)
            for t_start in t_starts]
