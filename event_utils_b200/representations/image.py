"""Event-image builders -- drop-in for the reference's lib/representations/image.py
(events_to_image, events_to_image_torch, interpolate_to_image, interpolate_to_derivative_img,
image_to_event_weights, events_to_image_drv).  Kernels: csrc/evk_image.cu.
"""
import numpy as np
import torch

from .. import _lib, config
from . import _events as E


def _canvas_and_clip(sensor_size, interpolation, padding):
    """image.py:64-67 (canvas) and :73-74 (clip thresholds)."""
    if interpolation == 'bilinear' and padding:
        img_size = (sensor_size[0] + 1, sensor_size[1] + 1)
    else:
        img_size = (sensor_size[0], sensor_size[1])
    clipx = img_size[1] if interpolation is None and padding == False else img_size[1] - 1  # noqa: E712
    clipy = img_size[0] if interpolation is None and padding == False else img_size[0] - 1  # noqa: E712
    return (int(img_size[0]), int(img_size[1])), float(clipx), float(clipy)


def _image_device(x, y, p, Himg, Wimg, clipx, clipy, flags, fill, out=None):
    L = _lib.lib()
    dev = x.device
    with torch.cuda.device(dev):
        if out is None:
            out = torch.empty((Himg, Wimg), dtype=torch.float32, device=dev)
        flags |= E.variant_flag()
        ws_bytes = L.evk_image_workspace_bytes(Himg, Wimg, flags)
        ws = _lib.scratch("image_ws", ws_bytes, dev)
        oob = _lib.oob_counter(dev)
        _lib.check(L.evk_image_f32(_lib.ptr(x), _lib.ptr(y), _lib.ptr(p), x.shape[0], Himg, Wimg, clipx, clipy,
                                   flags, float(fill), _lib.ptr(out), _lib.ptr(ws), ws.numel(), _lib.ptr(oob),
                                   _lib.stream()))
        if config.check_index_errors:
            bad = int(oob.item())
            if bad:
                print("Unable to put tensor {} positions into {}: {} events out of range".format(
                    tuple(p.shape), (Himg, Wimg), bad))
                raise IndexError("index out of range in events_to_image")
    return out


def events_to_image_torch(xs, ys, ps,
        device=None, sensor_size=(180, 240), clip_out_of_range=True,
        interpolation=None, padding=True, default=0):
    """
    Event tensor -> image, nearest or bilinear.  Drop-in for image.py:46-100; returns the
    un-cropped canvas ((H+1,W+1) when bilinear and padding).  Quirks kept on purpose:
    with clip_out_of_range the INDEX of a clipped event is zeroed but its weight is not in
    nearest mode (image.py:94-95), negative indices wrap, the default padding=True makes the
    last row/column count as out of range.
    Differentiable like the reference: bilinear w.r.t. xs, ys and ps, nearest w.r.t. ps
    (event_utils_b200.autograd).
    """
    xs_t = E.as_tensor(xs)
    if device is None:
        device = xs_t.device
    device = torch.device(device)
    if E.needs_grad(*((xs, ys, ps) if interpolation == 'bilinear' else (ps,))):
        from ..autograd import EventImage
        return EventImage.apply(xs, ys, ps, (device, sensor_size, clip_out_of_range, interpolation, padding, default))
    dev, (Himg, Wimg), clipx, clipy, flags, x, y, p = _image_inputs(xs, ys, ps, sensor_size, clip_out_of_range,
                                                                    interpolation, padding)
    img = _image_device(x, y, p, Himg, Wimg, clipx, clipy, flags, default)
    return img if img.device == device else img.to(device)


def _image_inputs(xs, ys, ps, sensor_size, clip_out_of_range, interpolation, padding):
    """events_to_image_torch's kernel inputs: compute device, canvas, clip thresholds, flags and f32 x, y, p."""
    xs_t = E.as_tensor(xs)
    dev = E.compute_device(xs, ys, ps)
    (Himg, Wimg), clipx, clipy = _canvas_and_clip(sensor_size, interpolation, padding)
    # image.py:78: integer coordinates fall back to the nearest branch (on the padded canvas)
    bilinear = interpolation == 'bilinear' and xs_t.dtype is not torch.long
    flags = (_lib.BILINEAR if bilinear else 0) | (_lib.CLIP if clip_out_of_range else 0)
    ps_t = E.as_tensor(ps)
    if ps_t.dtype == torch.float64:
        raise RuntimeError("Index put requires the source and destination dtypes match, "
                           "got Float for the destination and Double for the source.")
    if bilinear:
        x = E.to_device(xs_t.reshape(-1), dev).to(torch.float32).contiguous()
        y = E.to_device(E.as_tensor(ys).reshape(-1), dev).to(torch.float32).contiguous()
    else:
        x, y = E.coords_f32(xs, dev), E.coords_f32(ys, dev)
    p = E.weights_f32(ps_t.squeeze() if bilinear else ps_t, dev)
    return dev, (Himg, Wimg), clipx, clipy, flags, x, y, p


def events_to_image(xs, ys, ps, sensor_size=(180, 240), interpolation=None, padding=False, meanval=False, default=0):
    """
    numpy flavour; drop-in for image.py:5-44.  Nearest: integer coordinates scattered on an
    (H+1,W+1) canvas and cropped (float64 result).  bilinear delegates to the torch flavour
    WITHOUT forwarding sensor_size, exactly like image.py:21.
    """
    xs, ys, ps = np.asarray(xs), np.asarray(ys), np.asarray(ps)
    H, W = int(sensor_size[0]), int(sensor_size[1])
    dev = E.compute_device()
    if interpolation == 'bilinear':
        xt, yt, pt = (torch.from_numpy(np.ascontiguousarray(a)).float() for a in (xs, ys, ps))
        img = events_to_image_torch(xt, yt, pt, clip_out_of_range=True, interpolation='bilinear', padding=padding)
        img[img == 0] = default
        img = img.numpy()
        if meanval:
            cnt = events_to_image_torch(xt, yt, torch.ones_like(xt), clip_out_of_range=True, padding=padding).numpy()
    else:
        if not (np.issubdtype(xs.dtype, np.integer) and np.issubdtype(ys.dtype, np.integer)):
            raise TypeError("only int indices permitted")
        with torch.cuda.device(dev):
            x = E.to_device(torch.from_numpy(np.ascontiguousarray(xs).reshape(-1)), dev)
            y = E.to_device(torch.from_numpy(np.ascontiguousarray(ys).reshape(-1)), dev)
            if x.numel() and (int(x.min()) < 0 or int(y.min()) < 0 or int(x.max()) > W or int(y.max()) > H):
                print("Issue with input arrays! minx={}, maxx={}, miny={}, maxy={}, sensor_size={}".format(
                    int(x.min()), int(x.max()), int(y.min()), int(y.max()), (H + 1, W + 1)))
                raise ValueError
            xf, yf = x.to(torch.float32), y.to(torch.float32)
            p = E.to_device(torch.from_numpy(np.ascontiguousarray(ps, dtype=np.float64).reshape(-1)), dev).to(torch.float32)
            img = _image_device(xf, yf, p, H + 1, W + 1, 0.0, 0.0, 0, 0.0).double().cpu().numpy()
            if meanval:
                cnt = _image_device(xf, yf, torch.ones_like(xf), H + 1, W + 1, 0.0, 0.0, 0, 0.0).double().cpu().numpy()
    if meanval:
        img = np.divide(img, cnt, out=np.ones_like(img) * default, where=cnt != 0)
    return img[0:sensor_size[0], 0:sensor_size[1]]


def interpolate_to_image(pxs, pys, dxs, dys, weights, img):
    """
    In-place 4-tap bilinear accumulation at precomputed integer positions / fractions;
    drop-in for image.py:102-115.  img: 2-D float32 tensor (CUDA, or CPU -> round trip).
    """
    L = _lib.lib()
    dev = E.compute_device(img, pxs)
    with torch.cuda.device(dev):
        work = img if img.is_cuda else img.to(dev)
        if not work.is_contiguous() or work.dtype != torch.float32:
            raise RuntimeError("interpolate_to_image: img must be a contiguous float32 tensor")
        px = E.to_device(E.as_tensor(pxs).reshape(-1), dev).long().contiguous()
        py = E.to_device(E.as_tensor(pys).reshape(-1), dev).long().contiguous()
        dx, dy, w = (E.to_device(E.as_tensor(a).reshape(-1), dev).to(torch.float32).contiguous() for a in (dxs, dys, weights))
        oob = _lib.oob_counter(dev)
        _lib.check(L.evk_splat_idx_f32(_lib.ptr(px), _lib.ptr(py), _lib.ptr(dx), _lib.ptr(dy), _lib.ptr(w),
                                       px.shape[0], work.shape[0], work.shape[1], _lib.ptr(work), _lib.ptr(oob),
                                       _lib.stream()))
        E.raise_if_oob(oob, "image", work.shape)
        if work is not img:
            img.copy_(work)
    return img


def interpolate_to_derivative_img(pxs, pys, dxs, dys, d_img, w1, w2):
    """
    In-place Jacobian-weighted bilinear accumulation; drop-in for image.py:117-136.
    d_img: (K,H,W) float32; w1, w2: (K,N).
    """
    L = _lib.lib()
    dev = E.compute_device(d_img, pxs)
    with torch.cuda.device(dev):
        work = d_img if d_img.is_cuda else d_img.to(dev)
        if not work.is_contiguous() or work.dtype != torch.float32:
            raise RuntimeError("interpolate_to_derivative_img: d_img must be a contiguous float32 tensor")
        px = E.to_device(E.as_tensor(pxs).reshape(-1), dev).long().contiguous()
        py = E.to_device(E.as_tensor(pys).reshape(-1), dev).long().contiguous()
        dx, dy = (E.to_device(E.as_tensor(a).reshape(-1), dev).to(torch.float32).contiguous() for a in (dxs, dys))
        K = work.shape[0]
        a1 = E.to_device(E.as_tensor(w1), dev).to(torch.float32).reshape(K, -1).contiguous()
        a2 = E.to_device(E.as_tensor(w2), dev).to(torch.float32).reshape(K, -1).contiguous()
        oob = _lib.oob_counter(dev)
        _lib.check(L.evk_splat_drv_idx_f32(_lib.ptr(px), _lib.ptr(py), _lib.ptr(dx), _lib.ptr(dy), _lib.ptr(a1),
                                           _lib.ptr(a2), K, px.shape[0], work.shape[1], work.shape[2],
                                           _lib.ptr(work), _lib.ptr(oob), _lib.stream()))
        E.raise_if_oob(oob, "derivative image", work.shape)
        if work is not d_img:
            d_img.copy_(work)
    return d_img


def image_to_event_weights(xs, ys, img):
    """
    Reverse bilinear interpolation: the image value at each event; drop-in for image.py:138-160
    (numpy in, numpy float64 out).
    """
    L = _lib.lib()
    xs, ys = np.asarray(xs, dtype=np.float64).reshape(-1), np.asarray(ys, dtype=np.float64).reshape(-1)
    img = np.asarray(img)
    dev = E.compute_device()
    with torch.cuda.device(dev):
        x, y = E.to_device(torch.from_numpy(xs), dev), E.to_device(torch.from_numpy(ys), dev)
        im = E.to_device(torch.from_numpy(np.ascontiguousarray(img, dtype=np.float64)), dev)
        out = torch.empty_like(x)
        oob = _lib.oob_counter(dev)
        _lib.check(L.evk_gather_bilinear_f64(_lib.ptr(x), _lib.ptr(y), x.shape[0], _lib.ptr(im), im.shape[0],
                                             im.shape[1], _lib.ptr(out), _lib.ptr(oob), _lib.stream()))
        E.raise_if_oob(oob, "image", im.shape)
        return out.cpu().numpy()


def _ts_canvas_and_clip(sensor_size, interpolation, padding):
    """image.py:305-312: the canvas of the timestamp images and the clip thresholds."""
    if padding:
        img_size = (int(sensor_size[0]) + 1, int(sensor_size[1]) + 1)
    else:
        img_size = (int(sensor_size[0]), int(sensor_size[1]))
    clipx = img_size[1] if interpolation is None and padding == False else img_size[1] - 1  # noqa: E712
    clipy = img_size[0] if interpolation is None and padding == False else img_size[0] - 1  # noqa: E712
    return img_size, float(clipx), float(clipy)


def _ts_flags(clip_out_of_range, reverse, raw=False):
    return (_lib.CLIP if clip_out_of_range else 0) | (_lib.TS_REVERSE if reverse else 0) | (_lib.TS_RAW if raw else 0)


def _timestamp_images(x, y, t, p, t_first, t_last, sensor_size, clip_out_of_range, interpolation, padding, reverse,
                      raw=False, counts=False):
    """The two timestamp images; with `counts` also the two count images they were divided by (for the backward)."""
    L = _lib.lib()
    dev = x.device
    img_size, clipx, clipy = _ts_canvas_and_clip(sensor_size, interpolation, padding)
    with torch.cuda.device(dev):
        pos = torch.empty(img_size, dtype=torch.float32, device=dev)
        neg = torch.empty(img_size, dtype=torch.float32, device=dev)
        ws = _lib.scratch("tsimg_ws", L.evk_timestamp_image_workspace_bytes(*img_size), dev)
        oob = _lib.oob_counter(dev)
        flags = _ts_flags(clip_out_of_range, reverse, raw)
        if counts:
            cpos, cneg = torch.empty_like(pos), torch.empty_like(neg)
            _lib.check(L.evk_timestamp_image_counts_f32(_lib.ptr(x), _lib.ptr(y), _lib.ptr(t), _lib.ptr(p), x.shape[0],
                                                        t_first, t_last, img_size[0], img_size[1], clipx, clipy, flags,
                                                        _lib.ptr(pos), _lib.ptr(neg), _lib.ptr(cpos), _lib.ptr(cneg),
                                                        _lib.ptr(ws), ws.numel(), _lib.ptr(oob), _lib.stream()))
        else:
            _lib.check(L.evk_timestamp_image_f32(_lib.ptr(x), _lib.ptr(y), _lib.ptr(t), _lib.ptr(p), x.shape[0], t_first, t_last,
                                                 img_size[0], img_size[1], clipx, clipy, flags, _lib.ptr(pos),
                                                 _lib.ptr(neg), _lib.ptr(ws), ws.numel(), _lib.ptr(oob), _lib.stream()))
        E.raise_if_oob(oob, "timestamp image", img_size)
    if counts:
        return pos, neg, cpos, cneg
    return pos, neg


def _timestamp_inputs(xs, ys, ts, ps):
    """events_to_timestamp_image_torch's kernel inputs: compute device, f32 x, y, t, p and (ts[0], ts[-1])."""
    dev = E.compute_device(xs, ys, ts, ps)
    x, y, t, p = (E.to_device(E.as_tensor(a).squeeze().reshape(-1), dev).to(torch.float32).contiguous() for a in (xs, ys, ts, ps))
    fl = torch.stack((t[0], t[-1])).tolist()
    return dev, x, y, t, p, fl


def events_to_timestamp_image_torch(xs, ys, ts, ps,
        device=None, sensor_size=(180, 240), clip_out_of_range=True,
        interpolation='bilinear', padding=True, timestamp_reverse=False):
    """
    Average-timestamp images (Zhu et al. 2019) of the positive and negative events; drop-in for
    image.py:286-353.  Quirks kept: the count images start at one, and a clipped event keeps its
    weight (only its index is zeroed).  Differentiable like the reference w.r.t. xs, ys and ts
    (event_utils_b200.autograd).
    @returns img_pos, img_neg (canvas (H+1,W+1) with padding)
    """
    xs_t = E.as_tensor(xs)
    if device is None:
        device = xs_t.device
    device = torch.device(device)
    if E.needs_grad(xs, ys, ts):
        from ..autograd import TimestampImages
        return TimestampImages.apply(xs, ys, ts, ps, (device, sensor_size, clip_out_of_range, interpolation, padding,
                                                      timestamp_reverse))
    dev, x, y, t, p, fl = _timestamp_inputs(xs, ys, ts, ps)
    pos, neg = _timestamp_images(x, y, t, p, fl[0], fl[1], sensor_size, clip_out_of_range, interpolation, padding,
                                 timestamp_reverse)
    if pos.device != device:
        pos, neg = pos.to(device), neg.to(device)
    return pos, neg


def events_to_timestamp_image(xn, yn, ts, pn,
        device=None, sensor_size=(180, 240), clip_out_of_range=True,
        interpolation='bilinear', padding=True, normalize_timestamps=True):
    """
    numpy flavour; drop-in for image.py:219-284 (numpy in, numpy float32 out).  Timestamps are made
    relative to ts[0] in float64 before the cast to float32, like the reference (:241-243).
    normalize_timestamps=False (:261): the weights are those relative stamps themselves (EVK_TS_RAW).
    """
    dev = E.compute_device()
    ts = np.asarray(ts, dtype=np.float64).reshape(-1)
    rel = ts - ts[0]
    x, y, p = (E.to_device(torch.from_numpy(np.ascontiguousarray(a).reshape(-1)), dev).float().contiguous() for a in (xn, yn, pn))
    t = E.to_device(torch.from_numpy(rel), dev).float().contiguous()
    # the reference divides by (ts[-1] + 1e-6) of the RELATIVE stamps (image.py:261): first = 0
    pos, neg = _timestamp_images(x, y, t, p, 0.0, float(np.float32(rel[-1])), sensor_size, clip_out_of_range,
                                 interpolation, padding, False, raw=not normalize_timestamps)
    return pos.cpu().numpy(), neg.cpu().numpy()


def events_to_image_drv(xn, yn, pn, jacobian_xn, jacobian_yn,
        device=None, sensor_size=(180, 240), clip_out_of_range=True,
        interpolation='bilinear', padding=True, compute_gradient=False):
    """
    Image of warped events and its derivative images from per-event Jacobians; drop-in for
    image.py:162-217 (numpy float64 in -> numpy float32 out, always bilinear like the reference).
    @returns (img (H+1,W+1) f32, d_img (K,H+1,W+1) f32 or None)
    """
    L = _lib.lib()
    dev = E.compute_device()
    if padding:
        img_size = (sensor_size[0] + 1, sensor_size[1] + 1)
    else:
        img_size = (sensor_size[0], sensor_size[1])
    clipx = img_size[1] if interpolation is None and padding == False else img_size[1] - 1  # noqa: E712
    clipy = img_size[0] if interpolation is None and padding == False else img_size[0] - 1  # noqa: E712
    with torch.cuda.device(dev):
        # image.py:179-183: the f64 -> f32 rounding point
        x, y, p = (E.to_device(torch.from_numpy(np.ascontiguousarray(a).reshape(-1)), dev).float().contiguous()
                   for a in (xn, yn, pn))
        img = torch.empty(img_size, dtype=torch.float32, device=dev)
        K, jx, jy, d_img = 0, None, None, None
        if compute_gradient:
            jx = E.to_device(torch.from_numpy(np.ascontiguousarray(jacobian_xn)), dev).float().contiguous()
            jy = E.to_device(torch.from_numpy(np.ascontiguousarray(jacobian_yn)), dev).float().contiguous()
            K = jx.shape[0]
            d_img = torch.empty((K,) + tuple(img_size), dtype=torch.float32, device=dev)
        oob = _lib.oob_counter(dev)
        flags = _lib.CLIP if clip_out_of_range else 0
        _lib.check(L.evk_image_drv_f32(_lib.ptr(x), _lib.ptr(y), _lib.ptr(p), _lib.ptr(jx), _lib.ptr(jy), K,
                                       x.shape[0], img_size[0], img_size[1], float(clipx), float(clipy), flags,
                                       _lib.ptr(img), _lib.ptr(d_img), _lib.ptr(oob), _lib.stream()))
        E.raise_if_oob(oob, "image", img_size)
        return img.cpu().numpy(), (d_img.cpu().numpy() if d_img is not None else None)
