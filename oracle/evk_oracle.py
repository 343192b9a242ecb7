"""ctypes front-end to the C oracle (oracle/evk_oracle.c) -- TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
import this module.  The product package (event_utils_b200) never does.
Each function cites the reference lines it restates; see the C file for the arithmetic.

Exact mode (``exact=True`` on the scatter functions): besides the f32 result, the f64 sum of the f32 taps of
every output cell, the f64 sum of their absolute values and the number of non-zero taps, from the same tap code
as the f32 result (evk_oracle.c add_tap).  It returns the out-of-range event count instead of raising.
"""
import collections
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libevk_oracle.so")
_lib = None


def build(force=False):
    src = os.path.join(_HERE, "evk_oracle.c")
    if force or not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(src):
        subprocess.check_call(["make", "-s", "-C", _HERE, "libevk_oracle.so"])
    return _SO


def lib():
    global _lib
    if _lib is None:
        build()
        L = ctypes.CDLL(_SO)
        i64, f32, f64, ci = ctypes.c_int64, ctypes.c_float, ctypes.c_double, ctypes.c_int
        vp = ctypes.c_void_p
        L.evo_voxel_f32.restype = i64
        L.evo_voxel_f32.argtypes = [vp, vp, vp, vp, i64, f32, f32, ci, ci, ci, vp, vp]
        L.evo_voxel_f64.restype = i64
        L.evo_voxel_f64.argtypes = [vp, vp, vp, vp, i64, f64, f64, ci, ci, ci, vp]
        L.evo_image_nearest_f32.restype = i64
        L.evo_image_nearest_f32.argtypes = [vp, vp, vp, i64, ci, ci, ci, f32, f32, vp, vp]
        L.evo_image_bilinear_f32.restype = i64
        L.evo_image_bilinear_f32.argtypes = [vp, vp, vp, i64, ci, ci, ci, f32, f32, vp, vp]
        L.evo_timestamp_image_f32.restype = i64
        L.evo_timestamp_image_f32.argtypes = [vp, vp, vp, vp, i64, f32, f32, ci, ci, ci, ci, f32, f32, vp, vp]
        L.evo_warp_flow_f32.restype = None
        L.evo_warp_flow_f32.argtypes = [vp, vp, vp, i64, vp, ci, ci, f32, vp, vp]
        L.evo_iwe_linvel.restype = i64
        L.evo_iwe_linvel.argtypes = [vp, vp, vp, vp, i64, f64, f64, f64, ci, ci, ci, ci, ci, vp, vp, vp]
        L.evo_gaussian_filter_f32.restype = ci
        L.evo_gaussian_filter_f32.argtypes = [vp, vp, ci, f64]
        L.evo_variance_f.restype = f64
        L.evo_variance_f.argtypes = [vp, ci, ci, f64]
        L.evo_variance_g.restype = None
        L.evo_variance_g.argtypes = [vp, vp, ci, ci, f64, vp]
        L.evo_bounds_mask_f64.restype = None
        L.evo_bounds_mask_f64.argtypes = [vp, vp, i64, f64, f64, f64, f64, vp]
        _lib = L
    return _lib


def _c(a, dt):
    return np.ascontiguousarray(np.asarray(a), dtype=dt)


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


class OracleIndexError(IndexError):
    """The reference would have raised IndexError / ValueError on these inputs."""


# per output cell: f64 sum of the f32 taps, f64 sum of |tap|, number of non-zero taps (arrays shaped like the output)
Exact = collections.namedtuple("Exact", "sum abs cnt")


def _exact_buf(shape, want):
    return np.zeros((3,) + tuple(shape), np.float64) if want else None


def _exact(buf):
    return Exact(buf[0], buf[1], buf[2])


def voxel_f32(xs, ys, ts, ps, B, sensor_size=(180, 240), t0=None, dt=None, exact=False):
    """events_to_voxel_torch, voxel_grid.py:129-153 (f32).  t0/dt default to ts[0], ts[-1]-ts[0].
    exact=True -> (out, Exact, oob count)."""
    x, y, t, p = (_c(a, np.float32) for a in (xs, ys, ts, ps))
    n = x.shape[0]
    H, W = int(sensor_size[0]), int(sensor_size[1])
    if t0 is None:
        t0 = t[0]
    if dt is None:
        dt = np.float32(t[-1]) - np.float32(t[0])
    out = np.zeros((B, H, W), np.float32)
    ex = _exact_buf(out.shape, exact)
    oob = lib().evo_voxel_f32(_p(x), _p(y), _p(t), _p(p), n, float(t0), float(dt), B, H, W, _p(out),
                              _p(ex) if exact else None)
    if exact:
        return out, _exact(ex), oob
    if oob:
        raise OracleIndexError("%d events index outside the grid" % oob)
    return out


def voxel_f64(xs, ys, ts, ps, B, sensor_size=(180, 240), t0=None, dt=None):
    """events_to_voxel (numpy), voxel_grid.py:198-217 + image.py:17,29-44 (f64, int coords)."""
    x, y = _c(xs, np.int64), _c(ys, np.int64)
    t, p = _c(ts, np.float64), _c(ps, np.float64)
    H, W = int(sensor_size[0]), int(sensor_size[1])
    if t0 is None:
        t0 = t[0]
    if dt is None:
        dt = t[-1] - t[0]
    out = np.zeros((B, H, W), np.float64)
    bad = lib().evo_voxel_f64(_p(x), _p(y), _p(t), _p(p), x.shape[0], float(t0), float(dt), B, H, W, _p(out))
    if bad:
        raise OracleIndexError("%d events outside the (H+1,W+1) canvas" % bad)
    return out


def image_torch_f32(xs, ys, ps, sensor_size=(180, 240), clip_out_of_range=True,
                    interpolation=None, padding=True, default=0, exact=False):
    """events_to_image_torch, image.py:46-100 (+102-115): returns the un-cropped canvas.
    exact=True -> (canvas, Exact of the taps (the background not included), oob count)."""
    x, y, p = (_c(a, np.float32) for a in (xs, ys, ps))
    bil = interpolation == "bilinear"
    H, W = int(sensor_size[0]), int(sensor_size[1])
    if bil and padding:
        H, W = H + 1, W + 1
    if interpolation is None and padding is False:
        clipx, clipy = W, H
    else:
        clipx, clipy = W - 1, H - 1
    out = np.full((H, W), default, np.float32)
    ex = _exact_buf(out.shape, exact)
    fn = lib().evo_image_bilinear_f32 if bil else lib().evo_image_nearest_f32
    oob = fn(_p(x), _p(y), _p(p), x.shape[0], H, W, int(bool(clip_out_of_range)),
             float(clipx), float(clipy), _p(out), _p(ex) if exact else None)
    if exact:
        return out, _exact(ex), oob
    if oob:
        raise OracleIndexError("%d events index outside the image" % oob)
    return out


def timestamp_image_f32(xs, ys, ts, ps, sensor_size=(180, 240), clip_out_of_range=True, interpolation='bilinear',
                        padding=True, timestamp_reverse=False, normalize_timestamps=True, exact=False):
    """events_to_timestamp_image_torch, image.py:286-353 -> (img_pos, img_neg).
    normalize_timestamps=False: the numpy flavour's raw-stamp weights (image.py:261).
    exact=True -> (img_pos, img_neg, Exact of the four accumulations [Tpos, Cpos, Tneg, Cneg] -- the count images
    WITHOUT their initial one, oob count)."""
    x, y, t, p = (_c(np.asarray(a).reshape(-1), np.float32) for a in (xs, ys, ts, ps))
    H, W = int(sensor_size[0]), int(sensor_size[1])
    if padding:
        H, W = H + 1, W + 1
    if interpolation is None and padding is False:
        clipx, clipy = W, H
    else:
        clipx, clipy = W - 1, H - 1
    out = np.zeros((2, H, W), np.float32)
    ex = _exact_buf((4, H, W), exact)
    oob = lib().evo_timestamp_image_f32(_p(x), _p(y), _p(t), _p(p), x.shape[0], float(t[0]), float(t[-1]),
                                        int(bool(timestamp_reverse)) if normalize_timestamps else 2, H, W,
                                        int(bool(clip_out_of_range)),
                                        float(clipx), float(clipy), _p(out), _p(ex) if exact else None)
    if exact:
        return out[0], out[1], _exact(ex), oob
    if oob:
        raise OracleIndexError("%d events index outside the image" % oob)
    return out[0], out[1]


def warp_flow_f32(xs, ys, ts, flow, t0=None):
    """warp_events_flow_torch, optic_flow.py:23-46."""
    x, y, t = (_c(np.asarray(a).reshape(-1), np.float32) for a in (xs, ys, ts))
    f = _c(flow, np.float32)
    f = f.reshape(f.shape[-3:])
    assert f.shape[0] == 2
    if t0 is None:
        t0 = t[-1]
    xw, yw = np.empty_like(x), np.empty_like(y)
    lib().evo_warp_flow_f32(_p(x), _p(y), _p(t), x.shape[0], _p(f), f.shape[1], f.shape[2],
                            float(t0), _p(xw), _p(yw))
    return xw, yw


def iwe_linvel(params, xs, ys, ts, ps, img_size, compute_gradient=False, use_polarity=True,
               sensor_size=(180, 240), t_ref=None, exact=False):
    """get_iwe with linvel_warp, objectives.py:184-192 -> (iwe, d_iwe or None).
    t_ref: reference time of the warp; the reference uses ts[-1] (objectives.py:186), a shard of a
    longer stream passes the stream's last timestamp.
    exact=True -> (iwe, d_iwe or None, Exact of the planes [IWE, dIWE[0], dIWE[1]], out-of-canvas count)."""
    x, y, t, p = (_c(a, np.float64) for a in (xs, ys, ts, ps))
    Hs, Ws = int(sensor_size[0]), int(sensor_size[1])
    iwe = np.zeros((Hs + 1, Ws + 1), np.float32)
    d = np.zeros((2, Hs + 1, Ws + 1), np.float32) if compute_gradient else None
    ex = _exact_buf((3, Hs + 1, Ws + 1), exact)
    oob = lib().evo_iwe_linvel(_p(x), _p(y), _p(t), _p(p), x.shape[0], float(params[0]),
                               float(params[1]), float(t[-1] if t_ref is None else t_ref), int(img_size[0]), int(img_size[1]),
                               Hs, Ws, int(bool(use_polarity)), _p(iwe),
                               _p(d) if d is not None else None, _p(ex) if exact else None)
    if exact:
        return iwe, d, _exact(ex), oob
    if oob:
        raise OracleIndexError("%d warped events index outside the IWE canvas" % oob)
    return iwe, d


def gaussian_filter_f32(a, sigma):
    """scipy.ndimage.gaussian_filter(a, sigma) for an f32 array of <= 3 dims (all axes)."""
    b = np.array(a, dtype=np.float32, order="C", copy=True)
    shape = (ctypes.c_int * b.ndim)(*b.shape)
    rc = lib().evo_gaussian_filter_f32(_p(b), shape, b.ndim, float(sigma))
    assert rc == 0
    return b


def variance_f(iwe, blur_sigma=1.0):
    """variance_objective.evaluate_function on a precomputed IWE, objectives.py:231-236."""
    a = _c(iwe, np.float32)
    return lib().evo_variance_f(_p(a), a.shape[0], a.shape[1], float(blur_sigma))


def variance_g(iwe, d_iwe, blur_sigma=1.0):
    """variance_objective.evaluate_gradient on precomputed IWE/dIWE, objectives.py:251-264."""
    a, d = _c(iwe, np.float32), _c(d_iwe, np.float32)
    g = np.zeros(2, np.float64)
    lib().evo_variance_g(_p(a), _p(d), a.shape[0], a.shape[1], float(blur_sigma), _p(g))
    return g


def cmax_variance(params, xs, ys, ts, ps, img_size=(180, 240), blur_sigma=1.0, want_grad=True,
                  use_polarity=True):
    """f (and g) of variance_objective with linvel_warp on raw events."""
    iwe, d = iwe_linvel(params, xs, ys, ts, ps, img_size, compute_gradient=want_grad,
                        use_polarity=use_polarity)
    f = variance_f(iwe, blur_sigma)
    g = variance_g(iwe, d, blur_sigma) if want_grad else None
    return f, g


def bounds_mask(xs, ys, x_min, x_max, y_min, y_max):
    """events_bounds_mask, event_util.py:26-27."""
    x, y = _c(xs, np.float64), _c(ys, np.float64)
    m = np.empty_like(x)
    lib().evo_bounds_mask_f64(_p(x), _p(y), x.shape[0], x_min, x_max, y_min, y_max, _p(m))
    return m


def robust_norm_f32(x, low_perc=0, top_perc=95):
    """RobustNorm.__call__, data_augmentation.py:82-130 (numpy restatement: exact order statistics via
    np.partition, f32 clamp / subtract / divide)."""
    a = np.ascontiguousarray(x, dtype=np.float32)
    flat = a.reshape(-1)

    def kth(q):
        k = 1 + round(.01 * float(q) * (flat.size - 1))
        return np.float32(np.partition(flat, k - 1)[k - 1])
    t_max, t_min = kth(top_perc), kth(low_perc)
    if t_max == 0 and t_min == 0:
        return a.copy()
    c = np.clip(a, t_min, t_max)
    return ((c - c.min()) / np.float32(c.max() + np.float32(1e-6))).astype(np.float32)



# ---- the other objective functions, image-space part (objectives.py:266-596) ------------------------
OBJECTIVE_DEFAULTS = {   # name: (use_polarity, default_blur, parameter)
    "variance": (True, 1.0, None), "rms": (True, 1.0, None), "sos": (True, 1.0, None), "soe": (False, 2.5, None),
    "moa": (False, 3.0, None), "isoa": (False, 1.0, 0.5), "sosa": (False, 2.0, 3.0), "r1": (False, 1.0, 3.0),
}


def objective_of_images(name, iwe, d_iwe=None, blur_sigma=None, param=None):
    """f (and g, when d_iwe is given and the objective has a derivative) of a precomputed image of warped
    events -- the part of every evaluate_function / evaluate_gradient after get_iwe:
        rms   :266-307   f = -||G||_2^2 / P (spectral norm),  g_k = -2 mean(I  * G3(D)_k)
        sos   :308-357   f = -mean(G^2),                      g_k = -mean(G3(D)_k * 2 I)
        soe   :358-400   f = -mean(exp G),                    g_k = -mean(exp(G) * G3(D)_k)
        moa   :401-430   f = -max G
        isoa  :431-477   f = +#(G > thresh),                  g_k = -sum([G > thresh] * G3(D)_k)
        sosa  :478-523   f = -sum(exp(-p G)),                 g_k = -sum(-p exp(-p G) * G3(D)_k)
        r1    :560-596   f = -mean(G^2): with last_sosa initialised to 0 the branch `sosa > last_sosa` is always
                         taken and last_sosa never updated, so the product form -sos*sosa is unreachable
    with G = gaussian_filter(I), G3 = gaussian_filter of the (2,H,W) stack (all three axes), I un-blurred.
    Returns (f, g or None)."""
    _, default_blur, default_param = OBJECTIVE_DEFAULTS[name]
    sigma = default_blur if blur_sigma is None else blur_sigma
    prm = default_param if param is None else param
    img = np.asarray(iwe, dtype=np.float32)
    blurred = gaussian_filter_f32(img, sigma) if sigma > 0 else img
    npix = img.shape[0] * img.shape[1]
    if name == "rms":
        f = -(np.linalg.norm(blurred, 2) ** 2) / npix
    elif name == "sos":
        f = -np.mean(blurred * blurred)
    elif name == "soe":
        f = -np.mean(np.exp(blurred.astype(np.float64)))
    elif name == "moa":
        f = -np.max(blurred)
    elif name == "isoa":
        f = int(np.sum(blurred > prm))
    elif name == "sosa":
        f = -np.sum(np.exp(-prm * blurred.astype(np.float64)))
    elif name == "r1":
        f = -np.mean(blurred * blurred)
    else:
        raise KeyError(name)
    if d_iwe is None or name in ("moa", "r1"):
        return float(f), None
    stack = np.asarray(d_iwe, dtype=np.float32)
    stack = gaussian_filter_f32(stack, sigma) if sigma > 0 else stack
    if name == "rms":
        g = [-2.0 * np.mean(img * stack[k]) for k in range(2)]
    elif name == "sos":
        g = [-np.mean(stack[k] * (img * 2.0)) for k in range(2)]
    elif name == "soe":
        g = [-np.mean(np.exp(blurred.astype(np.float64)) * stack[k]) for k in range(2)]
    elif name == "isoa":
        g = [-np.sum(stack[k] * (blurred > prm).astype(np.float32)) for k in range(2)]
    else:  # sosa
        g = [-np.sum(stack[k] * (-prm * np.exp((-prm * blurred).astype(np.float64)))) for k in range(2)]
    return float(f), np.array(g, dtype=np.float64)


def cmax_objective(name, params, xs, ys, ts, ps, img_size=(180, 240), blur_sigma=None, param=None, want_grad=True):
    """Any of the objectives above with linvel_warp on raw events."""
    use_polarity = OBJECTIVE_DEFAULTS[name][0]
    iwe, d = iwe_linvel(params, xs, ys, ts, ps, img_size, compute_gradient=want_grad, use_polarity=use_polarity)
    return objective_of_images(name, iwe, d, blur_sigma, param)
