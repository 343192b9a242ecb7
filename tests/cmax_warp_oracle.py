"""Oracle of the rotation / 4-DoF contrast-maximisation models (test infrastructure only).

`image_drv` is a sequential restatement of events_to_image_drv (image.py:179-217) for a K-row Jacobian:
the f64 -> f32 casts, the clip mask, the IWE splat (image.py:199-207) and, per channel, the derivative
splat of interpolate_to_derivative_img (image.py:131-135) with d_img sized by the Jacobian.  Every tap is
added in f32 one after the other in event order (np.add.at is unbuffered), with the arithmetic of
oracle/evk_oracle.c's evo_iwe_linvel, so at K = 2 with linvel's Jacobians it reproduces that oracle's
d_iwe bit for bit.  `objective_of_images` is oracle.evk_oracle.objective_of_images for a K-channel stack:
the 3-D blur of the reference (objectives.py:253) at K = 2, a 2-D blur per channel otherwise.
`cmax_objective_warp` takes the model's own Python warp() as the definition of the warp.
"""
import numpy as np

from oracle import evk_oracle as O

SENSOR = (180, 240)


def image_drv(xw, yw, pw, jx=None, jy=None, sensor_size=SENSOR):
    """(iwe (H+1,W+1) f32, d_iwe (K,H+1,W+1) f32 or None, out-of-canvas count) of masked f64 events"""
    Hc, Wc = sensor_size[0] + 1, sensor_size[1] + 1
    xf, yf, pf = (np.asarray(a, np.float64).astype(np.float32) for a in (xw, yw, pw))
    clipx, clipy = np.float32(Wc - 1), np.float32(Hc - 1)
    one = np.float32(1.0)
    with np.errstate(invalid="ignore", over="ignore"):
        m2 = np.where(xf >= clipx, np.float32(0), one) * np.where(yf >= clipy, np.float32(0), one)
        pxf, pyf = np.floor(xf), np.floor(yf)
        dx, dy = xf - pxf, yf - pyf
        px, py = pxf * m2, pyf * m2
        finite = np.isfinite(px) & np.isfinite(py) & (np.abs(px) < 2 ** 40) & (np.abs(py) < 2 ** 40)
        px = np.where(finite, px, 0).astype(np.int64)
        py = np.where(finite, py, 0).astype(np.int64)

    def wrap(i, n):
        i = np.where(i < 0, i + n, i)
        return i, (i >= 0) & (i < n)
    x0, okx0 = wrap(px, Wc)
    x1, okx1 = wrap(px + 1, Wc)
    y0, oky0 = wrap(py, Hc)
    y1, oky1 = wrap(py + 1, Hc)
    ok = finite & okx0 & okx1 & oky0 & oky1
    oob = int((~ok).sum())
    x0, x1, y0, y1, dx, dy, m2, pf = (a[ok] for a in (x0, x1, y0, y1, dx, dy, m2, pf))
    w = pf * m2
    ox, oy = one - dx, one - dy
    idx = np.stack((y0 * Wc + x0, y0 * Wc + x1, y1 * Wc + x0, y1 * Wc + x1), axis=1).reshape(-1)
    iwe = np.zeros(Hc * Wc, np.float32)
    np.add.at(iwe, idx, np.stack(((w * ox) * oy, (w * dx) * oy, (w * ox) * dy, (w * dx) * dy), axis=1).reshape(-1))
    if jx is None:
        return iwe.reshape(Hc, Wc), None, oob
    jxf, jyf = (np.asarray(a, np.float64).astype(np.float32)[:, ok] for a in (jx, jy))
    K = jxf.shape[0]
    d = np.zeros((K, Hc * Wc), np.float32)
    for k in range(K):
        w1, w2 = jxf[k] * w, jyf[k] * w            # image.py:211-212
        taps = np.stack((w1 * (-oy) + w2 * (-ox), w1 * oy + w2 * (-dx), w1 * (-dy) + w2 * ox, w1 * dy + w2 * dx), axis=1)
        np.add.at(d[k], idx, taps.reshape(-1))
    return iwe.reshape(Hc, Wc), d.reshape(K, Hc, Wc), oob


def iwe_warp(warp, params, xs, ys, ts, ps, img_size=SENSOR, compute_gradient=False, use_polarity=True, t_ref=None):
    """get_iwe (objectives.py:184-192) with the model's warp(): (iwe, d_iwe or None, out-of-canvas count)"""
    xs, ys, ts, ps = (np.asarray(a, np.float64) for a in (xs, ys, ts, ps))
    if not use_polarity:
        ps = np.abs(ps)
    xw, yw, jx, jy = warp.warp(xs, ys, ts, ps, ts[-1] if t_ref is None else t_ref, params, compute_grad=compute_gradient)
    mask = O.bounds_mask(xw, yw, 0, img_size[1], 0, img_size[0])
    with np.errstate(invalid="ignore"):
        xw, yw, ps = xw * mask, yw * mask, ps * mask
        if compute_gradient:
            jx, jy = jx * mask, jy * mask
    return image_drv(xw, yw, ps, jx, jy) if compute_gradient else image_drv(xw, yw, ps)


def objective_of_images(name, iwe, d_iwe=None, blur_sigma=None, param=None):
    """(f, g[K] or None) of a precomputed image and a K-channel derivative stack"""
    f = objective_f(name, iwe, blur_sigma, param)
    if d_iwe is None:
        return f, None
    if np.asarray(d_iwe).shape[0] == 2:
        if name == "variance":
            return f, O.variance_g(iwe, d_iwe, 1.0 if blur_sigma is None else blur_sigma)
        return O.objective_of_images(name, iwe, d_iwe, blur_sigma, param)
    if name in ("moa", "r1"):
        return f, None
    _, default_blur, default_param = O.OBJECTIVE_DEFAULTS[name]
    sigma = default_blur if blur_sigma is None else blur_sigma
    prm = default_param if param is None else param
    img = np.asarray(iwe, dtype=np.float32)
    blurred = O.gaussian_filter_f32(img, sigma) if sigma > 0 else img
    stack = [O.gaussian_filter_f32(c, sigma) if sigma > 0 else np.asarray(c, np.float32) for c in np.asarray(d_iwe, np.float32)]
    if name == "variance":
        zero_mean = 2.0 * (img.astype(np.float64) - np.mean(img, dtype=np.float64))
        g = [-np.mean(zero_mean * s) for s in stack]       # objectives.py:256-264
    elif name == "rms":
        g = [-2.0 * np.mean(img * s) for s in stack]
    elif name == "sos":
        g = [-np.mean(s * (img * 2.0)) for s in stack]
    elif name == "soe":
        g = [-np.mean(np.exp(blurred.astype(np.float64)) * s) for s in stack]
    elif name == "isoa":
        g = [-np.sum(s * (blurred > prm).astype(np.float32)) for s in stack]
    else:  # sosa
        g = [-np.sum(s * (-prm * np.exp((-prm * blurred).astype(np.float64)))) for s in stack]
    return float(f), np.array(g, dtype=np.float64)


def objective_f(name, iwe, blur_sigma=None, param=None):
    """f of the variance objective (objectives.py:231-236) or of the others (oracle.evk_oracle)"""
    if name == "variance":
        sigma = 1.0 if blur_sigma is None else blur_sigma
        return O.variance_f(iwe, sigma)
    return O.objective_of_images(name, iwe, None, blur_sigma, param)[0]


def cmax_objective_warp(name, warp, params, xs, ys, ts, ps, img_size=SENSOR, blur_sigma=None, param=None, want_grad=True):
    """(f, g or None, iwe, d_iwe) of objective `name` with the model `warp` on raw events"""
    use_polarity = O.OBJECTIVE_DEFAULTS[name][0] if name != "variance" else True
    iwe, d, oob = iwe_warp(warp, params, xs, ys, ts, ps, img_size, compute_gradient=want_grad, use_polarity=use_polarity)
    if oob:
        raise O.OracleIndexError("%d warped events index outside the IWE canvas" % oob)
    f = objective_f(name, iwe, blur_sigma, param)
    g = objective_of_images(name, iwe, d, blur_sigma, param)[1] if want_grad else None
    return f, g, iwe, d
