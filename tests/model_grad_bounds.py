"""Per-component rounding bounds of the gradients of the newer motion families -- TEST INFRASTRUCTURE ONLY.

Covers the planar models (affine, homography), the camera rotation and camera motion (all K columns of the C entries,
the focal lengths included), the grid-flow and depth-grid node gradients of both losses, and the segmentation's
parameter and per-event weight gradients.  Every bound has the form

    |kernel - f64 reference| <= gamma(c) * M  +  u * E  (+ u |ref| where the kernel casts an f64 sum to f32)

per window and component, with u the f32 unit roundoff and
  * M = sum over the events of |p| S_e |J_e|: the magnitudes of the terms the backward adds, S_e the sum of the four
    image taps' magnitudes the event reads (Wm for the contrast loss, Am (|tau| + Tm) for the timestamp loss) and |J_e|
    the event's |dx'/dp| + |dy'/dp|.  gamma(c) covers the f32 images and the f32 image-space half of the backward
    (c_img, below) and the terms' own accumulation.
  * E = sum over the events of |p| S_e (eJ_e + |J_e| ex_e): the per-event error of the f32 Jacobian (eJ) and of the f32
    warp position the tap fractions are formed with (ex), both in units of u.  eJ and ex come from `Err`, a running
    first-order error bound of the kernel's f32 evaluation in its order of operations (csrc/evk_cmax.cu model_taps
    :404-525, cam_rotate / cam_project :358-393, depth_grid_grad_kernel :2746-2747; the library builds with
    -fmad=false, so every product and sum is rounded on its own).  A Jacobian that cancels in f32 keeps the error of
    the products that cancelled (the term of |vx| and |X vz| in vx - X vz) while |J| stays its small value.
    tests/test_model_grad_bounds_cpu.py checks eJ and ex against the f32 restatement and the f64 closed forms.
The position errors also move every bilinear weight of the IWE (or of S and C) by up to ex_x + ex_y; that image error is
carried into Wm and Tm through the image `ipos` below.

c_img, from the kernel's accumulation path:
  * k_I, the largest number of f32 taps summed into one pixel (four per event anchored there; the 2x2 blocks fold
    into one pixel), 3 for a tap weight, and 2 (2r + 2) per f32 blur pass (two axes of 2r + 1 taps and a rounded
    weight; the forward blurs G, the backward re-blurs it and stores W_b in f32), and TAIL_OPS for the coefficient
    (g_b 2 (G - mean) / P, exp, T = S / C, tau A + B, which batch_obj_backward_W :2197-2208 forms in f64 from f32 G).
  * the accumulation: the parametric passes sum per thread in f64 (motion_obj_event_kernel :2885-2891, the timestamp
    and segmentation passes alike), so 1 covers the f64 sums of up to 2^29 terms.  The grid passes form each term in
    f32 (tap_slopes, times the splat weight, t and the node weight: NODE_TERM_OPS) and sum the lanes of a warp that
    share a node cell in f32 by warp_key_sum's shuffle tree (:2347-2367), of depth log2(32) = 5 for any number of
    peers; the per-CTA f64 sums and the f64 atomics add nothing at f32 scale, and grid_flow_grad_cast_kernel (:2489)
    rounds the f64 sum to f32: u |ref|."""
import numpy as np

from exact_bounds import U32, gamma
from flow_objective_reference import blur_matrix

f32, f64 = np.float32, np.float64

TAIL_OPS = 12
NODE_TERM_OPS = 10       # f32 tap_slopes (4), tau A + B (2) or the splat weight, t and the node weight (3), one spare
TREE_OPS = 5             # warp_key_sum: a shuffle tree over at most 32 peers


def blur_radius(sigma):
    return int(4 * sigma + 0.5) if sigma > 0 else 0


def image_ops(kI, sigma):
    """c_img: the f32 roundings of the images and of the image-space half of the backward"""
    return kI + 3 + 8 * (blur_radius(sigma) + 1) + TAIL_OPS


class Err:
    """A value (f64) and a first-order bound e on the error of its f32 evaluation in the order written, in units of u:
    |fl32 - exact| <= u e (1 + O(u)).  Every operation is rounded once: a sum or difference adds e_a + e_b + |result|,
    a product e_a |b| + |a| e_b + |result|, a quotient e_a / |b| + |a / b| e_b / |b| + |result|.  An exact input has
    e = 0."""
    __array_priority__ = 100

    def __init__(self, v, e=0.0):
        self.v = np.asarray(v, f64)
        self.e = np.broadcast_to(np.asarray(e, f64), self.v.shape) if self.v.shape else np.asarray(e, f64)

    @staticmethod
    def of(o):
        return o if isinstance(o, Err) else Err(o)

    def __add__(self, o):
        o = Err.of(o)
        v = self.v + o.v
        return Err(v, self.e + o.e + np.abs(v))

    __radd__ = __add__

    def __sub__(self, o):
        o = Err.of(o)
        v = self.v - o.v
        return Err(v, self.e + o.e + np.abs(v))

    def __rsub__(self, o):
        return Err.of(o) - self

    def __mul__(self, o):
        o = Err.of(o)
        v = self.v * o.v
        return Err(v, self.e * np.abs(o.v) + np.abs(self.v) * o.e + np.abs(v))

    __rmul__ = __mul__

    def __truediv__(self, o):
        o = Err.of(o)
        with np.errstate(all="ignore"):
            v = self.v / o.v
            return Err(v, (self.e + np.abs(v) * o.e) / np.abs(o.v) + np.abs(v))

    def __rtruediv__(self, o):
        return Err.of(o) / self

    def __neg__(self):
        return Err(-self.v, self.e)


def rounded(c):
    """a constant the kernel rounds to f32: the exact value, with the rounding as its error"""
    return Err(c, np.abs(np.asarray(c, f64) - np.asarray(c, f32).astype(f64)) / U32)


def _where(m, a, b):
    a, b = Err.of(a), Err.of(b)
    return Err(np.where(m, a.v, b.v), np.where(m, a.e, b.e))


def _num(kind):
    """the arithmetic of one evaluation: f32 (the kernel's), f64, or Err"""
    if kind == "err":
        return Err
    dt = f32 if kind == "f32" else f64
    return lambda a: np.asarray(a, dt) if np.ndim(a) else dt(a)


def _param(kind):
    """a parameter the kernel reads as (float)M.m[k]"""
    return {"f32": lambda a: f32(a), "f64": lambda a: f64(a), "err": rounded}[kind]


def planar_warp_jac(model, x, y, d, prm, centre, kind="f32"):
    """x', y' and the (2, K, n) Jacobian of affine / homography in model_taps' order (evk_cmax.cu :485-513)"""
    n, q_ = _num(kind), _param(kind)
    x, y, d = n(x), n(y), n(d)
    m = [q_(v) for v in prm]
    hx, hy, a11, a12, a21, a22 = m[:6]
    u, v = x - q_(centre[0]), y - q_(centre[1])
    sx, sy = (hx + a11 * u) + a12 * v, (hy + a22 * v) + a21 * u
    mx, my = d * sx, d * sy
    xw, yw = x - mx, y - my
    du, dv = d * u, d * v
    z = 0 * d
    if model == "affine":
        return xw, yw, [[-d, z, -du, -dv, z, z], [z, -d, z, z, -du, -dv]]
    g1, g2 = m[6], m[7]
    nx, ny = u - mx, v - my
    with np.errstate(all="ignore"):
        q = d * (g1 * u + g2 * v)
        w = 1 - q
        xw = xw + nx * q / w
        yw = yw + ny * q / w
        w2 = w * w
        return xw, yw, [[-d / w, z, -du / w, -dv / w, z, z, nx * du / w2, nx * dv / w2],
                        [z, -d / w, z, z, -du / w, -dv / w, ny * du / w2, ny * dv / w2]]


SERIES = (1 / 6, 1 / 120, 1 / 5040, 1 / 362880)


def _rot_consts(p2, kind):
    """phi, sin and cos of phi / 2, A, B and C of cam_rotate / model_taps (:366-371, :455-457)"""
    if kind == "err":
        with np.errstate(all="ignore"):
            phi_v = np.sqrt(p2.v)
            phi = Err(phi_v, np.where(phi_v > 0, p2.e / (2 * phi_v), 0.0) + phi_v)       # sqrtf: correctly rounded
            half = Err(0.5 * phi.v, 0.5 * phi.e)                                          # exact
            # sincospif(half * f32(1/pi)): the argument's error (the rounded 1/pi and the product) through the
            # derivative pi cos, pi sin, then at most one ulp (2 u |v|) of the function
            c_pi = f64(f32(1 / np.pi))
            ang_v = half.v * c_pi
            e_ang = half.e * c_pi + half.v * abs(c_pi - 1 / np.pi) / U32 + np.abs(ang_v)
            sh_v, ch_v = np.sin(half.v), np.cos(half.v)
            sh = Err(sh_v, np.pi * np.abs(ch_v) * e_ang + 2 * np.abs(sh_v))
            ch = Err(ch_v, np.pi * np.abs(sh_v) * e_ang + 2 * np.abs(ch_v))
            r = _where(phi.v > 0, sh / _where(phi.v > 0, half, 1.0), Err(1.0))
            A, B = r * ch, 0.5 * (r * r)
            s0, s1, s2, s3 = (rounded(a) for a in SERIES)
            # the series' first omitted term is under 1e-10 below phi = 0.5
            series = s0 - p2 * (s1 - p2 * (s2 - p2 * s3)) + Err(0.0, 1e-10 / U32)
            C = _where(phi.v < 0.5, series, (phi - 2 * (sh * ch)) / (p2 * phi))
        return phi, sh, ch, A, B, C
    dt = f32 if kind == "f32" else f64
    with np.errstate(all="ignore"):
        phi = np.sqrt(p2).astype(dt)
        half = (dt(0.5) * phi).astype(dt)
        ang = (half * dt(0.318309886183790671)).astype(dt).astype(f64)
        sh, ch = np.sin(np.pi * ang).astype(dt), np.cos(np.pi * ang).astype(dt)       # sincospif: within an ulp
        r = np.where(phi > 0, sh / np.where(phi > 0, half, dt(1)), dt(1)).astype(dt)
        A, B = (r * ch).astype(dt), (dt(0.5) * (r * r)).astype(dt)
        series = dt(SERIES[0]) - p2 * (dt(SERIES[1]) - p2 * (dt(SERIES[2]) - p2 * dt(SERIES[3])))
        C = np.where(phi < dt(0.5), series, (phi - dt(2) * (sh * ch)) / (p2 * phi)).astype(dt)
    return phi, sh, ch, A, B, C


def camera_warp_jac(x, y, d, omega, intr, v=None, rho=None, kind="f32", depth_only=False):
    """x', y' and the Jacobian of the camera rotation (v None: (2, 5, n) in (w, fx, fy)) or camera motion ((2, 8, n) in
    (w, v, fx, fy)) in cam_rotate / cam_project / model_taps' order (:358-393, :436-484); depth_only: instead the
    (2, 1, n) dx'/drho, dy'/drho of depth_grid_grad_kernel (:2746-2747).  rho: the f32 inverse depth the kernel warps
    with (an exact input)."""
    n, q_ = _num(kind), _param(kind)
    x, y, d = n(x), n(y), n(d)
    fx, fy, cx, cy = (q_(a) for a in intr)
    wx, wy, wz = (q_(a) for a in omega)
    with np.errstate(all="ignore"):
        bx, by = (x - cx) / fx, (y - cy) / fy
        tx, ty, tz = d * wx, d * wy, d * wz
        p2 = (tx * tx + ty * ty) + tz * tz
        phi, sh, ch, A, B, C = _rot_consts(p2, kind)
        c0, c1, c2 = ty - tz * by, tz * bx - tx, tx * by - ty * bx
        e0, e1, e2 = ty * c2 - tz * c1, tz * c0 - tx * c2, tx * c1 - ty * c0
        Ux, Uy, Uz = (bx + A * c0) + B * e0, (by + A * c1) + B * e1, (1 + A * c2) + B * e2
        Px, Py, Pz = Ux, Uy, Uz
        if v is not None:
            vx, vy, vz = (q_(a) for a in v)
            s = n(rho) * d
            Px, Py, Pz = Ux + s * vx, Uy + s * vy, Uz + s * vz
        iz = 1 / Pz
        X, Y = Px * iz, Py * iz
        xw, yw = cx + fx * X, cy + fy * Y
        if depth_only:
            di = d * iz
            return xw, yw, [[(di * fx) * (vx - X * vz)], [(di * fy) * (vy - Y * vz)]]

        def jlt(w0, w1, w2, sc):
            k0, k1, k2 = ty * w2 - tz * w1, tz * w0 - tx * w2, tx * w1 - ty * w0
            q = C * ((tx * w0 + ty * w1) + tz * w2)
            return [sc * ((A * w0 - B * k0) + q * tx), sc * ((A * w1 - B * k1) + q * ty), sc * ((A * w2 - B * k2) + q * tz)]

        z = 0 * d
        if v is not None:
            Qx, Qy, Qz = Ux * iz, Uy * iz, Uz * iz
            jx = jlt(X * Qy, -(Qz + X * Qx), Qy, -(d * fx))
            jy = jlt(Qz + Y * Qy, -(Y * Qx), -Qx, -(d * fy))
            sx, sy = (s * fx) * iz, (s * fy) * iz
            jx += [sx, z, -(sx * X)]
            jy += [z, sy, -(sy * Y)]
        else:
            jx = jlt(X * Y, -(1 + X * X), Y, -(d * fx))
            jy = jlt(1 + Y * Y, -(X * Y), -X, -(d * fy))
        rxx, rxy, rxz = 1 - B * (ty * ty + tz * tz), A * tz + B * (tx * ty), B * (tx * tz) - A * ty
        ryx, ryy, ryz = B * (tx * ty) - A * tz, 1 - B * (tx * tx + tz * tz), A * tx + B * (ty * tz)
        ux, uy = bx * iz, by * iz
        jx += [X - ux * (rxx - X * rxz), -(uy * (fx / fy)) * (ryx - X * ryz)]
        jy += [-(ux * (fy / fx)) * (rxy - Y * rxz), Y - uy * (ryy - Y * ryz)]
    return xw, yw, [jx, jy]


def stack(rows, kind):
    """a kernel-order result (lists of rows) as an f64 array: values (kind f32 / f64 / err) or error bounds (kind "e")"""
    def get(r):
        if isinstance(r, Err):
            return r.e if kind == "e" else r.v
        return np.asarray(r, f64)
    shape = np.shape(get(rows[0][0]))
    return np.array([[np.broadcast_to(get(r), shape) for r in row] for row in rows])


# ---- image magnitudes -----------------------------------------------------------------------------------------------

def count_image(px, py, w, Hc, Wc):
    """|w| at all four taps of every event anchored at (px, py)"""
    img = np.zeros((Hc, Wc))
    for oy in (0, 1):
        for ox in (0, 1):
            np.add.at(img, (py + oy, px + ox), np.abs(w))
    return img


def taps_of(img, px, py):
    """the sum of the four taps of img at every event"""
    return img[py, px] + img[py, px + 1] + img[py + 1, px] + img[py + 1, px + 1]


def anchored(px, py, Wc):
    """k_I: four taps per event anchored at the busiest pixel (the 2x2 blocks fold into one pixel)"""
    return 4 * int(np.bincount(py * Wc + px).max()) if px.size else 0


def contrast_W_mag(iwe, cnt4, ipos, c_img, sigma, name, param, g):
    """Wm >= |W_b| and the scale of its error: blur(|g_b| Cm), Cm the magnitude of df/dG with the error of G.  G's
    error is at most u (c_img blur(cnt4) + blur(ipos)), ipos the weight changes the position errors cause (in units of
    u), so Ga = blur(cnt4) + blur(ipos) / c_img times gamma(c_img) covers it."""
    Hc, Wc = iwe.shape
    My, Mx = blur_matrix(Hc, sigma), blur_matrix(Wc, sigma)
    P = Hc * Wc
    G = My @ np.asarray(iwe, f64) @ Mx.T
    Ga = My @ (cnt4 + ipos / c_img) @ Mx.T
    if name in ("variance", "sos"):
        C = 2 * (np.abs(G) + Ga + (abs(G.mean()) + Ga.mean() if name == "variance" else 0)) / P
    elif name == "soe":
        C = np.exp(G) * (1 + Ga) / P
    else:
        C = abs(param) * np.exp(-param * G) * (1 + abs(param) * Ga)
    return My @ (abs(float(g)) * C) @ Mx.T, G, Ga


def timestamp_AB_mag(T, C, cnt4, ipos, c_img, sigma, g):
    """per polarity s: Am, the magnitude of A = dF/dS, and Tm >= |T| plus the scale of T's error: with 0 <= tau <= 1 and
    so |T| <= 1, the f32 sums change T by at most u c_img cnt4 / C and the moved bilinear weights by 2 u ipos / C"""
    Hc, Wc = T.shape[-2:]
    My, Mx = blur_matrix(Hc, sigma), blur_matrix(Wc, sigma)
    out = []
    for s in range(2):
        Cs = np.asarray(C[s], f64)
        Tm = np.abs(np.asarray(T[s], f64)) + (cnt4[s] + 2 * ipos[s] / c_img) / Cs
        Gm = My @ Tm @ Mx.T
        out.append(((My @ (4 * abs(float(g)) * Gm) @ Mx.T) / Cs, Tm))
    return out


# ---- per-family bounds ------------------------------------------------------------------------------------------------

def _window(offsets, b, n):
    lo, hi = max(int(offsets[b]), 0), min(int(offsets[b + 1]), n)
    return lo, max(lo, hi)


def _abs_err(rows):
    """(K, n) |dx'/dp_k| + |dy'/dp_k| and the (K, n) sum of their f32 error bounds"""
    return np.abs(stack(rows, "err")).sum(0), stack(rows, "e").sum(0)


def param_events(family, xb, yb, db, prm, centre, H, W, rb=None):
    """The events of one window the kernel keeps (the decisions of the family's reference), their floors, the (K, n)
    Jacobian |J| and its f32 error eJ, and the f32 error ex of the position (the larger of x' and y'), in units of u"""
    import camera_motion_reference as CM
    import camera_rotation_reference as CR
    import planar_motion_reference as P
    from motion_objective_reference import contributes
    prm = np.asarray(prm, f64)
    if family in ("affine", "homography"):
        xw, yw = P.warp_f32(family, xb, yb, db, prm, centre)
    elif family == "camera_rotation":
        xw, yw = CR.warp(xb, yb, db, prm[:3], (prm[3], prm[4]) + tuple(centre))
    else:
        xw, yw = CM.warp(xb, yb, db, rb, prm[:3], prm[3:6], (prm[6], prm[7]) + tuple(centre))
    k = np.flatnonzero(contributes(xw, yw, H, W))
    px, py = np.floor(xw[k]).astype(np.int64), np.floor(yw[k]).astype(np.int64)
    if family in ("affine", "homography"):
        xe, ye, rows = planar_warp_jac(family, xb[k], yb[k], db[k], prm, centre, "err")
    elif family == "camera_rotation":
        xe, ye, rows = camera_warp_jac(xb[k], yb[k], db[k], prm[:3], (prm[3], prm[4]) + tuple(centre), kind="err")
    else:
        xe, ye, rows = camera_warp_jac(xb[k], yb[k], db[k], prm[:3], (prm[6], prm[7]) + tuple(centre), v=prm[3:6],
                                       rho=rb[k], kind="err")
    J, eJ = _abs_err(rows)
    return k, px, py, J, eJ, np.maximum(xe.e, ye.e)


def param_contrast_bound(family, x, y, d, p, offsets, rows, sigma, name, param, g, iwe, centre, img_size, rho=None):
    """(M, c, E), each (B, K): the bound gamma(c) M + u E of the contrast gradient's every component.  rows: (B, K) rows
    of the C entries; iwe: the reference IWEs; g: the incoming gradient per window."""
    H, W = img_size
    B, K = np.shape(rows)
    M, c, E = np.zeros((B, K)), np.zeros((B, K)), np.zeros((B, K))
    for b in range(B):
        lo, hi = _window(offsets, b, x.shape[0])
        sl = slice(lo, hi)
        k, px, py, J, eJ, ex = param_events(family, x[sl], y[sl], d[sl], rows[b], centre, H, W,
                                            None if rho is None else rho[sl])
        w = np.abs(p[sl][k]).astype(f64)
        c[b] = image_ops(anchored(px, py, W + 1), sigma) + 1
        Wm, _, _ = contrast_W_mag(iwe[b], count_image(px, py, w, H + 1, W + 1), count_image(px, py, 2 * ex * w, H + 1, W + 1),
                                  c[b, 0], sigma, name, param, g[b])
        S = w * taps_of(Wm, px, py)
        M[b] = J @ S
        E[b] = (eJ + J * ex) @ S
    return M, c, E


def _timestamp_taps(px, py, pk, uk, ex, T, C, sigma, g, H, W, c_img):
    """per event the tap magnitude sum_4 Am (|tau| + Tm) of its polarity's images"""
    sels = (pk > 0, pk <= 0)
    cnt = np.array([count_image(px[s], py[s], np.ones(int(s.sum())), H + 1, W + 1) for s in sels])
    ipos = np.array([count_image(px[s], py[s], 2 * ex[s], H + 1, W + 1) for s in sels])
    S = np.zeros(px.size)
    for (Am, Tm), sel in zip(timestamp_AB_mag(T, C, cnt, ipos, c_img, sigma, g), sels):
        qx, qy = px[sel], py[sel]
        S[sel] = sum(Am[qy + oy, qx + ox] * (uk[sel] + Tm[qy + oy, qx + ox]) for oy in (0, 1) for ox in (0, 1))
    return S


def _ts_kI(px, py, pk, W):
    return max(anchored(px[s], py[s], W + 1) for s in (pk > 0, pk <= 0))


def param_timestamp_bound(family, x, y, d, tau, p, offsets, rows, sigma, g, T, C, centre, img_size, rho=None):
    """(M, c, E) of the timestamp gradient: per tap of the event's polarity the term (tau A + B) times the Jacobian"""
    H, W = img_size
    B, K = np.shape(rows)
    M, c, E = np.zeros((B, K)), np.zeros((B, K)), np.zeros((B, K))
    for b in range(B):
        lo, hi = _window(offsets, b, x.shape[0])
        sl = slice(lo, hi)
        k, px, py, J, eJ, ex = param_events(family, x[sl], y[sl], d[sl], rows[b], centre, H, W,
                                            None if rho is None else rho[sl])
        pk, uk = p[sl][k], np.abs(tau[sl][k]).astype(f64)
        c[b] = image_ops(_ts_kI(px, py, pk, W), sigma) + 1
        S = _timestamp_taps(px, py, pk, uk, ex, T[b], C[b], sigma, g[b], H, W, c[b, 0])
        M[b] = J @ S
        E[b] = (eJ + J * ex) @ S
    return M, c, E


def segmentation_bound(family, x, y, d, p, w, offsets, rows, sigma, g, iwe, centre, img_size):
    """(M, c, E) (B, Mo, K) of the parameter gradient and (Mw, cw, Ew) (n, Mo) of the per-event weight gradient of the
    variance segmentation loss (motion_seg_grad_kernel :3056-3103): a weight-gradient entry is the single f64 term
    p (bilinear gather of W_bm + c0) at the f32 tap fractions, cast to f32 (add u |ref|)"""
    H, W = img_size
    B, Mo, K = np.shape(rows)
    n = x.shape[0]
    P = (H + 1) * (W + 1)
    M, c, E = np.zeros((B, Mo, K)), np.zeros((B, Mo, K)), np.zeros((B, Mo, K))
    Mw, cw, Ew = np.zeros((n, Mo)), np.zeros((n, Mo)), np.zeros((n, Mo))
    for b in range(B):
        lo, hi = _window(offsets, b, n)
        sl = slice(lo, hi)
        for m in range(Mo):
            k, px, py, J, eJ, ex = param_events(family, x[sl], y[sl], d[sl], rows[b][m], centre, H, W)
            wt = np.abs(p[sl][k].astype(f64) * w[sl][k, m])
            kI = anchored(px, py, W + 1)
            c_img = image_ops(kI, sigma)
            Wm, G, Ga = contrast_W_mag(iwe[b][m], count_image(px, py, wt, H + 1, W + 1),
                                       count_image(px, py, 2 * ex * wt, H + 1, W + 1), c_img, sigma, "variance", 0.0,
                                       g[b][m])
            S = taps_of(Wm, px, py)
            M[b, m] = J @ (wt * S)
            E[b, m] = (eJ + J * ex) @ (wt * S)
            c[b, m] = c_img + 1
            c0 = 2 * abs(float(g[b][m])) * (abs(G.sum()) + Ga.sum()) / P ** 2
            pa = np.abs(p[sl][k]).astype(f64)
            Mw[lo + k, m] = pa * (S + c0)
            cw[lo + k, m] = c_img + 4
            Ew[lo + k, m] = pa * ex * S          # the tap fractions' error times the slope of the gather
    return M, c, E, Mw, cw, Ew


def grid_flow_bound(loss, x, y, d, p, offsets, grids, H, W, sigma, g, imgs, name="variance", param=3.0, tau=None):
    """(M, c, E) (B, 2, gh, gw) of the grid-flow node gradient; loss "contrast" (imgs: IWEs) or "timestamp" (imgs:
    (T, C)).  The Jacobian dx'/du = dy'/dv = d is exact; the position x + u d carries the error of node_flow's f32
    interpolation (four products and four sums, at most 4 sum_4 |q w|), of the product by d and of the sum."""
    import flow_objective_reference as FR
    import grid_flow_reference as GR
    B, _, gh, gw = np.shape(grids)
    M, c, E = np.zeros((B, 2, gh, gw)), np.zeros((B, 2, gh, gw)), np.zeros((B, 2, gh, gw))
    for b in range(B):
        lo, hi = _window(offsets, b, x.shape[0])
        xb, yb, db, pb = x[lo:hi], y[lo:hi], d[lo:hi], p[lo:hi]
        gb = np.asarray(grids[b], f32)
        u32, v32 = GR.event_flow_f32(xb, yb, gb, H, W)
        with np.errstate(all="ignore"):
            xw, yw = (xb + u32 * db).astype(f32), (yb + v32 * db).astype(f32)
        keep, _ = FR.keep_mask(xw, yw, H, W)
        if tau is not None:
            keep &= (pb > 0) | (pb <= 0)                     # a NaN polarity is in neither image
        k = np.flatnonzero(keep)
        if not k.size:
            continue
        rows_, cols, wn, _ = GR.node_taps(xb[k], yb[k], gh, gw, H, W)
        wn = wn.astype(f64)
        px, py = np.floor(xw[k]).astype(np.int64), np.floor(yw[k]).astype(np.int64)
        dk = np.abs(db[k]).astype(f64)
        ex = np.zeros(k.size)
        for ch, (pos, flow) in enumerate(((xw, u32), (yw, v32))):
            eu = 4 * (np.abs(gb[ch][rows_, cols]) * wn).sum(1)
            ex = np.maximum(ex, eu * dk + np.abs(flow[k].astype(f64)) * dk + np.abs(pos[k].astype(f64)))
        if loss == "contrast":
            wt = np.abs(pb[k]).astype(f64)
            kI = anchored(px, py, W + 1)
            c_img = image_ops(kI, sigma)
            Wm, _, _ = contrast_W_mag(imgs[b], count_image(px, py, wt, H + 1, W + 1),
                                      count_image(px, py, 2 * ex * wt, H + 1, W + 1), c_img, sigma, name, param, g[b])
            S = wt * taps_of(Wm, px, py)
        else:
            T, C = imgs
            kI = _ts_kI(px, py, pb[k], W)
            c_img = image_ops(kI, sigma)
            S = _timestamp_taps(px, py, pb[k], np.abs(tau[lo:hi][k]).astype(f64), ex, T[b], C[b], sigma, g[b], H, W,
                                c_img)
        t = S * dk
        for q in range(4):
            np.add.at(M[b, 0], (rows_[:, q], cols[:, q]), t * wn[:, q])
            np.add.at(E[b, 0], (rows_[:, q], cols[:, q]), t * ex * wn[:, q])
        M[b, 1], E[b, 1] = M[b, 0], E[b, 0]
        c[b] = c_img + NODE_TERM_OPS + TREE_OPS
    return M, c, E


def depth_grid_bound(loss, x, y, d, p, offsets, grids, motion, intr, sigma, g, imgs, img_size, name="variance",
                     param=3.0, tau=None):
    """(M, c, E) (B, gh, gw) of the depth-grid node gradient; per event the node weight times |p| S_e times
    |dx'/drho| + |dy'/drho| (and their f32 errors).  The reference warps at the kernel's f32 rho, so rho is an exact
    input of the warp and of dx'/drho."""
    import camera_motion_reference as CM
    from depth_grid_reference import event_rho_f32
    from grid_flow_reference import node_taps
    from motion_objective_reference import contributes
    H, W = img_size
    B, gh, gw = np.shape(grids)
    motion = np.asarray(motion, f64).reshape(B, 6)
    M, c, E = np.zeros((B, gh, gw)), np.zeros((B, gh, gw)), np.zeros((B, gh, gw))
    for b in range(B):
        lo, hi = _window(offsets, b, x.shape[0])
        xb, yb, db, pb = x[lo:hi], y[lo:hi], d[lo:hi], p[lo:hi]
        gb = np.asarray(grids[b], f32)
        r32 = event_rho_f32(xb, yb, gb, H, W)
        xw, yw = CM.warp(xb, yb, db, r32, motion[b, :3], motion[b, 3:], intr)
        keep = contributes(xw, yw, H, W)
        if tau is not None:
            keep &= (pb > 0) | (pb <= 0)
        k = np.flatnonzero(keep)
        if not k.size:
            continue
        rows_, cols, wn, _ = node_taps(xb[k], yb[k], gh, gw, H, W)
        wn = wn.astype(f64)
        xe, ye, Jr = camera_warp_jac(xb[k], yb[k], db[k], motion[b, :3], intr, v=motion[b, 3:], rho=r32[k], kind="err",
                                     depth_only=True)
        J, eJ = (a[0] for a in _abs_err(Jr))
        ex = np.maximum(xe.e, ye.e)
        px, py = np.floor(xw[k]).astype(np.int64), np.floor(yw[k]).astype(np.int64)
        if loss == "contrast":
            wt = np.abs(pb[k]).astype(f64)
            c_img = image_ops(anchored(px, py, W + 1), sigma)
            Wm, _, _ = contrast_W_mag(imgs[b], count_image(px, py, wt, H + 1, W + 1),
                                      count_image(px, py, 2 * ex * wt, H + 1, W + 1), c_img, sigma, name, param, g[b])
            S = wt * taps_of(Wm, px, py)
        else:
            T, C = imgs
            c_img = image_ops(_ts_kI(px, py, pb[k], W), sigma)
            S = _timestamp_taps(px, py, pb[k], np.abs(tau[lo:hi][k]).astype(f64), ex, T[b], C[b], sigma, g[b], H, W,
                                c_img)
        for q in range(4):
            np.add.at(M[b], (rows_[:, q], cols[:, q]), S * J * wn[:, q])
            np.add.at(E[b], (rows_[:, q], cols[:, q]), S * (eJ + J * ex) * wn[:, q])
        c[b] = c_img + NODE_TERM_OPS + TREE_OPS
    return M, c, E


def bound(M, c, E, ref=None):
    """gamma(c) M + u E, plus u |ref| for a gradient the kernel casts from f64 to f32"""
    out = gamma(c) * M + U32 * E
    return out if ref is None else out + U32 * np.abs(ref)


def check(got, ref, M, c, E, what, cast=False):
    """every component within its bound; returns the largest err / bound (0 where both are zero)"""
    got, ref = np.asarray(got, f64), np.asarray(ref, f64)
    bnd = bound(M, c, E, ref if cast else None)
    err = np.abs(got - ref)
    bad = err > bnd
    assert not bad.any(), "%s: %d components outside their bound, e.g. %s: got %r ref %r bound %r" % (
        what, int(bad.sum()), np.argwhere(bad)[:3].tolist(), got[bad][:3].tolist(), ref[bad][:3].tolist(),
        bnd[bad][:3].tolist())
    with np.errstate(all="ignore"):
        r = np.where(bnd > 0, err / bnd, 0.0)
    return float(r.max()) if r.size else 0.0
