"""Motion models for contrast maximisation -- drop-in for the reference's lib/contrast_max/warps.py
(`warp_function` ABC :6-42, `linvel_warp` :44-61, and the two models it declares with an empty
`warp()`, :63-83, defined here).

An objective from `event_utils_b200.contrast_max.objectives` that is handed one of these models never
calls `warp()`: it recognises the model through `fused_kind` and evaluates warp, bounds mask, image
formation, objective and gradient on the GPU over the device-resident events (csrc/evk_cmax.cu: one
fused pass for linvel, an image pass and a gradient pass for the rotation and 4-DoF models).  `warp()` is still provided, with the reference's semantics, for user code that
calls it directly and for the generic (non-fused) path taken by other `warp_function` subclasses.
"""
from abc import ABC, abstractmethod

import numpy as np


class warp_function(ABC):
    """A parametrised, differentiable motion model that transports events to a reference time.
    `name` identifies the model, `dims` is its number of degrees of freedom (used by the grid
    search drivers, events_cmax.py:282)."""

    fused_kind = None   # set by models the fused kernels implement natively

    def __init__(self, name, dims):
        self.name, self.dims = name, dims
        super().__init__()

    @abstractmethod
    def warp(self, xs, ys, ts, ps, t0, params, compute_grad=False):
        """Transport the events (xs, ys, ts, ps) to time t0 under `params`.
        Returns (xs_warped, ys_warped, jacobian_x, jacobian_y); the Jacobians have shape
        (dims, N) -- d x'/d params and d y'/d params per event -- or are None without
        compute_grad."""


class linvel_warp(warp_function):
    """Global optic flow: every event moves with one image-plane velocity (vx, vy) = params,
        x' = x - (t - t0) vx,      y' = y - (t - t0) vy,
    so d x'/d vx = d y'/d vy = -(t - t0) and the cross terms vanish (reference warps.py:51-61)."""

    fused_kind = "linvel"

    def __init__(self):
        super().__init__('linvel_warp', 2)

    def warp(self, xs, ys, ts, ps, t0, params, compute_grad=False):
        lag = ts - t0
        moved = (xs - lag * params[0], ys - lag * params[1])
        if not compute_grad:
            return moved[0], moved[1], None, None
        nothing = np.zeros_like(lag, dtype=np.float64)
        return moved[0], moved[1], np.stack((-lag, nothing)), np.stack((nothing, -lag))


class pure_rotation_warp(warp_function):
    """Rotation of the image plane about a centre (cx, cy) at angular velocity omega, params = (cx, cy, omega)
    -- the reference's "x,y center of rotation, theta angular velocity" (warps.py:74-83, where warp() is empty).
    With dt = t - t0 and a = omega dt, the warp undoes the rotation during dt:
        u = x - cx,  v = y - cy
        x' = cx + (cos(a) u + sin(a) v),          y' = cy + (cos(a) v - sin(a) u)
        d x'/d(cx, cy, omega) = (1 - cos a, -sin a,  dt (cos(a) v - sin(a) u))
        d y'/d(cx, cy, omega) = (sin a, 1 - cos a, -dt (cos(a) u + sin(a) v))
    f64 numpy in the order written.  dims is 3: the reference registers 4, which contradicts its own three
    parameters (its warp() returns None, so no caller can depend on the 4)."""

    fused_kind = "rotation"

    def __init__(self):
        super().__init__('pure_rotation_warp', 3)

    def model(self, params):
        """the parameter block of the fused GPU evaluation (evk_cmax_warp_objective_*)"""
        return [float(params[0]), float(params[1]), float(params[2])]

    def warp(self, xs, ys, ts, ps, t0, params, compute_grad=False):
        cx, cy, omega = (float(v) for v in params[:3])
        dt = ts - t0
        a = omega * dt
        c, s = np.cos(a), np.sin(a)
        u, v = xs - cx, ys - cy
        rx, ry = c * u + s * v, c * v - s * u
        xw, yw = cx + rx, cy + ry
        if not compute_grad:
            return xw, yw, None, None
        jx = np.stack((1.0 - c, -s, dt * ry))
        jy = np.stack((s, 1.0 - c, -(dt * rx)))
        return xw, yw, jx, jy


class xyztheta_warp(warp_function):
    """4-DoF model of Mitrokhin et al., "Event-based moving object detection and tracking" (the reference's
    warps.py:63-72 leaves warp() empty), in its first-order form: image-plane translation (hx, hy), expansion rate hz
    and in-plane angular velocity theta about a fixed centre, params = (hx, hy, hz, theta).  The default centre is
    the middle of the 180x240 sensor every objective forms its image on (objectives.py:191-192).
        u = x - cx,  v = y - cy
        x' = x - dt ((hx + hz u) - theta v),      y' = y - dt ((hy + hz v) + theta u)
        d x'/d(hx, hy, hz, theta) = (-dt, 0, -dt u,  dt v)
        d y'/d(hx, hy, hz, theta) = (0, -dt, -dt v, -dt u)
    f64 numpy in the order written; with hz = theta = 0 and finite coordinates this is linvel_warp(hx, hy)
    bit for bit (x - dt hx, no fused multiply-add on either side)."""

    fused_kind = "xyztheta"

    def __init__(self, center=(120.0, 90.0)):
        super().__init__('xyztheta_warp', 4)
        self.center = (float(center[0]), float(center[1]))

    def model(self, params):
        """the parameter block of the fused GPU evaluation (evk_cmax_warp_objective_*)"""
        return [float(params[0]), float(params[1]), float(params[2]), float(params[3])] + list(self.center)

    def warp(self, xs, ys, ts, ps, t0, params, compute_grad=False):
        hx, hy, hz, theta = (float(v) for v in params[:4])
        cx, cy = self.center
        dt = ts - t0
        u, v = xs - cx, ys - cy
        xw = xs - dt * ((hx + hz * u) - theta * v)
        yw = ys - dt * ((hy + hz * v) + theta * u)
        if not compute_grad:
            return xw, yw, None, None
        nothing = np.zeros_like(dt, dtype=np.float64)
        jx = np.stack((-dt, nothing, -(dt * u), dt * v))
        jy = np.stack((nothing, -dt, -(dt * v), -(dt * u)))
        return xw, yw, jx, jy


class affine_warp(warp_function):
    """6-DoF affine motion in its first-order form about a fixed centre, params = (hx, hy, a11, a12, a21, a22): the
    image-plane velocity of a point at (u, v) = (x - cx, y - cy) is (hx + a11 u + a12 v, hy + a21 u + a22 v).  It is the
    usual model for tracking an object or a patch that shears or scales unevenly.
        sx = (hx + a11 u) + a12 v,      sy = (hy + a22 v) + a21 u
        x' = x - dt sx,                 y' = y - dt sy
        d x'/dp = (-dt, 0, -dt u, -dt v, 0, 0)      d y'/dp = (0, -dt, 0, 0, -dt u, -dt v)
    f64 numpy in the order written.  The batched losses, fits and segmentation evaluate it natively on the GPU; the
    reference-API objectives (variance_objective, get_iwe, ...) take it through this warp() (fused_kind None).

    xyztheta_warp(hx, hy, hz, theta) is affine_warp(hx, hy, hz, -theta, theta, hz) bit for bit with the same centre
    (a + (-b) v is a - b v in IEEE arithmetic), so a 4-DoF fit embedded that way is the starting point of an affine
    fit.  A grid search over K = 6 parameters scores num_samples_per_param ** 6 points per window (15625 at 5 samples
    per parameter): start from an embedded 4-DoF fit instead."""

    def __init__(self, center=(120.0, 90.0)):
        super().__init__('affine_warp', 6)
        self.center = (float(center[0]), float(center[1]))

    def model(self, params):
        """the parameter block of the batched GPU evaluation: the 6 parameters, then the centre"""
        return [float(v) for v in params[:6]] + list(self.center)

    def warp(self, xs, ys, ts, ps, t0, params, compute_grad=False):
        hx, hy, a11, a12, a21, a22 = (float(v) for v in params[:6])
        cx, cy = self.center
        dt = ts - t0
        u, v = xs - cx, ys - cy
        sx, sy = (hx + a11 * u) + a12 * v, (hy + a22 * v) + a21 * u
        xw, yw = xs - dt * sx, ys - dt * sy
        if not compute_grad:
            return xw, yw, None, None
        nothing = np.zeros_like(dt, dtype=np.float64)
        du, dv = dt * u, dt * v
        jx = np.stack((-dt, nothing, -du, -dv, nothing, nothing))
        jy = np.stack((nothing, -dt, nothing, nothing, -du, -dv))
        return xw, yw, jx, jy


class homography_warp(warp_function):
    """8-DoF homography in its first-order form about a fixed centre, params = (hx, hy, a11, a12, a21, a22, g1, g2): the
    generator A = [[a11, a12, hx], [a21, a22, hy], [g1, g2, 0]] acts on (u, v, 1) = (x - cx, y - cy, 1), and a33 = 0
    fixes the scale, so the 8 values are a chart of the homography's Lie algebra.  It is the motion of a planar scene
    (or of any scene under a rotating camera, Gallego et al., CVPR 2018).  The warp undoes the motion during dt:
        sx, sy as affine_warp,   nx = u - dt sx,   ny = v - dt sy
        q = dt ((g1 u) + (g2 v)),   w = 1 - q
        x' = (x - dt sx) + nx q / w,      y' = (y - dt sy) + ny q / w          (= cx + nx / w, cy + ny / w)
        d x'/d(hx, .., a22) = affine_warp's row / w,   d x'/d(g1, g2) = (nx dt u, nx dt v) / w^2   (y' with ny)
    f64 numpy in the order written.  An event with w <= 0 has crossed the horizon: the batched losses drop it like an
    event off the canvas (no contribution, no gradient); this warp() returns its formula unchanged, which the reference
    API's bounds mask then judges.  The batched losses, fits and segmentation evaluate the model natively on the GPU;
    the reference-API objectives take it through this warp() (fused_kind None).

    With g1 = g2 = 0 (w = 1) this is affine_warp bit for bit, so an affine fit -- or a 4-DoF fit embedded as
    (hx, hy, hz, -theta, theta, hz), see affine_warp -- extended by g = (0, 0) is the starting point of a homography
    fit.  A grid search over K = 8 parameters scores num_samples_per_param ** 8 points per window (390625 at 5 samples
    per parameter): start from an embedded fit instead."""

    def __init__(self, center=(120.0, 90.0)):
        super().__init__('homography_warp', 8)
        self.center = (float(center[0]), float(center[1]))

    def model(self, params):
        """the parameter block of the batched GPU evaluation: the 8 parameters, then the centre"""
        return [float(v) for v in params[:8]] + list(self.center)

    def warp(self, xs, ys, ts, ps, t0, params, compute_grad=False):
        hx, hy, a11, a12, a21, a22, g1, g2 = (float(v) for v in params[:8])
        cx, cy = self.center
        dt = ts - t0
        u, v = xs - cx, ys - cy
        sx, sy = (hx + a11 * u) + a12 * v, (hy + a22 * v) + a21 * u
        mx, my = dt * sx, dt * sy
        nx, ny = u - mx, v - my
        q = dt * (g1 * u + g2 * v)
        w = 1.0 - q
        with np.errstate(divide="ignore", invalid="ignore"):
            xw, yw = (xs - mx) + nx * q / w, (ys - my) + ny * q / w
            if not compute_grad:
                return xw, yw, None, None
            nothing = np.zeros_like(dt, dtype=np.float64)
            du, dv, w2 = dt * u, dt * v, w * w
            jx = np.stack((-dt / w, nothing, -du / w, -dv / w, nothing, nothing, nx * du / w2, nx * dv / w2))
            jy = np.stack((nothing, -dt / w, nothing, nothing, -du / w, -dv / w, ny * du / w2, ny * dv / w2))
        return xw, yw, jx, jy


def _intrinsics(camera_matrix):
    """(fx, fy, cx, cy) of a 3x3 camera matrix without skew or of the four values themselves"""
    k = np.asarray(camera_matrix, dtype=np.float64)
    if k.shape == (3, 3):
        if k[0, 1] != 0.0 or k[1, 0] != 0.0 or k[2, 0] != 0.0 or k[2, 1] != 0.0 or k[2, 2] != 1.0:
            raise ValueError("camera_matrix must be [[fx, 0, cx], [0, fy, cy], [0, 0, 1]] (no skew), got %s" % k.tolist())
        k = np.array([k[0, 0], k[1, 1], k[0, 2], k[1, 2]])
    elif k.shape != (4,):
        raise ValueError("camera_matrix must be a 3x3 matrix or (fx, fy, cx, cy), got shape %s" % (k.shape,))
    fx, fy, cx, cy = (float(v) for v in k)
    if not (np.isfinite(k).all() and fx > 0.0 and fy > 0.0):
        raise ValueError("the focal lengths must be finite and positive and the principal point finite, got fx=%r, "
                         "fy=%r, cx=%r, cy=%r" % (fx, fy, cx, cy))
    return fx, fy, cx, cy


class camera_rotation_warp(warp_function):
    """A rotating camera, exact in the rotation: params = (wx, wy, wz), the camera's angular velocity (rad/s) in its own
    frame, with OpenCV's axes (x to the right, y down, z along the optical axis).  camera_matrix is the 3x3 K (no
    skew) or (fx, fy, cx, cy); the events are pixel coordinates that have already been undistorted.  With dt = t - t0:
        b = ((x - cx) / fx, (y - cy) / fy, 1),   theta = dt w,   phi = |theta|,   c = theta x b,   e = theta x c
        P = exp([theta]x) b = (b + A c) + B e,   A = sin(phi) / phi,   B = (1 - cos(phi)) / phi^2
        x' = cx + fx Px / Pz,   y' = cy + fy Py / Pz
    with A = r cos(phi/2), B = r^2 / 2 and r = sin(phi/2) / (phi/2) (1 at phi = 0).  A camera whose orientation is
    R(t0) exp([w]x dt) sees a static scene along the bearings exp(-[w]x dt) b(t0); the warp undoes that rotation.  So
    with fx = fy, w = (0, 0, wz) is pure_rotation_warp(cx, cy, -wz).  With X = Px / Pz, Y = Py / Pz and the SO(3) left
    Jacobian J_l = A I + B [theta]x + C theta theta^T, C = (phi - sin(phi)) / phi^3:
        d x'/dw = -dt fx J_l^T (X Y, -(1 + X X), Y),      d y'/dw = -dt fy J_l^T (1 + Y Y, -X Y, -X)
    f64 numpy, C from its series below phi = 1e-2.  An event with Pz <= 0 has rotated behind the camera: the batched
    losses drop it like an event off the canvas (no contribution, no gradient); this warp() returns its formula
    unchanged, which the reference API's bounds mask then judges.

    The batched losses, their candidates passes, the fits and motion segmentation evaluate the model natively on the
    GPU with K = 3 parameters: they append (fx, fy) to every row they hand the C entries (EVK_WARP_CAMERA_ROTATION,
    whose rows are (wx, wy, wz, fx, fy) about the principal point center = (cx, cy)).  The reference-API objectives
    take it through this warp() (fused_kind None).  homography_warp holds a rotation only to first order in dt w
    (A = K [w]x K^-1), which misplaces the scene by about f phi^2 / 2 at the window's edge."""

    def __init__(self, camera_matrix):
        super().__init__('camera_rotation_warp', 3)
        fx, fy, cx, cy = _intrinsics(camera_matrix)
        self.focal = (fx, fy)
        self.center = (cx, cy)

    def model(self, params):
        """the parameter block of the batched GPU evaluation: the angular velocity, the focal lengths (the row the C
        entries take), then the principal point"""
        return [float(v) for v in params[:3]] + list(self.focal) + list(self.center)

    def warp(self, xs, ys, ts, ps, t0, params, compute_grad=False):
        wx, wy, wz = (float(v) for v in params[:3])
        fx, fy = self.focal
        cx, cy = self.center
        dt = ts - t0
        bx, by = (xs - cx) / fx, (ys - cy) / fy
        tx, ty, tz = dt * wx, dt * wy, dt * wz
        p2 = (tx * tx + ty * ty) + tz * tz
        phi = np.sqrt(p2)
        half = 0.5 * phi
        sh, ch = np.sin(half), np.cos(half)
        r = np.where(phi > 0, sh / np.where(phi > 0, half, 1.0), 1.0)
        A, B = r * ch, 0.5 * (r * r)
        c0, c1, c2 = ty - tz * by, tz * bx - tx, tx * by - ty * bx
        e0, e1, e2 = ty * c2 - tz * c1, tz * c0 - tx * c2, tx * c1 - ty * c0
        Px, Py, Pz = (bx + A * c0) + B * e0, (by + A * c1) + B * e1, (1.0 + A * c2) + B * e2
        with np.errstate(divide="ignore", invalid="ignore"):
            xw, yw = cx + fx * Px / Pz, cy + fy * Py / Pz
            if not compute_grad:
                return xw, yw, None, None
            X, Y = Px / Pz, Py / Pz
            series = 1.0 / 6 - p2 * (1.0 / 120 - p2 * (1.0 / 5040))
            C = np.where(phi < 1e-2, series, (phi - 2.0 * (sh * ch)) / np.where(phi < 1e-2, 1.0, p2 * phi))

            def jlt(w0, w1, w2, s):
                k0, k1, k2 = ty * w2 - tz * w1, tz * w0 - tx * w2, tx * w1 - ty * w0
                q = C * ((tx * w0 + ty * w1) + tz * w2)
                return np.stack((s * ((A * w0 - B * k0) + q * tx), s * ((A * w1 - B * k1) + q * ty),
                                 s * ((A * w2 - B * k2) + q * tz)))
            jx = jlt(X * Y, -(1.0 + X * X), Y, -(dt * fx))
            jy = jlt(1.0 + Y * Y, -(X * Y), -X, -(dt * fy))
        return xw, yw, jx, jy


class camera_motion_warp(warp_function):
    """A camera that rotates and translates through a scene with known depth: params = (wx, wy, wz, vx, vy, vz), the
    camera's angular velocity w (rad/s) in its own frame, with camera_rotation_warp's axes (x to the right, y down, z
    along the optical axis), and its linear velocity v in the camera frame at t0, in depth units per second (m/s when
    the inverse depth is in 1/m).  camera_matrix is the 3x3 K (no skew) or (fx, fy, cx, cy); the events are undistorted
    pixel coordinates, and every event carries rho, the inverse depth 1/Z of its scene point at the event's time (Z
    along the optical axis; callers sample their depth or disparity map at the events).  With dt = t - t0 and b, theta,
    A, B exactly as in camera_rotation_warp:
        P = exp([theta]x) b + (rho dt) v,   iz = 1 / Pz,   X = Px iz,   Y = Py iz,   x' = cx + fx X,   y' = cy + fy Y
    This is exact for a camera whose pose at t, in the camera frame at t0, is (exp(dt [w]x), dt v): a constant rotation
    rate and a constant velocity.  rho = 0 (a point at infinity) or v = 0 is camera_rotation_warp.  With Q = exp([theta]x)
    b iz and the left Jacobian J_l of camera_rotation_warp:
        d x'/dw = -dt fx J_l^T (X Qy, -(Qz + X Qx), Qy),     d y'/dw = -dt fy J_l^T (Qz + Y Qy, -Y Qx, -Qx)
        d x'/dv = (rho dt) fx iz (1, 0, -X),                 d y'/dv = (rho dt) fy iz (0, 1, -Y)
    f64 numpy.  The batched losses drop an event with Pz <= 0 (behind the camera) or with a negative or non-finite rho,
    like an event off the canvas; this warp() returns its formula unchanged.

    The batched losses, their candidates passes and the fits evaluate the model natively on the GPU with K = 6
    parameters and an inv_depth array aligned with the events: they append (fx, fy) to every row they hand the C entries
    (the evk_*_depth_* entries with EVK_WARP_CAMERA_MOTION, whose rows are (wx, wy, wz, vx, vy, vz, fx, fy) about the
    principal point center = (cx, cy)).  warp() needs inv_depth, so the reference-API objectives, which call warp()
    without it (fused_kind None), reject the model; motion segmentation does not take it."""

    def __init__(self, camera_matrix):
        super().__init__('camera_motion_warp', 6)
        fx, fy, cx, cy = _intrinsics(camera_matrix)
        self.focal = (fx, fy)
        self.center = (cx, cy)

    def model(self, params):
        """the parameter block of the batched GPU evaluation: the angular and linear velocities, the focal lengths (the
        row the C entries take), then the principal point"""
        return [float(v) for v in params[:6]] + list(self.focal) + list(self.center)

    def warp(self, xs, ys, ts, ps, t0, params, compute_grad=False, inv_depth=None):
        if inv_depth is None:
            raise ValueError("camera_motion_warp.warp needs the inverse depth of every event (inv_depth=...); the "
                             "reference-API objectives do not pass it, use the batched motion losses and fits")
        wx, wy, wz, vx, vy, vz = (float(v) for v in params[:6])
        fx, fy = self.focal
        cx, cy = self.center
        dt = ts - t0
        s = np.asarray(inv_depth, np.float64) * dt
        bx, by = (xs - cx) / fx, (ys - cy) / fy
        tx, ty, tz = dt * wx, dt * wy, dt * wz
        p2 = (tx * tx + ty * ty) + tz * tz
        phi = np.sqrt(p2)
        half = 0.5 * phi
        sh, ch = np.sin(half), np.cos(half)
        r = np.where(phi > 0, sh / np.where(phi > 0, half, 1.0), 1.0)
        A, B = r * ch, 0.5 * (r * r)
        c0, c1, c2 = ty - tz * by, tz * bx - tx, tx * by - ty * bx
        e0, e1, e2 = ty * c2 - tz * c1, tz * c0 - tx * c2, tx * c1 - ty * c0
        Ux, Uy, Uz = (bx + A * c0) + B * e0, (by + A * c1) + B * e1, (1.0 + A * c2) + B * e2
        Px, Py, Pz = Ux + s * vx, Uy + s * vy, Uz + s * vz
        with np.errstate(divide="ignore", invalid="ignore"):
            xw, yw = cx + fx * Px / Pz, cy + fy * Py / Pz       # camera_rotation_warp's expressions at s v = 0
            if not compute_grad:
                return xw, yw, None, None
            iz = 1.0 / Pz
            X, Y = Px / Pz, Py / Pz
            Qx, Qy, Qz = Ux * iz, Uy * iz, Uz * iz
            series = 1.0 / 6 - p2 * (1.0 / 120 - p2 * (1.0 / 5040))
            C = np.where(phi < 1e-2, series, (phi - 2.0 * (sh * ch)) / np.where(phi < 1e-2, 1.0, p2 * phi))

            def jlt(w0, w1, w2, k):
                k0, k1, k2 = ty * w2 - tz * w1, tz * w0 - tx * w2, tx * w1 - ty * w0
                q = C * ((tx * w0 + ty * w1) + tz * w2)
                return [k * ((A * w0 - B * k0) + q * tx), k * ((A * w1 - B * k1) + q * ty), k * ((A * w2 - B * k2) + q * tz)]
            nothing = np.zeros_like(X)
            sx, sy = s * fx * iz, s * fy * iz
            jx = np.stack(jlt(X * Qy, -(Qz + X * Qx), Qy, -(dt * fx)) + [sx, nothing, -(sx * X)])
            jy = np.stack(jlt(Qz + Y * Qy, -(Y * Qx), -Qx, -(dt * fy)) + [nothing, sy, -(sy * Y)])
        return xw, yw, jx, jy
