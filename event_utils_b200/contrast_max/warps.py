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
