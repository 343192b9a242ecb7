"""Seeded generator of small adversarial event sets shared by the CPU (oracle vs reference) and GPU
(CUDA vs oracle) edge-case tests: tiny sensors, coordinates around and beyond the borders (negative
wrap, exact integers, out of range), repeated / identical timestamps, zero / fractional / NaN
polarities, single events."""
import numpy as np


def cases(seed, count):
    rng = np.random.default_rng(seed)
    for k in range(count):
        H, W = int(rng.integers(2, 18)), int(rng.integers(2, 22))
        B = int(rng.integers(1, 10))
        n = int(rng.integers(1, 260))
        spread = rng.choice([0.0, 0.0, 1.5, 3.0])            # how far beyond the border coordinates may go
        x = rng.uniform(-spread, W - 1 + spread, n)
        y = rng.uniform(-spread, H - 1 + spread, n)
        snap = rng.random(n) < 0.3                            # exact integers (incl. borders)
        x[snap], y[snap] = np.round(x[snap]), np.round(y[snap])
        t = np.sort(rng.random(n)) * rng.choice([1.0, 1e-3, 50.0])
        if rng.random() < 0.2:
            t[: n // 2] = t[0]                                # repeated stamps
        if rng.random() < 0.1:
            t[:] = t[0]                                       # dt == 0 -> NaN weights
        p = rng.choice([-1.0, 1.0, 0.0, 0.37, 2.5], n)
        yield dict(k=k, B=B, H=H, W=W, x=x.astype(np.float32), y=y.astype(np.float32), t=t.astype(np.float32),
                   p=p.astype(np.float32), clip=bool(rng.random() < 0.5), padding=bool(rng.random() < 0.5))


# ---- harder cases: values on the kernels' internal limits ------------------------------------------------------------
# cases() above is pinned by tests/golden/edge_cases.npz; hard_cases() is a separate stream with its own draws.
_F32 = np.float32
POLARITY_LIMITS = np.array([1.0, -1.0, 1.0 + 2.0 ** -23, -(1.0 + 2.0 ** -23), 2.0 ** 20, -2.0 ** 20, -0.0, 0.0,
                            2.0 ** -10, -3 * 2.0 ** -10, 1023 * 2.0 ** -10, 0.999999], np.float32)
NONFINITE = np.array([np.inf, -np.inf, np.nan, -np.nan], np.float32)


def _edge_coords(rng, n, size, spread):
    """Coordinates on a 1-D axis of `size` pixels: uniform, plus exact borders (size-1, just below size, -0.0,
    -ulp, -2^-24) and, with spread > 0, whole pixels beyond either border."""
    v = rng.uniform(-spread, size - 1 + spread, n).astype(_F32)
    special = np.array([size - 1, np.nextafter(_F32(size), _F32(0)), -0.0, -np.finfo(_F32).smallest_subnormal,
                        -2.0 ** -24, 0.0, np.nextafter(_F32(size - 1), _F32(size)), size - 0.5], np.float32)
    pick = rng.random(n) < 0.35
    v[pick] = rng.choice(special, int(pick.sum()))
    return v


def hard_cases(seed, count, nonfinite=True):
    """Adversarial sets with explicit t0 / dt: polarities on the fixed-point limits (multiples of 2^-10, +-1, 1 + ulp,
    +-2^20, -0.0; +-inf and NaN of either sign when `nonfinite`), coordinates on the borders (W-1, just below W,
    -0.0, -ulp), unsorted stamps and t0 / dt that put tau below 0 and above B-1.  Every case has clip / padding
    flags and a `fill` for the image functions."""
    rng = np.random.default_rng(seed)
    for k in range(count):
        H, W = int(rng.integers(2, 12)), int(rng.integers(2, 14))
        if k % 4 == 0:
            H, W = 2, 3
        B = int(rng.integers(1, 8))
        n = int(rng.integers(1, 300))
        spread = float(rng.choice([0.0, 0.0, 1.0]))
        x, y = _edge_coords(rng, n, W, spread), _edge_coords(rng, n, H, spread)
        p = rng.choice(POLARITY_LIMITS, n)
        q = rng.random(n) < 0.3
        p[q] = (rng.integers(-2048, 2049, int(q.sum())) * 2.0 ** -10).astype(_F32)
        if nonfinite and k % 5 == 3:
            m = rng.random(n) < 0.03
            p[m] = rng.choice(NONFINITE, int(m.sum()))
        t = (rng.random(n) * rng.choice([1.0, 1e-3, 50.0])).astype(_F32)
        if k % 3 != 0:
            t = np.sort(t)
        span = float(t.max() - t.min()) if n > 1 else 1.0
        mode = k % 4
        if mode == 0:
            t0, dt = float(t[0]), float(_F32(t[-1]) - _F32(t[0]))        # the reference's own t0 / dt
        elif mode == 1:
            t0, dt = float(t.min()) + 0.3 * span, 0.5 * span + 1e-6      # tau < 0 and > B-1
        elif mode == 2:
            t0, dt = float(t.min()) - 0.2 * span, 0.4 * span + 1e-6
        else:
            t0, dt = float(t.min()), float(span) + 1e-6
        yield dict(k=k, B=B, H=H, W=W, x=x, y=y, t=t, p=p.astype(_F32), t0=_F32(t0), dt=_F32(dt),
                   clip=bool(rng.random() < 0.5), padding=bool(rng.random() < 0.5),
                   fill=_F32(rng.choice([0.0, 0.0, 0.25, -3.0])))


def replicate(case, n):
    """The case's events tiled up to n events (same sensor, t0 / dt): past a size threshold the kernels take another
    path, and on a small sensor every pixel is contended."""
    c = dict(case)
    for key in "xytp":
        c[key] = np.resize(case[key], n).astype(_F32)
    c["k"] = "%s*%d" % (case["k"], n)
    return c
