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


# ---- exactly summable streams ----------------------------------------------------------------------------------------
# Every tap of these streams is a multiple of 2^-g and every partial sum a kernel can form stays below 2^(24-g): any
# summation order, fixed-point quantisation, flush and carry is then exact, and a kernel's output must equal the f64
# sum of the taps BIT FOR BIT (tests/exact_bounds.py assert_exactly_summable / assert_exact).
#   hot cells   a few pixels with most of the events, signs in one run of + then one run of - by event index, so that
#               the fixed-point table slot of every CTA that holds a hot cell wraps upward and back downward at the
#               launch geometry of the exact-sum tests (exact_bounds.table_wraps checks it; values below)
#   fine cells  everything else: taps on a 2^-12 grid, a |tap| sum per cell below the wrap threshold of any table,
#               quarter-pixel coordinates on and beyond the borders, polarities with |p| > 1 that bypass the tables
# No output cell receives taps of both classes.
EXACT_FINE_P = np.array([1.0, -1.0, -1.25, 3.0, 0.5, -0.75, 2.5, 0.25], np.float32)
EXACT_KINDS = ("voxel", "nearest", "bilinear", "cmax")


def _fine_coords(rng, n, size):
    """Quarter-pixel coordinates over [-1, size], with the border values size-1, size-1/4, -1/4 (trunc 0, floor -1),
    -1 (wraps) and, for ~1 % of the events, whole pixels out of range (size, -size-1)."""
    v = rng.integers(-4, 4 * size + 1, n) / 4.0
    special = np.array([size - 1, size - 0.25, -0.25, -1.0, 0.0, size - 0.5])
    pick = rng.random(n) < 0.1
    v[pick] = rng.choice(special, int(pick.sum()))
    out = rng.random(n) < 0.01
    v[out] = rng.choice(np.array([float(size), -size - 1.0]), int(out.sum()))
    return v


# events per stream of the exact-sum tests: the voxel table launches with 1024 events per CTA reach their one-wave cap
# (4 waves of at most 5 CTAs per SM) only from about 3.4 M events, and need ~1300 same-slot events per CTA to wrap both ways
EXACT_SIZES = dict(voxel=(4 << 20) + 4099, nearest=(1 << 20) + 5, bilinear=(1 << 20) + 5, cmax=(4 << 20) + 3)


def exact_streams(seed, kind, n, fine=20000, pos_frac=None):
    """One exactly summable stream of `n` events for the scatter path `kind`:
      voxel     B = 5, t0 = 0.5, dt = 2: tau = (t - t0) / dt * 4 is a multiple of 2^-6 in [-1, 5].  Hot pixel A (96 %
                of the hot events): p = +-1 at tau = 0, one integer tap in bin 0 (g = 0), so that one table slot takes
                all of it; hot pixel B (4 %): tau = 7/2, taps of 1/2 in bins 3 and 4 (g = 1), so that hot events with
                two taps are summed too.  + run 60 %, - run 40 %: every CTA of the table launches wraps
                up and back down (mostly with a zero net carry, so a carry of one direction that is lost or
                mis-signed shows)
      nearest   hot p = +-2^19: in the 2^10 image table q = 2^29, so a slot wraps every four same-sign adds
      bilinear  one hot point at (i + 1/2, j), p = +-1: taps of 1/2 into the top-left and top-right cells, g = 1 (an
                image CTA takes four 2048-event rounds: 1/2-unit taps are what wraps its slot both ways)
      cmax      f64 events, velocity (32, -16), t_ref = 0, stamps on a 2^-6 grid in [-1, 0]: the warped coordinates are
                quarter pixels; each hot event warps onto one of two half-pixel points (taps 1/4), |d| <= 2^-5 so that
                the dIWE taps stay small
    `fine` events (at most) are fine, the rest hot; the first `pos_frac` of the hot events are +, the rest - (default
    0.6 for voxel, 0.7 for the others: their cells also end with net carries, since up and down wraps that cancel
    would hide a carry sent to the wrong cell).  Returns a dict: x, y, t, p (float32; float64 for cmax), `hot` (the
    class of each event), `group` (0 fine, 1 hot point A, 2 hot point B), `pos_frac` and the parameters of the call
    (B, H, W, t0, dt; cmax: vx, vy, t_ref, Hs, Ws)."""
    assert kind in EXACT_KINDS
    rng = np.random.default_rng(seed)
    H, W = (40, 56) if kind == "cmax" else (32, 48)
    hot = np.zeros(n, bool)
    hot[rng.permutation(n)[:max(n - fine, n // 2)]] = True
    nh, nf = int(hot.sum()), int(n - hot.sum())
    # the hot points: interior pixels, (hx, hy) and (hx2, hy2), each with half of the hot events (alternating by index)
    hx, hy, hx2, hy2 = W // 3, H // 3, 2 * W // 3, 2 * H // 3
    if pos_frac is None:
        pos_frac = 0.6 if kind == "voxel" else 0.7
    which = {"voxel": (np.arange(nh) % 25 == 0).astype(int), "bilinear": np.zeros(nh, int)}.get(kind, np.arange(nh) % 2)
    sign = np.where(np.arange(nh) < int(pos_frac * nh), 1.0, -1.0)
    # fine events stay out of a 7x7 moat around each hot point (no tap of one class lands in a cell of the other)
    fx, fy = _fine_coords(rng, 2 * nf + 64, W), _fine_coords(rng, 2 * nf + 64, H)
    keep = ~(((np.abs(fx - hx) < 4) & (np.abs(fy - hy) < 4)) | ((np.abs(fx - hx2) < 4) & (np.abs(fy - hy2) < 4)))
    fx, fy = fx[keep][:nf], fy[keep][:nf]
    assert fx.shape[0] == nf
    fp = rng.choice(EXACT_FINE_P, nf)
    x, y, p, t = np.empty(n), np.empty(n), np.empty(n), np.empty(n)
    x[~hot], y[~hot], p[~hot] = fx, fy, fp
    group = np.zeros(n, int)
    group[hot] = 1 + which
    c = dict(kind=kind, H=H, W=W, hot=hot, group=group, pos_frac=pos_frac)
    if kind == "cmax":
        vx, vy = 32.0, -16.0
        ft = -rng.integers(0, 65, nf) / 64.0                         # d = t - t_ref in [-1, 0], 2^-6 grid
        t[~hot] = ft
        x[~hot] += ft * vx                                            # warped x - d vx: the fine grid above
        y[~hot] += ft * vy
        ht = -rng.integers(0, 3, nh) / 64.0
        t[hot] = ht
        x[hot] = np.where(which, hx2, hx) + 0.5 + ht * vx
        y[hot] = np.where(which, hy2, hy) + 0.5 + ht * vy
        p[hot] = sign
        c.update(vx=vx, vy=vy, t_ref=0.0, Hs=H, Ws=W)
        c.update(x=x, y=y, t=t, p=p)
        return c
    B, t0, dt = 5, 0.5, 2.0
    t[~hot] = t0 + dt * rng.integers(-64, 321, nf) / 256.0           # tau in [-1, 5] on a 2^-6 grid
    if kind == "voxel":
        x[hot] = np.where(which, hx2 + 0.75, hx + 0.25)
        y[hot] = np.where(which, hy2 + 0.5, hy)
        t[hot] = t0 + dt * np.where(which, 3.5, 0.0) / 4.0
        p[hot] = sign
    elif kind == "nearest":
        x[hot] = np.where(which, hx2 + 0.75, hx)
        y[hot] = np.where(which, hy2 + 0.25, hy + 0.5)
        t[hot] = t0 + dt * rng.integers(0, 257, nh) / 256.0
        p[hot] = sign * 2.0 ** 19
    else:
        x[hot] = np.where(which, hx2, hx) + 0.5
        y[hot] = np.where(which, hy2, hy)
        t[hot] = t0 + dt * rng.integers(0, 257, nh) / 256.0
        p[hot] = sign
    t[0], t[-1] = t0, t0 + dt                                        # EVK_AUTO_SPAN finds the same span
    c.update(B=B, t0=_F32(t0), dt=_F32(dt))
    c.update({k: v.astype(_F32) for k, v in dict(x=x, y=y, t=t, p=p).items()})
    return c


def packed_of(c, T0=1.7e9):
    """The storage-layout (int16 x / y, float64 absolute stamps, uint8 polarity) form of a float32 stream, as the
    HDF5 / memmap loaders hand it over, plus the float32 events the kernel turns it into:
      x, y  floor to int16 (a coordinate at -ulp becomes -1 and wraps)
      t     T0 + t in float64; t_first = T0 + t0, t_last = t_first + dt
      p     uint8 [p > 0], which the kernel maps to +-1 (finite polarities only: uint8 holds no NaN)
    Returns (x16, y16, T, p8, t_first, t_last, f32) with f32 = dict(x, y, t, p, t0, dt) for the oracle."""
    x16 = np.floor(c["x"].astype(np.float64)).astype(np.int16)
    y16 = np.floor(c["y"].astype(np.float64)).astype(np.int16)
    T = T0 + c["t"].astype(np.float64)
    t_first = T0 + float(c["t0"])
    t_last = t_first + float(c["dt"])
    p8 = (c["p"] > 0).astype(np.uint8)
    f32 = dict(x=x16.astype(_F32), y=y16.astype(_F32), t=(T - t_first).astype(_F32),
               p=np.where(p8 != 0, 1.0, -1.0).astype(_F32), t0=_F32(0.0), dt=_F32(t_last - t_first))
    return x16, y16, T, p8, t_first, t_last, f32


# ---- exactly computable gradient streams -------------------------------------------------------------------------------
# Every per-event gradient of these streams is exact in f32: quarter-pixel coordinates, integer or dyadic polarities and
# incoming gradients, tn on quarter bins with dt and B-1 powers of two; for the warp W-1 and H-1 powers of two (the
# normalise round trip is exact), a dyadic flow and dt.  The window sums sum G and sum G tn of the voxel backward and
# sum grad_t of the warp need MORE than 24 significant bits: the incoming gradient rises with the bin (voxel) and the
# flow and gradients are biased positive (warp), so the sums grow with n on a fine dyadic grid.  Only f64 accumulation
# then gives the value the tests expect, rounded once to f32.
EXACT_GRAD_P = np.array([1.0, 2.0, 3.0, -1.0, 0.5, 3 * 2.0 ** -12, 5 * 2.0 ** -12, -7 * 2.0 ** -12], np.float32)


def exact_grad_streams(seed, kind, n, windows=None):
    """One exactly computable gradient stream of n events for kind "voxel", "image" or "warp".
      voxel  B = 5, 12x16 sensor (coordinates also beyond it, wrapping or dropped); per window [s, e) the stamps are
             w + q/16 (q = 0..16, the first 0 and the last 16): t0 = w, dt = 1, tn = q/4.  `windows`: [nw][2] pairs
             (default one window [0, n)).  g: the incoming gradient [nw][1][B][H][W], 4b + an integer in [-2, 2]
      image  canvas 13x17, quarter-pixel coordinates over [-1, size], integer polarities, integer g [H][W]
      warp   33x33 field (W-1 = H-1 = 32), quarter-pixel coordinates over [-2, 34], stamps k/8 in [0, 2] with t0 = 0,
             flow in quarters biased positive, incoming gradients integers biased positive
    Returns a dict of f32 arrays and the parameters."""
    rng = np.random.default_rng(seed)
    if kind == "voxel":
        B, H, W = 5, 12, 16
        if windows is None:
            windows = np.array([[0, n]], np.int64)
        windows = np.asarray(windows, np.int64).reshape(-1, 2)
        t = np.zeros(n, np.float32)
        for w, (s, e) in enumerate(windows):
            if e > s:
                q = rng.integers(0, 17, e - s)
                q[0], q[-1] = 0, 16
                t[s:e] = w + q / 16.0
        x = (rng.integers(-4 * W, 8 * W, n) / 4.0).astype(np.float32)
        y = (rng.integers(-4 * H, 8 * H, n) / 4.0).astype(np.float32)
        p = rng.choice(EXACT_GRAD_P, n)
        g = (4 * np.arange(B)[None, None, :, None, None]
             + rng.integers(-2, 3, (len(windows), 1, B, H, W))).astype(np.float32)
        return dict(kind=kind, x=x, y=y, t=t, p=p, B=B, H=H, W=W, g=g, pairs=windows)
    if kind == "image":
        H, W = 13, 17
        x = (rng.integers(-4, 4 * W + 1, n) / 4.0).astype(np.float32)
        y = (rng.integers(-4, 4 * H + 1, n) / 4.0).astype(np.float32)
        p = rng.integers(-3, 4, n).astype(np.float32)
        g = rng.integers(-8, 9, (H, W)).astype(np.float32)
        return dict(kind=kind, x=x, y=y, p=p, H=H, W=W, g=g)
    assert kind == "warp"
    H = W = 33
    x = (rng.integers(-8, 4 * (W + 1) + 1, n) / 4.0).astype(np.float32)
    y = (rng.integers(-8, 4 * (H + 1) + 1, n) / 4.0).astype(np.float32)
    t = (rng.integers(0, 17, n) / 8.0).astype(np.float32)
    flow = (rng.integers(-4, 13, (2, H, W)) / 4.0).astype(np.float32)
    gx = rng.integers(-2, 7, n).astype(np.float32)
    gy = rng.integers(-2, 7, n).astype(np.float32)
    return dict(kind=kind, x=x, y=y, t=t, flow=flow, gxw=gx, gyw=gy, H=H, W=W, t0=np.float32(0.0))
