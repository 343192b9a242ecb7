"""Skewed batches of event windows for the window-count limits of the batched losses, candidate passes and fits -- TEST
INFRASTRUCTURE ONLY.

B concatenated windows on a 6x10 sensor (a 7x11 canvas): about 20 % empty, about 10 % with one event, the rest with 2 to
7 events, and optionally one giant window of GIANT events at a chosen index.  The batched entries size their event grid
from the MEAN window (n / batch CTAs' worth), so the giant window runs on one CTA inside such a batch and on hundreds
alone.

exact_stream: the linvel variant.  Warped coordinates x' = x - d vx on the quarter-pixel grid over [-1, size] with the
border values of edge_cases._fine_coords, d = t - t0 on the 2^-6 grid in [-1, 0], p = +-1 and, for the timestamp
entries, tau on the 1/16 grid (passed to the C entries as is).  Under any velocity whose components are multiples of 16
(EXACT_VELOCITIES) every warped coordinate stays on the quarter grid, every tap on the 1/16 grid and every per-pixel sum
below 2^20 (assert_exactly_summable checks it), so every image is exact in f32 whatever the order of its reductions.

random_stream: the rotation and 4-DoF variant: positions uniform in the sensor, d on the 2^-12 grid in [-0.1, 0).

voxel_stream: the windows of evk_voxel_windows_f32 / the windowed evk_voxel_grad_f32 (VOXEL_BINS bins).  Window w has
its own t0_w = w mod 64 and a power-of-two span dt_w; its stamps are t0_w + dt_w k / 64 with k in 0..64, the first
event at k = 0 and the last at k = 64 (windows of two or more events), so that the window's own t0 and dt are t0_w and
dt_w and tn = (t - t0) / dt * (B - 1) = k / 16 exactly in f32.  Pixels are whole-pixel truncations of quarter-pixel
positions inside the sensor and p = +-1, so every bin weight is on the 1/16 grid and every cell sum is exact.  A
one-event window has dt = 0 (tn NaN, as in the reference)."""
import numpy as np

from edge_cases import _fine_coords

H, W = 6, 10
HC, WC = H + 1, W + 1
GIANT = (1 << 21) + 3
V = (32.0, -16.0)
CENTRE = (5.0, 3.0)
MOTION_CAP = 65535        # evk_cmax_motion_objective_f32, evk_cmax_flow_objective_f32: batch <= 65535 tail canvases
TIMESTAMP_CAP = 32767     # the timestamp entries: two tail images per window
MAX_CANDIDATES = 32


def exact_velocities():
    """the 5x5 grid around V with a step of 16 (motion_contrast_fit_torch's grid over V +- 32), in its meshgrid order"""
    ax = np.array([-32.0, -16.0, 0.0, 16.0, 32.0])
    gx, gy = np.meshgrid(V[0] + ax, V[1] + ax)
    return np.column_stack((gx.ravel(), gy.ravel()))


EXACT_RANGES = [[V[0] - 32.0, V[0] + 32.0], [V[1] - 32.0, V[1] + 32.0]]


def window_sizes(B, giant_at=None, seed=0):
    rng = np.random.default_rng(seed)
    u = rng.random(B)
    sizes = np.where(u < 0.2, 0, np.where(u < 0.3, 1, rng.integers(2, 8, B))).astype(np.int64)
    if giant_at is not None:
        sizes[giant_at] = GIANT
    return sizes


def _offsets(sizes):
    return np.concatenate(([0], np.cumsum(sizes))).astype(np.int64)


def exact_stream(B, giant_at=None, seed=0):
    """dict x, y, d, tau, p (float32), off (B+1 int64), sizes"""
    sizes = window_sizes(B, giant_at, seed)
    n = int(sizes.sum())
    rng = np.random.default_rng(seed + 1)
    xw, yw = _fine_coords(rng, n, W), _fine_coords(rng, n, H)
    d = -rng.integers(0, 65, n) / 64.0
    x, y = xw + d * V[0], yw + d * V[1]
    p = rng.choice(np.array([-1.0, 1.0]), n)
    tau = rng.integers(0, 17, n) / 16.0
    f = np.float32
    return dict(x=x.astype(f), y=y.astype(f), d=d.astype(f), tau=tau.astype(f), p=p.astype(f), off=_offsets(sizes),
                sizes=sizes)


def random_stream(B, giant_at=None, seed=0):
    sizes = window_sizes(B, giant_at, seed)
    n = int(sizes.sum())
    rng = np.random.default_rng(seed + 1)
    f = np.float32
    return dict(x=(rng.random(n) * (W - 1)).astype(f), y=(rng.random(n) * (H - 1)).astype(f),
                d=(-rng.integers(1, 410, n) / 4096.0).astype(f), tau=rng.random(n).astype(f),
                p=(rng.integers(0, 2, n) * 2 - 1).astype(f), off=_offsets(sizes), sizes=sizes)


EVENT_KEYS = ("x", "y", "d", "tau", "p", "t", "k", "r", "w")


def reversed_stream(s):
    """the same windows in reverse order"""
    off, B = s["off"], len(s["sizes"])
    idx = np.concatenate([np.arange(off[b], off[b + 1]) for b in range(B - 1, -1, -1)]) if B else np.zeros(0, np.int64)
    out = {k: s[k][idx] for k in EVENT_KEYS if k in s}
    out["sizes"] = s["sizes"][::-1].copy()
    out["off"] = _offsets(out["sizes"])
    return out


def window_ids(off):
    return np.repeat(np.arange(len(off) - 1), np.diff(off))


def linvel_taps(s, v, flow=False):
    """the bilinear taps of every contributing event under linvel velocity v ((2,) or per window (B,2)), in f64: (window,
    pixel index y*WC+x of the top-left tap, dx, dy, keep).  Exact for exact_stream under a velocity of EXACT_VELOCITIES.
    The motion entries keep 0 < x' < W, 0 < y' < H (x' = W has zero weight); with `flow`, the keep rule of the flow and
    grid-flow entries, 0 <= x' < W, 0 <= y' < H"""
    b = window_ids(s["off"])
    v = np.asarray(v, np.float64)
    vx, vy = (v[b, 0], v[b, 1]) if v.ndim == 2 else (v[0], v[1])
    xw = s["x"].astype(np.float64) - s["d"].astype(np.float64) * vx
    yw = s["y"].astype(np.float64) - s["d"].astype(np.float64) * vy
    lo = (xw >= 0) & (yw >= 0) if flow else (xw > 0) & (yw > 0)
    keep = np.isfinite(xw) & np.isfinite(yw) & lo & (xw < W) & (yw < H)
    px, py = np.floor(np.where(keep, xw, 0)), np.floor(np.where(keep, yw, 0))
    return b, (py * WC + px).astype(np.int64), xw - px, yw - py, keep


def _splat(B, b, pix, dx, dy, keep, w):
    img = np.zeros(B * HC * WC)
    base = b * HC * WC + pix
    for o, k in ((0, (1 - dx) * (1 - dy)), (1, dx * (1 - dy)), (WC, (1 - dx) * dy), (WC + 1, dx * dy)):
        img += np.bincount(base[keep] + o, weights=(w * k)[keep], minlength=B * HC * WC)
    return img.reshape(B, HC, WC)


def linvel_iwe(s, v, flow=False, weight=None):
    """(B, HC, WC) f64 images of p of the contrast loss under linvel velocity v (each event's p times `weight`, a
    segmentation's membership, when given)"""
    B = len(s["sizes"])
    b, pix, dx, dy, keep = linvel_taps(s, v, flow)
    w = s["p"].astype(np.float64) * (1.0 if weight is None else np.asarray(weight, np.float64))
    return _splat(B, b, pix, dx, dy, keep, w)


def linvel_ts_images(s, v, flow=False):
    """(S, C) of the timestamp loss, each (B, 2, HC, WC) f64, polarity 0 positive"""
    B = len(s["sizes"])
    b, pix, dx, dy, keep = linvel_taps(s, v, flow)
    S, C = np.zeros((B, 2, HC, WC)), np.ones((B, 2, HC, WC))
    for i, sel in enumerate((s["p"] > 0, s["p"] <= 0)):
        S[:, i] = _splat(B, b, pix, dx, dy, keep & sel, s["tau"].astype(np.float64))
        C[:, i] += _splat(B, b, pix, dx, dy, keep & sel, np.ones(b.shape[0]))
    return S, C


def variance_f(iwe):
    """f of the variance objective at sigma 0, as the kernel forms it from its (exact) f64 sums"""
    P = float(HC * WC)
    m = iwe.sum(axis=(1, 2)) / P
    return -((iwe * iwe).sum(axis=(1, 2)) / P - m * m)


def timestamp_f(S, C):
    """f of the timestamp loss at sigma 0 (T = S / C rounded to f32, as the kernel's fold stores it)"""
    T = (S.astype(np.float32) / C.astype(np.float32)).astype(np.float64)
    return (T * T).sum(axis=(1, 2, 3)), T


def tap_magnitudes(s, v, flow=False):
    """per window and pixel: the sum of |tap| of the contrast image and the sum of |tau tap| of the timestamp images"""
    B = len(s["sizes"])
    b, pix, dx, dy, keep = linvel_taps(s, v, flow)
    ones = np.ones(b.shape[0])
    return _splat(B, b, pix, dx, dy, keep, ones), _splat(B, b, pix, dx, dy, keep, np.abs(s["tau"].astype(np.float64)))


def assert_exactly_summable(s, velocities, flow=False):
    """Every warped coordinate on the quarter grid, so every tap weight on the 1/16 grid (tau taps on the 1/256 grid),
    and per pixel sum |tap| <= 2^20 and sum |tau tap| <= 2^16: every partial sum of every image, in any order, is then
    an f32 value, and so is C = 1 + sum |tap|.  A segmentation's memberships on the 1/4 grid keep every tap on the
    1/64 grid and every sum below 2^20."""
    for v in velocities:
        _, _, dx, dy, keep = linvel_taps(s, v, flow)
        for a in (dx[keep], dy[keep]):
            assert (a * 4 == np.round(a * 4)).all(), v
        mag, tmag = tap_magnitudes(s, v, flow)
        assert mag.max() <= 2.0 ** 20 and tmag.max() <= 2.0 ** 16, (v, mag.max(), tmag.max())
        assert ((s["tau"].astype(np.float64) * 16) == np.round(s["tau"].astype(np.float64) * 16)).all()


def window_chunk(B, J, cap, per_window_bytes, budget):
    """the window chunk of motion_contrast_candidates_torch / motion_timestamp_candidates_torch (`_candidates` /
    `_ts_candidates`): wb = max(1, min(B, budget // per_window, cap // min(J, 32)))"""
    return max(1, min(B, budget // per_window_bytes, cap // min(J, MAX_CANDIDATES)))


def chunk_sizes(B, wb):
    return [min(wb, B - b0) for b0 in range(0, B, wb)]


def sampled_windows(sizes, giant, tail_images_per_window, seed=0, count=40):
    """0, 1, B-2, B-1, the giant and its neighbours, the nearest empty and one-event windows on either side of it, the
    windows whose tail index z crosses 2^15 and the last one, then seeded random windows up to `count`"""
    B = len(sizes)
    pick = {0, 1, B - 2, B - 1, giant, giant - 1, giant + 1}
    for want in (0, 1):
        below = np.flatnonzero(sizes[:giant] == want)
        above = np.flatnonzero(sizes[giant + 1:] == want)
        if below.size:
            pick.add(int(below[-1]))
        if above.size:
            pick.add(int(giant + 1 + above[0]))
    for z in ((1 << 15) - 1, 1 << 15, 65534):
        pick.add(z // tail_images_per_window)
    pick = {b for b in pick if 0 <= b < B}
    rng = np.random.default_rng(seed)
    while len(pick) < count:
        pick.add(int(rng.integers(0, B)))
    return np.array(sorted(pick))


# ---- the newer families: affine, homography, camera rotation, camera motion, grid flow, depth grid, segmentation ----
FAMILIES = ("affine", "homography", "camera_rotation", "camera_motion", "grid_flow", "depth_grid", "segmentation")
# every family but the camera rotation, which has no translation, reproduces the linvel warp exactly (exact_rows)
EXACT_FAMILIES = ("affine", "homography", "camera_motion", "grid_flow", "depth_grid", "segmentation")
FOCAL = 8.0                          # a power of two: (x - cx) / fx and fx X are exact
INTR = (FOCAL, FOCAL, 4.5, 2.5)      # fx, fy and a dyadic principal point
EXACT_RHOS = np.array([0.5, 1.0, 2.0])
# the depth grid's candidate nodes under motion rows built for rho 1 (exact_rows("camera_motion", vel, 1)): node rho r
# moves the events at r vel, a multiple of 16 for r in {1, 2}
DEPTH_CANDIDATE_RHOS = np.array([1.0, 2.0])
RANDOM_GRID = (3, 4)                 # the random variant's node grid: rx = 9/3 and ry = 5/2 are not dyadic
K = {"affine": 6, "homography": 8, "camera_rotation": 5, "camera_motion": 8, "segmentation": 6}


def _sensor_events(rng, n):
    x = rng.integers(0, 4 * (W - 1) + 1, n) / 4.0
    y = rng.integers(0, 4 * (H - 1) + 1, n) / 4.0
    d = -rng.integers(0, 5, n) / 64.0
    return x, y, d, rng.choice(np.array([-1.0, 1.0]), n), rng.integers(0, 17, n) / 16.0


def sensor_stream(B, giant_at=None, seed=0, M=None):
    """exact_stream for the newer families: every event on the quarter grid inside [0, W-1] x [0, H-1], where the grid
    families interpolate their nodes (a node tap outside the grid is zero), d on the 2^-6 grid in [-1/16, 0], so that
    under EXACT_VELOCITIES x' = x - d vx moves by at most 4 px and stays on the quarter grid; tau on the 1/16 grid and
    p = +-1.  The giant window's events come from their own seed, so the giant is the same window wherever it sits.
    Also `r`, each event's inverse depth: its window's rho of window_rhos(B, seed), and with M, `w`, memberships (n, M)
    on the 1/4 grid in [1/4, 1]."""
    sizes = window_sizes(B, giant_at, seed)
    off = _offsets(sizes)
    n = int(off[-1])
    x, y, d, p, tau = _sensor_events(np.random.default_rng(seed + 1), n)
    if giant_at is not None:
        sl = slice(off[giant_at], off[giant_at + 1])
        for a, v in zip((x, y, d, p, tau), _sensor_events(np.random.default_rng(seed + 2), GIANT)):
            a[sl] = v
    f = np.float32
    s = dict(x=x.astype(f), y=y.astype(f), d=d.astype(f), tau=tau.astype(f), p=p.astype(f), off=off, sizes=sizes)
    s["r"] = window_rhos(B, seed)[window_ids(off)].astype(f)
    if M is not None:
        s["w"] = (np.random.default_rng(seed + 3).integers(1, 5, (n, M)) / 4.0).astype(f)
    return s


def window_rhos(B, seed):
    """a constant inverse depth per window, of EXACT_RHOS"""
    return EXACT_RHOS[np.random.default_rng(seed + 4).integers(0, len(EXACT_RHOS), B)]


def exact_rows(family, vel, rho=None):
    """The family's parameters that reproduce the linvel warp at velocity vel ((B,2); the segmentation's (B,M,2)) bit
    for bit (tests/test_batch_limits_models_cpu.py proves it with the kernels' f32 restatements):
      affine, homography, segmentation (affine models): (hx, hy) = (vx, vy), every other term 0;
      camera_motion: w = 0, vz = 0, (vx, vy) = -vel / (FOCAL rho) for the window's rho, rows with (fx, fy);
      grid_flow: a uniform full-resolution grid (B,2,H,W) f32 of u = -vx, v = -vy;
      depth_grid: (motion rows (B,8) of camera_motion, a uniform full-resolution grid (B,H,W) f32 of rho)."""
    vel = np.asarray(vel, np.float64)
    if family in ("affine", "homography", "segmentation"):
        rows = np.zeros(vel.shape[:-1] + (K[family],))
        rows[..., :2] = vel
        return rows
    if family == "grid_flow":
        return np.broadcast_to(-vel[:, :, None, None], (vel.shape[0], 2, H, W)).astype(np.float32)
    rows = np.zeros((vel.shape[0], 8))
    rows[:, 3:5] = -vel / (FOCAL * np.asarray(rho, np.float64)[:, None])
    rows[:, 6:] = FOCAL
    if family == "camera_motion":
        return rows
    return rows, np.broadcast_to(np.asarray(rho, np.float64)[:, None, None], (vel.shape[0], H, W)).astype(np.float32)


def exact_velocity_set(shape, seed):
    """a velocity of EXACT_VELOCITIES per entry of `shape` (windows, models, candidates)"""
    vel = exact_velocities()
    return vel[np.random.default_rng(seed).integers(0, len(vel), shape)]


def random_stream_models(B, giant_at=None, seed=0, M=None):
    """random_stream with every event's inverse depth `r` in [1/8, 1] and, with M, random memberships `w` (n, M)"""
    s = random_stream(B, giant_at, seed)
    rng = np.random.default_rng(seed + 5)
    n = int(s["off"][-1])
    s["r"] = rng.uniform(0.125, 1.0, n).astype(np.float32)
    if M is not None:
        s["w"] = rng.random((n, M)).astype(np.float32)
    return s


def random_rows(family, B, seed, M=None):
    """The random variant's parameters, every term in play: a non-zero perspective, a non-zero w and vz, non-uniform
    node grids (RANDOM_GRID).  About a pixel of motion at |d| <= 0.1 on the 6x10 sensor.  grid_flow: (B,2,3,4) f32;
    depth_grid: (motion rows (B,8), nodes (B,3,4) f32 in [1/8, 1]); segmentation: (B,M,6) affine rows."""
    rng = np.random.default_rng(seed)
    gh, gw = RANDOM_GRID
    if family == "grid_flow":
        return rng.uniform(-20, 20, (B, 2, gh, gw)).astype(np.float32)
    shape = (B,) if M is None else (B, M)
    if family in ("affine", "homography", "segmentation"):
        a = [rng.uniform(-20, 20, shape + (2,)), rng.uniform(-3, 3, shape + (4,))]
        if family == "homography":
            a.append(rng.uniform(-0.3, 0.3, shape + (2,)))
        return np.concatenate(a, axis=-1)
    w = rng.uniform(-3, 3, (B, 3))
    if family == "camera_rotation":
        return np.column_stack((w, np.full((B, 2), FOCAL)))
    rows = np.column_stack((w, rng.uniform(-2, 2, (B, 3)), np.full((B, 2), FOCAL)))
    if family == "camera_motion":
        return rows
    return rows, rng.uniform(0.125, 1.0, (B, gh, gw)).astype(np.float32)


def family_warp(family, x, y, d, r, prm):
    """(x', y') of the events of one window under the family's parameters prm (the node grid for grid_flow, (motion
    row, nodes) for depth_grid) in the kernel's f32 order of operations: the warp whose distance from the integers
    decides whether f32 and f64 may take different taps"""
    import camera_motion_reference as CM
    import camera_rotation_reference as CR
    import depth_grid_reference as DR
    import grid_flow_reference as GR
    import planar_motion_reference as P
    with np.errstate(all="ignore"):
        if family in ("affine", "homography", "segmentation"):
            return P.warp_f32("affine" if family == "segmentation" else family, x, y, d, prm, CENTRE)
        if family == "camera_rotation":
            return CR.warp(x, y, d, prm[:3], tuple(prm[3:5]) + INTR[2:])
        if family == "camera_motion":
            return CM.warp(x, y, d, r, prm[:3], prm[3:6], tuple(prm[6:8]) + INTR[2:])
        if family == "grid_flow":
            u, v = GR.event_flow_f32(x, y, prm, H, W)
            return (x + u * d).astype(np.float32), (y + v * d).astype(np.float32)
        rows, nodes = prm
        r32 = DR.event_rho_f32(x, y, nodes, H, W)
        return CM.warp(x, y, d, r32, rows[:3], rows[3:6], tuple(rows[6:8]) + INTR[2:])


def drop_unsafe(s, family, windows, params, drop):
    """Give the events of `windows` that lie within 1e-3 px of an integer under any of `params` (a function of the
    window returning a list of the family's parameter sets) the polarity `drop`, which adds no term (0 for the
    contrast losses, NaN for the timestamp losses), so that f32 and the f64 references take the same taps and keep
    decisions there.  In place; returns the fraction of events dropped."""
    off, dropped, total = s["off"], 0, 0
    for b in windows:
        lo, hi = int(off[b]), int(off[b + 1])
        if hi == lo:
            continue
        ev = [s[k][lo:hi] for k in ("x", "y", "d")] + [s["r"][lo:hi]]
        bad = np.zeros(hi - lo, bool)
        for prm in params(b):
            xw, yw = family_warp(family, *ev, prm)
            with np.errstate(invalid="ignore"):
                bad |= np.isfinite(xw) & np.isfinite(yw) & ((np.abs(xw - np.round(xw)) < 1e-3) |
                                                            (np.abs(yw - np.round(yw)) < 1e-3))
        s["p"][lo:hi][bad] = drop
        dropped, total = dropped + int(bad.sum()), total + hi - lo
    return dropped / max(total, 1)


VOXEL_BINS = 5


def voxel_stream(n_windows, giant_at=None, seed=0):
    """dict x, y, t, p (float32), k (the stamp index), off, sizes"""
    sizes = window_sizes(n_windows, giant_at, seed)
    off = _offsets(sizes)
    n = int(off[-1])
    rng = np.random.default_rng(seed + 1)
    w = window_ids(off)
    t0 = (np.arange(n_windows) % 64).astype(np.float64)
    dt = 2.0 ** (np.arange(n_windows) % 4 - 1)
    k = rng.integers(0, 65, n)
    two = sizes >= 2
    k[off[:-1][two]] = 0
    k[off[1:][two] - 1] = 64
    t = t0[w] + dt[w] * k / 64.0
    x = rng.integers(0, W, n) + rng.integers(0, 4, n) / 4.0
    y = rng.integers(0, H, n) + rng.integers(0, 4, n) / 4.0
    p = rng.choice(np.array([-1.0, 1.0]), n)
    f = np.float32
    return dict(x=x.astype(f), y=y.astype(f), t=t.astype(f), p=p.astype(f), k=k, off=off, sizes=sizes)


def voxel_taps(s):
    """per event of a window of two or more events: (window, cell index of bin floor(tn), floor(tn), w0, w1, mask),
    tn = k / 16; bin floor(tn) gets p w0 and bin floor(tn) + 1 gets p w1 (if < VOXEL_BINS)"""
    w = window_ids(s["off"])
    mask = s["sizes"][w] >= 2
    tn = s["k"] / 16.0
    fl = np.floor(tn).astype(np.int64)
    pix = s["y"].astype(np.int64) * W + s["x"].astype(np.int64)
    return w, pix, fl, 1.0 - (tn - fl), tn - fl, mask


def voxel_grids(s):
    """(n_windows, VOXEL_BINS, H, W) f64 grids of the windows of two or more events (the others zero)"""
    nw, B = len(s["sizes"]), VOXEL_BINS
    w, pix, fl, w0, w1, mask = voxel_taps(s)
    p = s["p"].astype(np.float64)
    out = np.zeros(nw * B * H * W)
    for b, wt in ((fl, w0), (fl + 1, w1)):
        m = mask & (b < B)
        out += np.bincount(((w * B + b) * H * W + pix)[m], weights=(p * wt)[m], minlength=nw * B * H * W)
    return out.reshape(nw, B, H, W)


def voxel_grad_p(s, g):
    """grad_p of every event of the windows of two or more events (others NaN): sum_b g[b] max(0, 1 - |tn - b|)"""
    w, pix, fl, w0, w1, mask = voxel_taps(s)
    B = VOXEL_BINS
    gf = g.reshape(len(s["sizes"]), B, H * W).astype(np.float64)
    out = np.full(w.shape[0], np.nan)
    hi = np.minimum(fl + 1, B - 1)
    out[mask] = (gf[w, fl, pix] * w0 + np.where(fl + 1 < B, gf[w, hi, pix], 0.0) * w1)[mask]
    return out


def voxel_incoming(n_windows, seed):
    """an incoming gradient on the 1/16 grid in [-8, 8]: every per-event gradient and every f64 window sum of the
    backward is then exact"""
    return (np.random.default_rng(seed).integers(-128, 129, (n_windows, VOXEL_BINS, H, W)) / 16.0).astype(np.float32)
