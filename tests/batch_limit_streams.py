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


EVENT_KEYS = ("x", "y", "d", "tau", "p", "t", "k")


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


def linvel_taps(s, v):
    """the bilinear taps of every contributing event under linvel velocity v ((2,) or per window (B,2)), in f64: (window,
    pixel index y*WC+x of the top-left tap, dx, dy, keep).  Exact for exact_stream under a velocity of EXACT_VELOCITIES"""
    b = window_ids(s["off"])
    v = np.asarray(v, np.float64)
    vx, vy = (v[b, 0], v[b, 1]) if v.ndim == 2 else (v[0], v[1])
    xw = s["x"].astype(np.float64) - s["d"].astype(np.float64) * vx
    yw = s["y"].astype(np.float64) - s["d"].astype(np.float64) * vy
    keep = np.isfinite(xw) & np.isfinite(yw) & (xw > 0) & (xw < W) & (yw > 0) & (yw < H)
    px, py = np.floor(np.where(keep, xw, 0)), np.floor(np.where(keep, yw, 0))
    return b, (py * WC + px).astype(np.int64), xw - px, yw - py, keep


def _splat(B, b, pix, dx, dy, keep, w):
    img = np.zeros(B * HC * WC)
    base = b * HC * WC + pix
    for o, k in ((0, (1 - dx) * (1 - dy)), (1, dx * (1 - dy)), (WC, (1 - dx) * dy), (WC + 1, dx * dy)):
        img += np.bincount(base[keep] + o, weights=(w * k)[keep], minlength=B * HC * WC)
    return img.reshape(B, HC, WC)


def linvel_iwe(s, v):
    """(B, HC, WC) f64 images of p of the contrast loss under linvel velocity v"""
    B = len(s["sizes"])
    b, pix, dx, dy, keep = linvel_taps(s, v)
    return _splat(B, b, pix, dx, dy, keep, s["p"].astype(np.float64))


def linvel_ts_images(s, v):
    """(S, C) of the timestamp loss, each (B, 2, HC, WC) f64, polarity 0 positive"""
    B = len(s["sizes"])
    b, pix, dx, dy, keep = linvel_taps(s, v)
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


def tap_magnitudes(s, v):
    """per window and pixel: the sum of |tap| of the contrast image and the sum of |tau tap| of the timestamp images"""
    B = len(s["sizes"])
    b, pix, dx, dy, keep = linvel_taps(s, v)
    ones = np.ones(b.shape[0])
    return _splat(B, b, pix, dx, dy, keep, ones), _splat(B, b, pix, dx, dy, keep, np.abs(s["tau"].astype(np.float64)))


def assert_exactly_summable(s, velocities):
    """Every warped coordinate on the quarter grid, so every tap weight on the 1/16 grid (tau taps on the 1/256 grid),
    and per pixel sum |tap| <= 2^20 and sum |tau tap| <= 2^16: every partial sum of every image, in any order, is then
    an f32 value, and so is C = 1 + sum |tap|"""
    for v in velocities:
        _, _, dx, dy, keep = linvel_taps(s, v)
        for a in (dx[keep], dy[keep]):
            assert (a * 4 == np.round(a * 4)).all(), v
        mag, tmag = tap_magnitudes(s, v)
        assert mag.max() <= 2.0 ** 20 and tmag.max() <= 2.0 ** 16, (v, mag.max(), tmag.max())
        assert ((s["tau"].astype(np.float64) * 16) == np.round(s["tau"].astype(np.float64) * 16)).all()


def window_chunk(B, J, cap, per_window_bytes, budget):
    """the window chunk of motion_contrast_candidates_torch / motion_timestamp_candidates_torch (`_candidates` /
    `_ts_candidates`): wb = max(1, min(B, budget // per_window, cap // min(J, 32)))"""
    return max(1, min(B, budget // per_window_bytes, cap // min(J, MAX_CANDIDATES)))


def chunk_sizes(B, wb):
    return [min(wb, B - b0) for b0 in range(0, B, wb)]


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
