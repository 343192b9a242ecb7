"""The backward kernels of csrc/evk_grad.cu against the f64 references of tests/grad_reference.py, event by event:
within the derived per-event bound (exact_bounds.assert_within_grad_bound), or bit for bit on the exactly computable
streams of tests/edge_cases.py exact_grad_streams.  The C entry points are called directly, so that every launch path
runs: sizes around the vector width and the CTA slice, views misaligned by 1, 2 and 3 elements (alike and differently:
the scalar instantiations and the vector head/tail peel), every B from 1 to 17, the neg/pos and (N,4) layouts, more than
128 windows, windows split across CTAs at every start residue mod 4, one-event, empty and overlapping windows, and
20 M-event streams.  The public functions are checked with every non-empty subset of their differentiable inputs
requiring grad."""
import itertools

import numpy as np
import pytest
import torch

import grad_reference as G
from edge_cases import exact_grad_streams, hard_cases, replicate
from exact_bounds import (assert_exact, assert_exactly_summable, assert_scalar_within, assert_within_exact,
                          assert_within_grad_bound)

pytestmark = pytest.mark.gpu

SIZES = [1, 2, 3, 5, 7, 2047, 2049, 4 * 4096 - 1, 4 * 4096 + 1, 64 * 4096 - 1, 64 * 4096 + 1]
BIG = 20 << 20
WAVE = (1 << 20) + (1 << 18) + 3          # past one wave of every grid-stride backward on a 132-SM H100


def _lib():
    from event_utils_b200 import _lib
    return _lib


def ptr(t):
    return _lib().ptr(t)


def dev(a, off=0, dtype=torch.float32):
    """numpy array -> device view at element offset `off` of a fresh buffer (the allocator's buffers are 256-byte
    aligned: off = 0 is 16-byte aligned, 1..3 are not)."""
    a = np.ascontiguousarray(a)
    buf = torch.empty(a.size + off + 4, dtype=dtype, device="cuda")
    v = buf[off:off + a.size].view(a.shape)
    v.copy_(torch.from_numpy(a).to(dtype))
    return v


def out(n, off=0):
    """An output view prefilled with NaN: an event the kernel does not write shows up as NaN."""
    buf = torch.full((n + off + 4,), float("nan"), device="cuda")
    return buf[off:off + n]


def host(t):
    torch.cuda.synchronize()
    return t.cpu().numpy().astype(np.float64)


# offsets of the (inputs..., outputs...) views: aligned, all alike misaligned by 1 / 2 / 3, misaligned differently
def offsets(k, n=0):
    """Every offset pattern up to 2 x 4096 + 1 events, where the size still changes the launch shape (the vector
    body, the head / tail peel, the number of CTAs); beyond, aligned and one differently misaligned pattern."""
    mixed = tuple((i % 4) for i in range(k))
    if n > 2 * 4096 + 1:
        return [(0,) * k, mixed]
    return [(0,) * k, (1,) * k, (2,) * k, (3,) * k, mixed, (0,) * (k - 1) + (3,), (1,) + (0,) * (k - 1)]


def _events(n, seed, H, W, spread=1.5):
    """Events around and beyond the borders with exact integers and ulp-off borders."""
    rng = np.random.default_rng(seed)
    x = rng.uniform(-spread, W - 1 + spread, n).astype(np.float32)
    y = rng.uniform(-spread, H - 1 + spread, n).astype(np.float32)
    snap = rng.random(n) < 0.15
    x[snap], y[snap] = np.floor(x[snap]), np.floor(y[snap])
    sp = rng.random(n) < 0.05
    x[sp] = rng.choice(np.array([W - 1, np.nextafter(np.float32(W), np.float32(0)), -0.0, -2.0 ** -24], np.float32),
                       int(sp.sum()))
    t = np.sort(rng.random(n)).astype(np.float32)
    p = rng.choice(np.array([1.0, -1.0, 0.0, 0.37, 2.0 ** 20], np.float32), n)
    return x, y, t, p


# ---- event image -------------------------------------------------------------------------------------------------------
def run_image(x, y, p, g, bil, clip, clipx, clipy, offs=(0,) * 6):
    L, lib = _lib().lib(), _lib()
    n = x.shape[0]
    H, W = g.shape
    X, Y, P = dev(x, offs[0]), dev(y, offs[1]), dev(p, offs[2])
    outs = [out(n, o) for o in offs[3:]]
    flags = (lib.BILINEAR if bil else 0) | (lib.CLIP if clip else 0)
    Gd = dev(g)                    # held until the results are read: a freed buffer may be handed out again
    lib.check(L.evk_image_grad_f32(ptr(X), ptr(Y), ptr(P), n, H, W, clipx, clipy, flags, ptr(Gd),
                                   *(ptr(o) for o in outs), lib.stream()))
    return dict(zip(("gx", "gy", "gp"), (host(o) for o in outs)))


@pytest.mark.parametrize("bil", [True, False], ids=["bilinear", "nearest"])
def test_image_sizes_and_alignments(bil):
    H, W = 21, 29
    for n in SIZES:
        clip = n % 2 == 1
        x, y, t, p = _events(n, n, H, W)
        g = np.random.default_rng(n).standard_normal((H, W)).astype(np.float32)
        ref = G.image_grad(x, y, p, g, clip, W - 1.0, H - 1.0, bil)
        for offs in offsets(6, n):
            got = run_image(x, y, p, g, bil, clip, W - 1.0, H - 1.0, offs)
            for k, r in ref.items():
                assert_within_grad_bound(got[k], r, "image %s n=%d offs=%s %s" % (bil, n, offs, k))
            if not bil:
                assert np.isnan(got["gx"]).all() and np.isnan(got["gy"]).all(), "nearest writes no coordinate gradient"


def test_image_exact_streams():
    """Bit for bit, 4095 events and a 20 M-event tiling of a 1 M-event stream."""
    for n, reps in ((4095, 1), (1 << 20, 20)):
        s = exact_grad_streams(7, "image", n)
        ref = G.image_grad(s["x"], s["y"], s["p"], s["g"], True, s["W"] - 1.0, s["H"] - 1.0)
        t = lambda a: np.tile(a, reps)
        got = run_image(t(s["x"]), t(s["y"]), t(s["p"]), s["g"], True, True, s["W"] - 1.0, s["H"] - 1.0)
        for k, r in ref.items():
            v = t(r.v)
            assert_exact(got[k], G.Exact(v, np.abs(v), np.ones_like(v)), what="image exact n=%d %s" % (n * reps, k))


# ---- timestamp images ----------------------------------------------------------------------------------------------
def run_tsimg(x, y, t, p, t_first, t_last, gpos, gneg, clip, reverse, H, W, offs=(0,) * 7):
    L, lib = _lib().lib(), _lib()
    n = x.shape[0]
    flags = (lib.CLIP if clip else 0) | (lib.TS_REVERSE if reverse else 0)
    Xa, Ya, Ta, Pa = (dev(a) for a in (x, y, t, p))
    imgs = [torch.empty((H, W), device="cuda") for _ in range(4)]
    ws = torch.empty(L.evk_timestamp_image_workspace_bytes(H, W), dtype=torch.uint8, device="cuda")
    oob = torch.zeros(1, dtype=torch.int64, device="cuda")
    lib.check(L.evk_timestamp_image_counts_f32(ptr(Xa), ptr(Ya), ptr(Ta), ptr(Pa), n, t_first, t_last, H, W, W - 1.0,
                                               H - 1.0, flags, *(ptr(i) for i in imgs), ptr(ws), ws.numel(), ptr(oob),
                                               None))
    X, Y, T, P = (dev(a, o) for a, o in zip((x, y, t, p), offs))
    outs = [out(n, o) for o in offs[4:]]
    sums = torch.empty(2, dtype=torch.float64, device="cuda")
    gws = torch.empty(L.evk_timestamp_image_grad_workspace_bytes(H, W), dtype=torch.uint8, device="cuda")
    Gp, Gn = dev(gpos), dev(gneg)
    lib.check(L.evk_timestamp_image_grad_f32(ptr(X), ptr(Y), ptr(T), ptr(P), n, t_first, t_last, H, W, W - 1.0, H - 1.0,
                                             flags, ptr(Gp), ptr(Gn), ptr(imgs[0]), ptr(imgs[1]),
                                             ptr(imgs[2]), ptr(imgs[3]), *(ptr(o) for o in outs), ptr(sums), ptr(gws),
                                             gws.numel(), None))
    r = dict(zip(("gx", "gy", "gt"), (host(o) for o in outs)))
    r["sums"] = host(sums)
    return r


def check_tsimg(got, ref, what):
    for k in ("gx", "gy", "gt"):
        assert_within_grad_bound(got[k], ref[k], "%s %s" % (what, k))
    assert_scalar_within(got["sums"][0], *ref["s0"], what=what + " sum g_tn")
    assert_scalar_within(got["sums"][1], *ref["s1"], what=what + " sum g_tn tn")


def test_tsimg_sizes_and_alignments():
    H, W = 22, 30
    for n in SIZES:
        clip, reverse = n % 2 == 1, n % 3 == 0
        x, y, t, p = _events(n, 100 + n, H - 1, W - 1)
        p[np.random.default_rng(n).random(n) < 0.03] = np.nan
        rng = np.random.default_rng(n + 1)
        gpos, gneg = (rng.standard_normal((H, W)).astype(np.float32) for _ in range(2))
        ref = G.tsimg_grad(x, y, t, p, t[0], t[-1], gpos, gneg, clip, W - 1.0, H - 1.0, reverse)
        for offs in offsets(7, n):
            got = run_tsimg(x, y, t, p, float(t[0]), float(t[-1]), gpos, gneg, clip, reverse, H, W, offs)
            check_tsimg(got, ref, "tsimg n=%d offs=%s" % (n, offs))


def test_tsimg_20m():
    """A 20 M-event tiling of a 1 M-event stream: per-event values against the reference of one copy, the sums
    against 20 times its sums."""
    H, W = 181, 241
    x, y, t, p = _events(1 << 20, 5, H - 1, W - 1)
    rng = np.random.default_rng(6)
    gpos, gneg = (rng.standard_normal((H, W)).astype(np.float32) for _ in range(2))
    reps = BIG // (1 << 20)
    ref = G.tsimg_grad(x, y, t, p, t[0], t[-1], gpos, gneg, True, W - 1.0, H - 1.0, reps=reps)
    got = run_tsimg(*(np.tile(a, reps) for a in (x, y, t, p)), float(t[0]), float(t[-1]), gpos, gneg, True, False, H, W)
    tiled = {k: G.Grad(*(np.tile(np.broadcast_to(a, ref[k].v.shape), reps) for a in ref[k])) for k in ("gx", "gy", "gt")}
    check_tsimg(got, dict(ref, **tiled), "tsimg 20M")


# ---- flow warp -----------------------------------------------------------------------------------------------------------
def run_warp(x, y, t, flow, gxw, gyw, t0=0.0, offs=(0,) * 8):
    L, lib = _lib().lib(), _lib()
    n = x.shape[0]
    H, W = flow.shape[1:]
    ins = [dev(a, o) for a, o in zip((x, y, t, gxw, gyw), offs)]
    outs = [out(n, o) for o in offs[5:]]
    gf = torch.empty((2, H, W), device="cuda")
    s = torch.empty(1, dtype=torch.float64, device="cuda")
    ws = torch.empty(L.evk_warp_flow_grad_workspace_bytes(H, W), dtype=torch.uint8, device="cuda")
    F = dev(flow)
    lib.check(L.evk_warp_flow_grad_f32(ptr(ins[0]), ptr(ins[1]), ptr(ins[2]), n, ptr(F), H, W, t0, ptr(ins[3]),
                                       ptr(ins[4]), *(ptr(o) for o in outs), ptr(gf), ptr(s), ptr(ws), ws.numel(), None))
    r = dict(zip(("gx", "gy", "gt"), (host(o) for o in outs)))
    r["flow"], r["sum_gt"] = host(gf), host(s)[0]
    return r


def check_warp(got, ref, x, y, t, t0, gxw, gyw, H, W, what):
    for k in ("gx", "gy", "gt"):
        assert_within_grad_bound(got[k], ref[k], "%s %s" % (what, k))
    assert_scalar_within(got["sum_gt"], *ref["sum_gt"], what=what + " sum gt")
    tr = (t - np.float32(t0)).astype(np.float32)
    assert_within_exact(got["flow"], G.flow_grad_exact(x, y, tr, gxw, gyw, H, W), what=what + " flow")


def test_warp_sizes_and_alignments():
    H, W = 23, 31
    for n in SIZES:
        x, y, t, _ = _events(n, 200 + n, H, W, spread=2.0)
        rng = np.random.default_rng(n)
        flow = (rng.standard_normal((2, H, W)) * 5).astype(np.float32)
        gxw, gyw = (rng.standard_normal(n).astype(np.float32) for _ in range(2))
        t0 = float(t[n // 2])
        ref = G.warp_grad(x, y, t, flow, gxw, gyw, t0)
        for offs in offsets(8, n):
            got = run_warp(x, y, t, flow, gxw, gyw, t0, offs)
            check_warp(got, ref, x, y, t, t0, gxw, gyw, H, W, "warp n=%d offs=%s" % (n, offs))


def test_warp_border_fields_and_one_footprint():
    """Fields of 2 x W and H x 2, where every footprint touches the border, and one footprint taking a million events."""
    n = 300001
    for H, W in ((2, 37), (41, 2), (2, 2)):
        x, y, t, _ = _events(n, H * 100 + W, H, W, spread=1.0)
        rng = np.random.default_rng(H + W)
        flow = (rng.standard_normal((2, H, W)) * 5).astype(np.float32)
        gxw, gyw = (rng.standard_normal(n).astype(np.float32) for _ in range(2))
        ref = G.warp_grad(x, y, t, flow, gxw, gyw, 0.5)
        check_warp(run_warp(x, y, t, flow, gxw, gyw, 0.5), ref, x, y, t, 0.5, gxw, gyw, H, W, "warp %dx%d" % (H, W))
    n, H, W = 1 << 20, 24, 32
    rng = np.random.default_rng(9)
    x = np.full(n, 13.25, np.float32)
    y = np.full(n, 7.625, np.float32)
    t = rng.random(n).astype(np.float32)
    flow = (rng.standard_normal((2, H, W)) * 5).astype(np.float32)
    gxw, gyw = (rng.standard_normal(n).astype(np.float32) for _ in range(2))
    ref = G.warp_grad(x, y, t, flow, gxw, gyw, 0.25)
    check_warp(run_warp(x, y, t, flow, gxw, gyw, 0.25), ref, x, y, t, 0.25, gxw, gyw, H, W, "warp one footprint")


def test_warp_exact_streams():
    """Bit for bit: per-event outputs, sum grad_t (> 24 significant bits, so f32 accumulation would differ) and, where
    every partial sum of a cell is exact in any order (assert_exactly_summable), the flow cells.  A 20 M-event tiling
    of the 1 M-event stream checks the per-event values and the sum."""
    for n, reps in ((200003, 1), (1 << 20, 20)):
        s = exact_grad_streams(11, "warp", n)
        ref = G.warp_grad(s["x"], s["y"], s["t"], s["flow"], s["gxw"], s["gyw"])
        S = ref["sum_gt"][0] * reps
        assert np.float64(np.float32(S)) != S, "sum grad_t fits in f32"
        ti = lambda a: np.tile(a, reps)
        got = run_warp(ti(s["x"]), ti(s["y"]), ti(s["t"]), s["flow"], ti(s["gxw"]), ti(s["gyw"]))
        for k in ("gx", "gy", "gt"):
            v = ti(ref[k].v)
            assert_exact(got[k], G.Exact(v, np.abs(v), np.ones_like(v)), what="warp exact %s" % k)
        assert got["sum_gt"] == S, (got["sum_gt"], S)
        if reps == 1:
            ex = assert_exactly_summable(
                lambda m: G.flow_grad_exact(s["x"][m], s["y"][m], s["t"][m], s["gxw"][m], s["gyw"][m], s["H"], s["W"]),
                np.zeros(n, int), 0, g_fine=7, what="flow cells")
            assert_exact(got["flow"], ex[0], what="warp exact flow")


# ---- voxel grid ----------------------------------------------------------------------------------------------------------
def run_voxel(x, y, t, p, B, g, pairs=None, negpos=False, overlap=False, aos=False, offs=(0,) * 6, want=("gp", "gt")):
    L, lib = _lib().lib(), _lib()
    n = x.shape[0]
    nw = 1 if pairs is None else len(pairs)
    H, W = g.shape[-2:]
    flags = ((lib.WINDOW_NEGPOS if negpos else 0) | (lib.WINDOW_OVERLAP if overlap else 0) |
             (lib.EVENTS_AOS if aos else 0))
    if aos:
        rec = dev(np.stack([x, y, t, p], 1))
        ins = [rec, None, None, None]
    else:
        ins = [dev(a, o) for a, o in zip((x, y, t, p), offs)]
    gp = out(n, offs[4]) if "gp" in want else None
    gt = out(n, offs[5]) if "gt" in want else None
    pr = None if pairs is None else dev(np.asarray(pairs, np.int64), dtype=torch.int64)
    ws = torch.empty(L.evk_voxel_grad_workspace_bytes(nw, B, H, W, flags), dtype=torch.uint8, device="cuda")
    Gd = dev(g)
    lib.check(L.evk_voxel_grad_f32(*(ptr(a) for a in ins), n, ptr(pr), nw, B, H, W, flags, ptr(Gd), ptr(gp), ptr(gt),
                                   ptr(ws), ws.numel(), None))
    return {k: (host(v) if v is not None else None) for k, v in (("gp", gp), ("gt", gt))}


def check_voxel(got, ref, what, negpos=False):
    if negpos:
        assert np.isnan(got["gp"]).all(), what + ": the neg/pos backward writes no ps gradient"
    elif got["gp"] is not None:
        assert_within_grad_bound(got["gp"], ref["gp"], what + " gp")
    if got["gt"] is not None:
        assert_within_grad_bound(got["gt"], ref["gt"], what + " gt")


def _voxel_g(rng, nw, grids, B, H, W):
    return rng.standard_normal((nw, grids, B, H, W)).astype(np.float32)


def test_voxel_every_B_and_layout():
    """B = 1 .. 17 (rows of 4 .. 20 floats), single grid, neg/pos and (N,4) records, aligned and misaligned."""
    H, W = 9, 13
    for B in range(1, 18):
        n = 4097 + B
        x, y, t, p = _events(n, B, H, W, spread=W)
        rng = np.random.default_rng(B)
        for negpos in (False, True):
            g = _voxel_g(rng, 1, 2 if negpos else 1, B, H, W)
            ref = G.voxel_grad(x, y, t, p, B, g, negpos=negpos)
            for offs in offsets(6)[:5]:
                check_voxel(run_voxel(x, y, t, p, B, g, negpos=negpos, offs=offs), ref,
                            "voxel B=%d negpos=%s offs=%s" % (B, negpos, offs), negpos)
            if not negpos:
                # aligned outputs: the 16-byte record loads; misaligned ones: the scalar (N,4) instantiation
                for offs in ((0,) * 6, (0, 0, 0, 0, 1, 3)):
                    check_voxel(run_voxel(x, y, t, p, B, g, aos=True, offs=offs), ref, "voxel B=%d aos %s" % (B, offs))


def test_voxel_sizes_and_alignments():
    H, W, B = 10, 14, 5
    for n in SIZES:
        x, y, t, p = _events(n, 300 + n, H, W, spread=W)
        g = _voxel_g(np.random.default_rng(n), 1, 1, B, H, W)
        ref = G.voxel_grad(x, y, t, p, B, g)
        for offs in offsets(6, n):
            check_voxel(run_voxel(x, y, t, p, B, g, offs=offs), ref, "voxel n=%d offs=%s" % (n, offs))


def _windows(rng, n):
    """More than 128 windows over n events: one-event and empty windows, short ones, and windows of 2 x 2048 and more
    events starting at every residue mod 4.  The windows average more than 2048 events, so the big ones are split
    across several CTAs, each with a scalar head and tail."""
    cuts, pos, nbig = [], 0, 0
    for i in range(200):
        k = ("big", "big", "big", "one", "big", "empty", "big", "small")[i % 8]
        if k == "big":
            pos += (nbig - pos) % 4                      # start at residue nbig mod 4
            nbig += 1
        size = {"big": 4096 + int(rng.integers(1, 4000)), "one": 1, "empty": 0, "small": int(rng.integers(2, 700))}[k]
        if pos + size > n:
            break
        cuts.append((pos, pos + size))
        pos += size
    cuts = np.array(cuts, np.int64)
    big = cuts[cuts[:, 1] - cuts[:, 0] > 4096]
    assert len(cuts) > 128 and set(big[:, 0] % 4) == {0, 1, 2, 3} and n / len(cuts) > 2048
    return cuts


def _exact_voxel_expected(s, ref, pairs):
    """The kernel's gt on an exact stream: each window's end terms (f64, exactly summed) cast to f32 and added in f32 to
    the exact per-event value."""
    gt = ref["gt"].v.astype(np.float32)
    with np.errstate(all="ignore"):                       # one-event windows: dt = 0, NaN
        for (first, last), ((S0, _), (S1, _)) in zip(pairs, ref["sums"]):
            if last <= first:
                continue
            dt = np.float64(np.float32(s["t"][last - 1] - s["t"][first]))
            bm1 = np.float64(s["B"] - 1)
            gt[first] = np.float32(gt[first] + np.float32((S1 - bm1 * S0) / dt))
            gt[last - 1] = np.float32(gt[last - 1] + np.float32(-S1 / dt))
    return gt


def _exact_check(got, s, ref, pairs, what, negpos=False):
    if not negpos:
        v = ref["gp"].v
        assert_exact(got["gp"], G.Exact(v, np.abs(v), np.ones_like(v)), what=what + " gp")
    gt = _exact_voxel_expected(s, ref, pairs).astype(np.float64)
    assert_exact(got["gt"], G.Exact(gt, np.abs(gt), np.ones_like(gt)), what=what + " gt")


def test_voxel_windows_exact():
    """Bit for bit on an exact stream cut into > 128 windows (empty, one-event, and split across CTAs at every start
    residue): single grid, neg/pos and (N,4) records, aligned and misaligned; also every window against the bound."""
    rng = np.random.default_rng(41)
    n = 800000
    pairs = _windows(rng, n)
    s = exact_grad_streams(41, "voxel", n, windows=pairs)
    for negpos in (False, True):
        g = s["g"] if not negpos else np.concatenate([s["g"], s["g"][:, :, ::-1]], 1)
        ref = G.voxel_grad(s["x"], s["y"], s["t"], s["p"], s["B"], g, pairs=pairs, negpos=negpos, want_gt=False)
        full = G.voxel_grad(s["x"], s["y"], s["t"], s["p"], s["B"], g, pairs=pairs, negpos=negpos)
        for offs in offsets(6)[:5]:
            got = run_voxel(s["x"], s["y"], s["t"], s["p"], s["B"], g, pairs, negpos=negpos, offs=offs)
            what = "windows negpos=%s offs=%s" % (negpos, offs)
            _exact_check(got, s, ref, pairs, what, negpos)
            check_voxel(got, full, what, negpos)
        if not negpos:
            for offs in ((0,) * 6, (0, 0, 0, 0, 3, 1)):
                got = run_voxel(s["x"], s["y"], s["t"], s["p"], s["B"], g, pairs, aos=True, offs=offs)
                _exact_check(got, s, ref, pairs, "windows aos %s" % (offs,))


def test_voxel_one_window_exact_20m():
    """One window of 20 M events (a tiling of a 1 M-event stream that starts at t = 0 and ends at t = 1): per event bit
    for bit, and the end stamps, whose sums sum G and sum G tn need more than 24 significant bits: summed or combined
    in f32 they would give another first stamp."""
    base = exact_grad_streams(47, "voxel", 1 << 20)
    reps = BIG // (1 << 20)
    ref = G.voxel_grad(base["x"], base["y"], base["t"], base["p"], base["B"], base["g"], want_gt=False)
    (S0, _), (S1, _) = ref["sums"][0]
    S0, S1 = S0 * reps, S1 * reps
    assert np.float32(S0) != S0 and np.float32(S1) != S1, "the window sums fit in f32"
    g0, bm1 = np.float32(ref["gt"].v[0]), np.float32(base["B"] - 1)
    assert np.float32(g0 + np.float32(S1 - float(bm1) * S0)) != np.float32(g0 + (np.float32(S1) - bm1 * np.float32(S0))), \
        "the first stamp does not tell f64 from f32 end-stamp sums"
    x, y, t, p = (np.tile(base[k], reps) for k in "xytp")
    got = run_voxel(x, y, t, p, base["B"], base["g"])
    tiled = dict(gp=G.Grad(np.tile(ref["gp"].v, reps), 0, 0, 0), gt=G.Grad(np.tile(ref["gt"].v, reps), 0, 0, 0),
                 sums=[((S0, 0), (S1, 0))])
    _exact_check(got, dict(base, t=t), tiled, np.array([[0, t.shape[0]]]), "voxel 20M")


def test_voxel_overlapping_windows():
    """EVK_WINDOW_OVERLAP: windows that share events, heads and tails included: > 128 short ones (one CTA each), and a
    few long ones split across many CTAs, whose per-event outputs are then added atomically by several slices."""
    H, W, B = 8, 11, 4
    n = 200000
    x, y, t, p = _events(n, 51, H, W, spread=W)
    rng = np.random.default_rng(52)
    starts = np.sort(rng.integers(0, n - 5000, 160))
    pairs = np.stack([starts, starts + rng.integers(1, 5000, 160)], 1).astype(np.int64)
    pairs[:3] = [[5, 5], [7, 8], [1, 4099]]
    g = _voxel_g(rng, len(pairs), 1, B, H, W)
    ref = G.voxel_grad(x, y, t, p, B, g, pairs=pairs)
    for offs in offsets(6)[:5]:
        check_voxel(run_voxel(x, y, t, p, B, g, pairs, overlap=True, offs=offs), ref, "overlap offs=%s" % (offs,))
    check_voxel(run_voxel(x, y, t, p, B, g, pairs, overlap=True, aos=True), ref, "overlap aos")
    long_ = np.array([[1, 60002], [30001, 90003], [45002, 150001], [149999, 199998], [3, 199997]], np.int64)
    g = _voxel_g(rng, len(long_), 1, B, H, W)
    ref = G.voxel_grad(x, y, t, p, B, g, pairs=long_)
    for offs in offsets(6)[:5]:
        check_voxel(run_voxel(x, y, t, p, B, g, long_, overlap=True, offs=offs), ref, "long overlap offs=%s" % (offs,))


def test_voxel_hard_cases():
    """hard_cases with non-finite polarities: unsorted stamps (tn outside [0, B-1] and beyond 1e9), +-inf and NaN,
    -0.0 and +-2^20; as given, replicated past the vector threshold (4099) and, for a few, past one wave."""
    for c in hard_cases(31, 24, nonfinite=True):
        k = int(c["k"])
        B = 1 + k % 17
        sizes = [c["x"].shape[0], 4099] + ([WAVE] if k == 3 else [])
        for n in sizes:
            cc = replicate(c, n)
            g = _voxel_g(np.random.default_rng(k), 1, 2, B, c["H"], c["W"])
            for negpos in (False, True):
                gg = g if negpos else g[:, :1]
                ref = G.voxel_grad(cc["x"], cc["y"], cc["t"], cc["p"], B, gg, negpos=negpos)
                check_voxel(run_voxel(cc["x"], cc["y"], cc["t"], cc["p"], B, gg, negpos=negpos,
                                      offs=(k % 4,) * 6), ref, "hard k=%d n=%d negpos=%s" % (k, n, negpos), negpos)


def test_hard_cases_past_one_wave():
    """The existing hard-case kinds (image, timestamp images, warp) replicated past one wave of their kernels."""
    for c in list(hard_cases(31, 24, nonfinite=False))[1::8]:
        cc = replicate(c, WAVE)
        x, y, p = cc["x"], cc["y"], cc["p"]
        t = np.sort(cc["t"])
        H, W = c["H"] + 1, c["W"] + 1
        rng = np.random.default_rng(int(c["k"]))
        g = rng.standard_normal((H, W)).astype(np.float32)
        ref = G.image_grad(x, y, p, g, True, W - 1.0, H - 1.0)
        got = run_image(x, y, p, g, True, True, W - 1.0, H - 1.0)
        for k2, r in ref.items():
            assert_within_grad_bound(got[k2], r, "hard image k=%s %s" % (c["k"], k2))
        gneg = rng.standard_normal((H, W)).astype(np.float32)
        ref = G.tsimg_grad(x, y, t, p, t[0], t[-1], g, gneg, True, W - 1.0, H - 1.0)
        check_tsimg(run_tsimg(x, y, t, p, float(t[0]), float(t[-1]), g, gneg, True, False, H, W), ref,
                    "hard tsimg k=%s" % c["k"])
        flow = (rng.standard_normal((2, c["H"], c["W"])) * 3).astype(np.float32)
        gxw, gyw = (rng.standard_normal(WAVE).astype(np.float32) for _ in range(2))
        ref = G.warp_grad(x, y, t, flow, gxw, gyw, float(t[-1]))
        check_warp(run_warp(x, y, t, flow, gxw, gyw, float(t[-1])), ref, x, y, t, t[-1], gxw, gyw, c["H"], c["W"],
                   "hard warp k=%s" % c["k"])


# ---- the public functions: every subset of the differentiable inputs ------------------------------------------------
def _subsets(names):
    return [s for r in range(1, len(names) + 1) for s in itertools.combinations(names, r)]


def _public(kind, opts, a, req, B=None, negpos=False):
    from event_utils_b200.representations.image import events_to_image_torch, events_to_timestamp_image_torch
    from event_utils_b200.representations.voxel_grid import events_to_neg_pos_voxel_torch, events_to_voxel_torch
    from event_utils_b200.transforms.optic_flow import warp_events_flow_torch
    leaves = {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in a.items()}
    for k in req:
        leaves[k].requires_grad_(True)
    L = leaves
    if kind == "image":
        outs = (events_to_image_torch(L["xs"], L["ys"], L["ps"], **opts),)
    elif kind == "tsimg":
        outs = events_to_timestamp_image_torch(L["xs"], L["ys"], L["ts"], L["ps"], **opts)
    elif kind == "warp":
        outs = warp_events_flow_torch(L["xs"], L["ys"], L["ts"], L["ps"], L["flow"], t0=L.get("t0"))
    elif negpos:
        outs = events_to_neg_pos_voxel_torch(L["xs"], L["ys"], L["ts"], L["ps"], B, sensor_size=opts["sensor_size"])
    else:
        outs = (events_to_voxel_torch(L["xs"], L["ys"], L["ts"], L["ps"], B, sensor_size=opts["sensor_size"]),)
    rng = np.random.default_rng(len(req))
    weights = [rng.standard_normal(tuple(o.shape)).astype(np.float32) for o in outs]
    sum((o * torch.from_numpy(w).cuda()).sum() for o, w in zip(outs, weights)).backward()
    return weights, {k: leaves[k].grad for k in leaves}


@pytest.mark.parametrize("kind", ["image_bil", "image_nearest", "tsimg", "warp", "warp_t0", "voxel", "negpos"])
def test_every_subset_requiring_grad(kind):
    n, H, W = 6001, 19, 27
    x, y, t, p = _events(n, 61, H, W)
    a = dict(xs=x, ys=y, ts=t, ps=np.where(np.isfinite(p), p, 1).astype(np.float32))
    B, negpos, opts = None, kind == "negpos", dict(sensor_size=(H, W))
    if kind == "image_bil":
        fn, names, opts = "image", ["xs", "ys", "ps"], dict(sensor_size=(H, W), interpolation='bilinear', padding=True,
                                                            clip_out_of_range=True)
    elif kind == "image_nearest":
        fn, names = "image", ["ps"]
        opts.update(interpolation=None, padding=False, clip_out_of_range=True)
    elif kind == "tsimg":
        fn, names = "tsimg", ["xs", "ys", "ts"]
        opts.update(clip_out_of_range=True, padding=True, timestamp_reverse=True)
    elif kind.startswith("warp"):
        fn, names = "warp", ["xs", "ys", "ts", "flow"]
        a["flow"] = (np.random.default_rng(62).standard_normal((2, H, W)) * 5).astype(np.float32)
        if kind == "warp_t0":
            a["t0"] = np.array(t[n // 3], np.float32)
            names.append("t0")
    else:
        fn, B = "voxel", 7
        # pixels in [-size, size): the public grids raise IndexError beyond, as the reference does
        a["xs"] = np.clip(a["xs"] * 2 - W, -W, W - 1).astype(np.float32)
        a["ys"] = np.clip(a["ys"] * 2 - H, -H, H - 1).astype(np.float32)
        names = ["ts"] if negpos else ["ts", "ps"]
    for req in _subsets(names):
        weights, grads = _public(fn, opts, a, req, B=B, negpos=negpos)
        ref = G.public_grads(fn, a, weights, opts, B=B, negpos=negpos)
        for k in set(a) | set(names):
            what = "%s requires %s: %s" % (kind, req, k)
            if k not in req:
                assert grads.get(k) is None, what + " got a gradient"
                continue
            got = grads[k]
            assert got is not None, what + " got none"
            got = got.cpu().numpy()
            if k == "flow":
                assert_within_exact(got, ref[k], what=what)
            else:
                assert_within_grad_bound(got, ref[k], what)
