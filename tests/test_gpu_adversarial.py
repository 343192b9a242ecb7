"""Every scatter entry point, every variant, on the hard edge cases (tests/edge_cases.py hard_cases), small and tiled
past the size at which AUTO switches to the contended-stream kernels -- each output checked CELL BY CELL against the
oracle's exact per-cell sums (exact_bounds.assert_within_exact: |gpu - exact| <= gamma(k+4) S + k q), and the
out-of-range counts exactly.  A tap that is lost, doubled or sent to the wrong cell shows up in the cell it belongs to,
however hot the rest of the image is."""
import os

import numpy as np
import pytest
import torch

from exact_bounds import Q22, assert_within_exact
from edge_cases import hard_cases, replicate

pytestmark = pytest.mark.gpu

SMALL = list(hard_cases(31, 24))
# tiled past AUTO's thresholds: voxel quad / hot table at 2^20 events, image hot kernel at 2^18, cmax on-chip at 4 * 2^20
BIG_FROM = [c for c in SMALL if c["k"] % 6 == 0]
VOXEL_BIG, IMAGE_BIG, CMAX_BIG = (1 << 20) + 3, (1 << 18) + 5, (4 << 20) + 3


def _cases(big, n):
    return [replicate(c, n) for c in BIG_FROM] if big else SMALL


def dev(a, offset=0):
    """Device copy of a numpy array; offset > 0: a view `offset` elements into a larger buffer (not 16-byte aligned)."""
    a = np.ascontiguousarray(a)
    if not offset:
        return torch.from_numpy(a).cuda()
    buf = torch.zeros(a.shape[0] + offset, dtype=torch.from_numpy(a[:0]).dtype, device="cuda")
    buf[offset:] = torch.from_numpy(a).cuda()
    return buf[offset:]


def _p(t):
    return t.data_ptr() if t is not None else None


def _lib():
    from event_utils_b200 import _lib
    return _lib, _lib.lib()


def _sel(ex, k):
    return type(ex)(*(a[k] for a in ex))


def _voxel_variants():
    _l, _ = _lib()
    v = [("auto", _l.VARIANT_AUTO), ("global_red", _l.VARIANT_GLOBAL_RED), ("vector_red", _l.VARIANT_VECTOR_RED),
         ("smem_tile", _l.VARIANT_SMEM_TILE)]
    if os.environ.get("EVK_TEST_ROUTED", "1") != "0":
        v.append(("routed", _l.VARIANT_ROUTED))
    return v


# ---- voxel grids -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("big", [False, True])
def test_voxel(oracle, big):
    _l, L = _lib()
    for c in _cases(big, VOXEL_BIG):
        B, H, W, n = c["B"], c["H"], c["W"], c["x"].shape[0]
        t0, dt = float(c["t0"]), float(c["dt"])
        _, ex, o_oob = oracle.voxel_f32(c["x"], c["y"], c["t"], c["p"], B, (H, W), t0=t0, dt=dt, exact=True)
        ws = torch.empty(max(L.evk_voxel_workspace_bytes(B, H, W, 0), 256) * 2 + 4096, dtype=torch.uint8, device="cuda")
        oob = torch.zeros(1, dtype=torch.int64, device="cuda")
        out = torch.empty((B, H, W), device="cuda")
        for off in (0, 1):
            X, Y, T, P = (dev(c[k], off) for k in "xytp")
            for name, var in _voxel_variants():
                for accum in (False, True):
                    what = "voxel case %s %s off=%d accum=%d" % (c["k"], name, off, accum)
                    fill = float(c["fill"]) if accum else 0.0
                    out.fill_(fill)
                    oob.zero_()
                    _l.check(L.evk_voxel_f32(_p(X), _p(Y), _p(T), _p(P), n, t0, dt, B, H, W,
                                             var | (_l.ACCUMULATE if accum else 0), _p(out), _p(ws), ws.numel(),
                                             _p(oob), None))
                    torch.cuda.synchronize()
                    assert int(oob.item()) == o_oob, what
                    assert_within_exact(out.cpu().numpy(), ex, Q22, offset=fill, what=what)
        # AoS (N,4) layout
        ev = dev(np.stack([c[k] for k in "xytp"], axis=1))
        for name, var in _voxel_variants():
            oob.zero_()
            _l.check(L.evk_voxel_aos_f32(_p(ev), n, t0, dt, B, H, W, var, _p(out), _p(ws), ws.numel(), _p(oob), None))
            torch.cuda.synchronize()
            assert int(oob.item()) == o_oob
            assert_within_exact(out.cpu().numpy(), ex, Q22, what="voxel aos case %s %s" % (c["k"], name))


@pytest.mark.parametrize("big", [False, True])
def test_voxel_negpos(oracle, big):
    """events_to_neg_pos_voxel_torch ([p>0] / [p<=0]) and the numpy flavour's truthiness split ([p!=0] / [p==0])."""
    _l, L = _lib()
    for c in _cases(big, VOXEL_BIG):
        B, H, W, n = c["B"], c["H"], c["W"], c["x"].shape[0]
        t0, dt = float(c["t0"]), float(c["dt"])
        X, Y, T, P = (dev(c[k]) for k in "xytp")
        ws = torch.empty(L.evk_voxel_workspace_bytes(B, H, W, 0) * 2 + 4096, dtype=torch.uint8, device="cuda")
        oob = torch.zeros(1, dtype=torch.int64, device="cuda")
        out = torch.empty((2, B, H, W), device="cuda")
        p = c["p"]
        for truthy in (False, True):
            split = ((p != 0), (p == 0)) if truthy else ((p > 0), (p <= 0))
            refs = [oracle.voxel_f32(c["x"], c["y"], c["t"], s.astype(np.float32), B, (H, W), t0=t0, dt=dt, exact=True)
                    for s in split]
            for name, var in _voxel_variants():
                oob.zero_()
                _l.check(L.evk_voxel_negpos_f32(_p(X), _p(Y), _p(T), _p(P), n, t0, dt, B, H, W,
                                                var | (_l.NEGPOS_TRUTHY if truthy else 0), _p(out), _p(ws), ws.numel(),
                                                _p(oob), None))
                torch.cuda.synchronize()
                assert int(oob.item()) == refs[0][2]
                o = out.cpu().numpy()
                for s in range(2):
                    assert_within_exact(o[s], refs[s][1], Q22, what="negpos case %s %s truthy=%d grid %d" % (
                        c["k"], name, truthy, s))


@pytest.mark.parametrize("big", [False, True])
def test_voxel_trilinear(oracle, big):
    """The trilinear extension: per bin, the bilinear image of p * max(0, 1 - |tau - b|) -- including footprints that
    wrap around the canvas (coordinates at -ulp floor to -1)."""
    _l, L = _lib()
    for c in _cases(big, VOXEL_BIG):
        B, H, W, n = c["B"], c["H"], c["W"], c["x"].shape[0]
        Hc, Wc = H + 1, W + 1
        t0, dt = c["t0"], c["dt"]
        tn = ((c["t"] - t0) / dt) * np.float32(B - 1)
        refs = []
        for b in range(B):
            wgt = np.float32(1) - np.abs(tn - np.float32(b))
            wb = np.where(np.isnan(wgt), wgt, np.maximum(wgt, np.float32(0))).astype(np.float32)
            refs.append(oracle.image_torch_f32(c["x"], c["y"], (c["p"] * wb).astype(np.float32), sensor_size=(H, W),
                                               clip_out_of_range=c["clip"], interpolation="bilinear", exact=True))
        X, Y, T, P = (dev(c[k]) for k in "xytp")
        ws = torch.empty(L.evk_voxel_workspace_bytes(B, Hc, Wc, _l.BILINEAR) + 4096, dtype=torch.uint8, device="cuda")
        oob = torch.zeros(1, dtype=torch.int64, device="cuda")
        out = torch.empty((B, Hc, Wc), device="cuda")
        for name, var in (("global_red", _l.VARIANT_GLOBAL_RED), ("vector_red", _l.VARIANT_VECTOR_RED),
                          ("auto", _l.VARIANT_AUTO)):
            oob.zero_()
            _l.check(L.evk_voxel_f32(_p(X), _p(Y), _p(T), _p(P), n, float(t0), float(dt), B, Hc, Wc,
                                     var | _l.BILINEAR | (_l.CLIP if c["clip"] else 0), _p(out), _p(ws), ws.numel(),
                                     _p(oob), None))
            torch.cuda.synchronize()
            assert int(oob.item()) == refs[0][2], (c["k"], name)
            o = out.cpu().numpy()
            for b in range(B):
                assert_within_exact(o[b], refs[b][1], Q22, what="trilinear case %s %s bin %d" % (c["k"], name, b))


def test_voxel_windows_pairs_negpos(oracle):
    """Overlapping (start, end) windows, each with its own t0 / dt, in both the combined and the neg/pos form."""
    _l, L = _lib()
    c = replicate(SMALL[1], 5000)
    c["t"] = np.sort(c["t"])
    B, H, W, n = c["B"], c["H"], c["W"], c["x"].shape[0]
    pairs = np.array([0, 5000, 10, 11, 100, 2600, 2500, 4999, 4999, 5000], np.int64)
    nw = pairs.shape[0] // 2
    X, Y, T, P = (dev(c[k]) for k in "xytp")
    offs = dev(pairs)
    oob = torch.zeros(1, dtype=torch.int64, device="cuda")
    for negpos in (False, True):
        out = torch.empty((nw, 2 if negpos else 1, B, H, W), device="cuda")
        _l.check(L.evk_voxel_windows_f32(_p(X), _p(Y), _p(T), _p(P), _p(offs), nw, n, B, H, W,
                                         _l.WINDOW_PAIRS | (_l.WINDOW_NEGPOS if negpos else 0), _p(out), _p(oob), None))
        torch.cuda.synchronize()
        o = out.cpu().numpy()
        for w in range(nw):
            a, b = pairs[2 * w], pairs[2 * w + 1]
            sl = slice(a, b)
            ps = [(c["p"][sl] > 0), (c["p"][sl] <= 0)] if negpos else [c["p"][sl]]
            for s, pw in enumerate(ps):
                _, ex, _ = oracle.voxel_f32(c["x"][sl], c["y"][sl], c["t"][sl], pw.astype(np.float32), B, (H, W), exact=True)
                assert_within_exact(o[w, s], ex, Q22, what="window %d negpos=%d grid %d" % (w, negpos, s))


# ---- event images ----------------------------------------------------------------------------------------------------
def _image_variants():
    _l, _ = _lib()
    return [("auto", _l.VARIANT_AUTO), ("global_red", _l.VARIANT_GLOBAL_RED), ("vector_red", _l.VARIANT_VECTOR_RED),
            ("warp_agg", _l.VARIANT_WARP_AGG), ("smem_tile", _l.VARIANT_SMEM_TILE)]


@pytest.mark.parametrize("big", [False, True])
def test_image(oracle, big):
    from event_utils_b200.representations.image import _canvas_and_clip
    _l, L = _lib()
    for c in _cases(big, IMAGE_BIG):
        n = c["x"].shape[0]
        X, Y, P = dev(c["x"]), dev(c["y"]), dev(c["p"])
        oob = torch.zeros(1, dtype=torch.int64, device="cuda")
        for interp in (None, "bilinear"):
            for clip, padding in ((c["clip"], c["padding"]), (not c["clip"], not c["padding"])):
                (Hi, Wi), clipx, clipy = _canvas_and_clip((c["H"], c["W"]), interp, padding)
                if interp and (Hi < 2 or Wi < 2):
                    continue
                fill = float(c["fill"])
                _, ex, o_oob = oracle.image_torch_f32(c["x"], c["y"], c["p"], sensor_size=(c["H"], c["W"]),
                                                      clip_out_of_range=clip, interpolation=interp, padding=padding,
                                                      exact=True)
                ws = torch.empty(L.evk_image_workspace_bytes(Hi, Wi, _l.BILINEAR) + 256, dtype=torch.uint8, device="cuda")
                out = torch.empty((Hi, Wi), device="cuda")
                q = Q22 if interp else 0.0
                for name, var in _image_variants():
                    for accum in (False, True):
                        flags = var | (_l.BILINEAR if interp else 0) | (_l.CLIP if clip else 0)
                        if accum:
                            out.fill_(fill)
                            flags |= _l.ACCUMULATE
                        oob.zero_()
                        _l.check(L.evk_image_f32(_p(X), _p(Y), _p(P), n, Hi, Wi, clipx, clipy, flags,
                                                 0.0 if accum else fill, _p(out), _p(ws), ws.numel(), _p(oob), None))
                        torch.cuda.synchronize()
                        what = "image case %s %s clip=%d pad=%d %s accum=%d" % (c["k"], interp, clip, padding, name, accum)
                        assert int(oob.item()) == o_oob, what
                        assert_within_exact(out.cpu().numpy(), ex, q, offset=fill, what=what)


@pytest.mark.parametrize("big", [False, True])
def test_count_u32_with_clipping(oracle, big):
    from event_utils_b200.representations.image import _canvas_and_clip
    _l, L = _lib()
    for c in _cases(big, IMAGE_BIG):
        n = c["x"].shape[0]
        X, Y = dev(c["x"]), dev(c["y"])
        oob = torch.zeros(1, dtype=torch.int64, device="cuda")
        for clip, padding in ((True, True), (True, False), (False, True)):
            (Hi, Wi), clipx, clipy = _canvas_and_clip((c["H"], c["W"]), None, padding)
            _, ex, o_oob = oracle.image_torch_f32(c["x"], c["y"], np.ones(n, np.float32), sensor_size=(c["H"], c["W"]),
                                                  clip_out_of_range=clip, padding=padding, exact=True)
            cnt = torch.empty((Hi, Wi), dtype=torch.int32, device="cuda")
            for name, var in (("auto", _l.VARIANT_AUTO), ("global_red", _l.VARIANT_GLOBAL_RED),
                              ("warp_agg", _l.VARIANT_WARP_AGG), ("smem_tile", _l.VARIANT_SMEM_TILE)):
                oob.zero_()
                _l.check(L.evk_count_u32(_p(X), _p(Y), n, Hi, Wi, clipx, clipy, var | (_l.CLIP if clip else 0), _p(cnt),
                                         _p(oob), None))
                torch.cuda.synchronize()
                what = "count case %s clip=%d pad=%d %s" % (c["k"], clip, padding, name)
                assert int(oob.item()) == o_oob, what
                assert np.array_equal(cnt.cpu().numpy().astype(np.float64), ex.sum), what


@pytest.mark.parametrize("big", [False, True])
def test_timestamp_images(oracle, big):
    from exact_bounds import assert_ratio_within_exact
    from event_utils_b200.representations.image import _timestamp_images
    for c in _cases(big, VOXEL_BIG):
        X, Y, T, P = (dev(c[k]) for k in "xytp")
        t_first, t_last = float(c["t"][0]), float(c["t"][-1])
        for mode in ("default", "reverse", "raw", "nopad"):
            po, no, ex, o_oob = oracle.timestamp_image_f32(c["x"], c["y"], c["t"], c["p"], sensor_size=(c["H"], c["W"]),
                                                           clip_out_of_range=c["clip"], padding=mode != "nopad",
                                                           timestamp_reverse=mode == "reverse",
                                                           normalize_timestamps=mode != "raw", exact=True)
            try:
                pos, neg = _timestamp_images(X, Y, T, P, t_first, t_last, (c["H"], c["W"]), c["clip"], "bilinear",
                                             mode != "nopad", mode == "reverse", raw=mode == "raw")
            except IndexError:
                assert o_oob > 0, (c["k"], mode)
                continue
            assert o_oob == 0, (c["k"], mode)
            for s, img in enumerate((pos, neg)):
                assert_ratio_within_exact(img.cpu().numpy(), _sel(ex, 2 * s), _sel(ex, 2 * s + 1),
                                          what="tsimg case %s %s %s" % (c["k"], mode, ("pos", "neg")[s]))


# ---- image of warped events: derivative images and the fused contrast-maximisation pass --------------------------------
def _cmax_events(c, Hs, Ws, Hm, Wm):
    """f64 events of a case, scaled onto an Hs x Ws sensor, plus events exactly on the (0, W] / (0, H] mask edges."""
    x = c["x"].astype(np.float64) * (Ws / max(c["W"], 1))
    y = c["y"].astype(np.float64) * (Hs / max(c["H"], 1))
    x[::9], y[::13] = float(Wm), float(Hm)
    x[4::17], y[5::19] = 0.0, 0.0
    t = np.sort(c["t"].astype(np.float64))
    p = c["p"].astype(np.float64)
    p[~np.isfinite(p)] = 1.0            # non-finite polarities poison the objective; the scatter tests cover them
    return x, y, t, p


def test_image_drv(oracle):
    """evk_image_drv_f32 with K = 0, 1, 2 Jacobian rows, against the oracle's IWE / dIWE for a zero velocity (the
    jacobian rows [-d, 0] and [0, -d] of warps.py:57-60)."""
    _l, L = _lib()
    for c in SMALL[:12]:
        Hs, Ws = c["H"] + 3, c["W"] + 4
        x, y, t, p = _cmax_events(c, Hs, Ws, Hs, Ws)
        t_ref = float(t[-1])
        iwe, d, ex, o_oob = oracle.iwe_linvel((0.0, 0.0), x, y, t, p, (Hs, Ws), compute_gradient=True,
                                              sensor_size=(Hs, Ws), t_ref=t_ref, exact=True)
        dd = t - t_ref
        mk = (~((x <= 0) | (x > Ws)) & ~((y <= 0) | (y > Hs))).astype(np.float64)
        xf, yf, pf, jf = ((x * mk).astype(np.float32), (y * mk).astype(np.float32), (p * mk).astype(np.float32),
                          ((-dd) * mk).astype(np.float32))
        z = np.zeros_like(jf)
        n, Hc, Wc = x.shape[0], Hs + 1, Ws + 1
        X, Y, P = dev(xf), dev(yf), dev(pf)
        oob = torch.zeros(1, dtype=torch.int64, device="cuda")
        for K, jx, jy in ((0, None, None), (1, [jf], [z]), (2, [jf, z], [z, jf])):
            JX = dev(np.concatenate(jx)) if K else None
            JY = dev(np.concatenate(jy)) if K else None
            img = torch.empty((Hc, Wc), device="cuda")
            dimg = torch.empty((max(K, 1), Hc, Wc), device="cuda")
            oob.zero_()
            _l.check(L.evk_image_drv_f32(_p(X), _p(Y), _p(P), _p(JX), _p(JY), K, n, Hc, Wc, float(Wc - 1), float(Hc - 1),
                                         _l.CLIP, _p(img), _p(dimg) if K else None, _p(oob), None))
            torch.cuda.synchronize()
            assert int(oob.item()) == o_oob
            assert_within_exact(img.cpu().numpy(), _sel(ex, 0), what="drv img case %s K=%d" % (c["k"], K))
            for k in range(K):
                assert_within_exact(dimg[k].cpu().numpy(), _sel(ex, 1 + k), what="drv dimg case %s K=%d %d" % (c["k"], K, k))


def _f_g_close(res, f_o, g_o, iwe_o, d_o):
    """f and g with the tolerances of the existing cmax parity tests."""
    assert abs(res[0] - f_o) <= 1e-5 * abs(f_o) + 1e-12, (res[0], f_o)
    scale = np.sqrt(np.mean((2 * (iwe_o - iwe_o.mean())) ** 2) * np.mean(d_o.astype(np.float64) ** 2))
    assert np.abs(res[1:3] - g_o).max() <= 1e-5 * scale + 1e-12, (res[1:3], g_o)


@pytest.mark.parametrize("big", [False, True])
def test_cmax_f64(oracle, big):
    _l, L = _lib()
    cases = [replicate(c, CMAX_BIG) for c in BIG_FROM[:2]] if big else SMALL[:10]
    for c in cases:
        Hs, Ws = c["H"] + 5, c["W"] + 7
        Hm, Wm = Hs - 1, Ws + 2                     # bounds mask size != sensor size
        x, y, t, p = _cmax_events(c, Hs, Ws, Hm, Wm)
        n = x.shape[0]
        span = max(float(t[-1] - t[0]), 1e-6)
        X, Y, T, P = (dev(a) for a in (x, y, t, p))
        ws = torch.empty(L.evk_cmax_workspace_bytes(Hs, Ws) + 256, dtype=torch.uint8, device="cuda")
        wsa = ws[(-ws.data_ptr()) % 256:]
        res = torch.zeros(12, dtype=torch.float64, device="cuda")
        iwe = torch.empty((Hs + 1, Ws + 1), device="cuda")
        diwe = torch.empty((2, Hs + 1, Ws + 1), device="cuda")
        # velocities that push events across every canvas edge
        for vx, vy in ((0.0, 0.0), (1.5 * Ws / span, -0.7 * Hs / span), (-1.2 * Ws / span, 1.3 * Hs / span)):
            for p_scale in (1.0, 100.0):
                for absp in (False, True):
                    iwe_o, d_o, ex, o_oob = oracle.iwe_linvel((vx, vy), x, y, t, p * p_scale, (Hm, Wm), True,
                                                              use_polarity=not absp, sensor_size=(Hs, Ws), exact=True)
                    f_o = oracle.variance_f(iwe_o, 1.0)
                    g_o = oracle.variance_g(iwe_o, d_o, 1.0)
                    for name, var in (("l2_block", _l.VARIANT_VECTOR_RED), ("onchip", _l.VARIANT_SMEM_TILE),
                                      ("global_red", _l.VARIANT_GLOBAL_RED), ("auto", _l.VARIANT_AUTO)):
                        for nomix in (False, True):
                            flags = var | _l.CMAX_WANT_GRAD | (_l.CMAX_ABS_POLARITY if absp else 0) | (
                                _l.CMAX_NO_CHANNEL_MIX if nomix else 0)
                            _l.check(L.evk_cmax_linvel_variance_f64(_p(X), _p(Y), _p(T), _p(P), n, p_scale, vx, vy,
                                                                    float(t[-1]), Hm, Wm, Hs, Ws, 1.0, flags, _p(res),
                                                                    _p(iwe), _p(diwe), _p(wsa), wsa.numel(), None))
                            torch.cuda.synchronize()
                            r = res.cpu().numpy()
                            what = "cmax case %s v=(%g,%g) ps=%g abs=%d %s nomix=%d" % (c["k"], vx, vy, p_scale, absp,
                                                                                      name, nomix)
                            assert int(r[4]) == o_oob, what
                            q = Q22
                            assert_within_exact(iwe.cpu().numpy(), _sel(ex, 0), q, what=what + " iwe")
                            dn = diwe.cpu().numpy()
                            assert_within_exact(dn[0], _sel(ex, 1), q, what=what + " diwe0")
                            assert_within_exact(dn[1], _sel(ex, 2), q, what=what + " diwe1")
                            if o_oob:
                                continue
                            # the objective tail against the oracle's objective of the kernel's own images (checked
                            # above cell by cell): in the contended cases the f32 images -- the oracle's sequential sums
                            # included -- differ by more than the f / g tolerance from any other summation order
                            gi, gd = iwe.cpu().numpy(), dn
                            f_k, g_k = oracle.variance_f(gi, 1.0), oracle.variance_g(gi, gd, 1.0)
                            if nomix:
                                assert np.array_equal(r[1:3], r[6:8]), what     # un-mixed gradient == result[6..7]
                                assert abs(r[0] - f_k) <= 1e-5 * abs(f_k) + 1e-12, what
                            else:
                                _f_g_close(r, f_k, g_k, gi, gd)
                                if not big:
                                    _f_g_close(r, f_o, g_o, iwe_o, d_o)


def test_cmax_batch_vs_single(oracle):
    """K = 1 and K = 32 candidates in one pass against the oracle of each candidate."""
    _l, L = _lib()
    c = replicate(SMALL[2], 300001)
    Hs, Ws = c["H"] + 5, c["W"] + 7
    x, y, t, p = _cmax_events(c, Hs, Ws, Hs, Ws)
    span = max(float(t[-1] - t[0]), 1e-6)
    X, Y, T, P = (dev(a) for a in (x, y, t, p))
    ws = torch.empty(L.evk_cmax_workspace_bytes(Hs, Ws) + 256, dtype=torch.uint8, device="cuda")
    wsa = ws[(-ws.data_ptr()) % 256:]
    rng = np.random.default_rng(4)
    for K in (1, 32):
        params = np.ascontiguousarray((rng.uniform(-1.5, 1.5, (K, 2)) * [Ws / span, Hs / span]).astype(np.float64))
        res = torch.zeros((K, 12), dtype=torch.float64, device="cuda")
        _l.check(L.evk_cmax_linvel_objective_batch_f64(_p(X), _p(Y), _p(T), _p(P), x.shape[0], 1.0, params.ctypes.data,
                                                       K, float(t[-1]), Hs, Ws, Hs, Ws, 1.0, _l.CMAX_WANT_GRAD,
                                                       _l.OBJ_VARIANCE, 0.0, _p(res), _p(wsa), wsa.numel(), None))
        torch.cuda.synchronize()
        r = res.cpu().numpy()
        for k in range(K):
            iwe_o, d_o = oracle.iwe_linvel(params[k], x, y, t, p, (Hs, Ws), True, sensor_size=(Hs, Ws))
            _f_g_close(r[k], oracle.variance_f(iwe_o, 1.0), oracle.variance_g(iwe_o, d_o, 1.0), iwe_o, d_o)


def test_cmax_f32_fast_mode_objective_only(oracle):
    """The f32 fast mode warps in f32, so an event on a mask edge may fall on the other side of it than in the f64
    reference: its images are not comparable cell by cell, only f and g are (with the existing tolerances)."""
    _l, L = _lib()
    c = replicate(SMALL[4], 200001)
    Hs, Ws = c["H"] + 5, c["W"] + 7
    x, y, t, p = _cmax_events(c, Hs, Ws, Hs, Ws)
    span = max(float(t[-1] - t[0]), 1e-6)
    vx, vy = 0.8 * Ws / span, -0.5 * Hs / span
    X, Y, P = dev(x.astype(np.float32)), dev(y.astype(np.float32)), dev(p.astype(np.float32))
    TR = dev((t - t[-1]).astype(np.float32))
    ws = torch.empty(L.evk_cmax_workspace_bytes(Hs, Ws) + 256, dtype=torch.uint8, device="cuda")
    wsa = ws[(-ws.data_ptr()) % 256:]
    res = torch.zeros(12, dtype=torch.float64, device="cuda")
    iwe_o, d_o = oracle.iwe_linvel((vx, vy), x, y, t, p, (Hs, Ws), True, sensor_size=(Hs, Ws))
    f_o = oracle.variance_f(iwe_o, 1.0)
    _l.check(L.evk_cmax_linvel_variance_f32(_p(X), _p(Y), _p(TR), _p(P), x.shape[0], 1.0, vx, vy, Hs, Ws, Hs, Ws, 1.0,
                                            _l.CMAX_WANT_GRAD, _p(res), None, None, _p(wsa), wsa.numel(), None))
    torch.cuda.synchronize()
    assert abs(res[0].item() - f_o) <= 1e-3 * abs(f_o)


# ---- RobustNorm --------------------------------------------------------------------------------------------------------
def test_robust_norm_edges(oracle):
    """Order statistics against torch.kthvalue on the CPU (the reference's own call) and the output against the oracle:
    ties, +-0, subnormals, +-inf, NaN of either sign below and at the selected ranks, tiny sizes, last-10-bit values,
    q = 0 / 100 and an inverted range.  A NaN anywhere makes every output NaN unless the identity short-cut is taken."""
    from event_utils_b200.data_loaders.data_augmentation import RobustNorm
    from test_exact_oracle_cpu import reference_robust_norm, robust_norm_cases
    for name, a, qs in robust_norm_cases():
        x = torch.from_numpy(a.copy())
        for lo, hi in qs:
            ref, t_min, t_max = reference_robust_norm(x, lo, hi)
            got = [RobustNorm.percentile(x.cuda(), q) for q in (lo, hi)]
            assert np.array_equal(np.float32(got), np.float32([t_min, t_max]), equal_nan=True), (name, lo, hi, got)
            out = RobustNorm(low_perc=lo, top_perc=hi)(x.cuda()).cpu().numpy()
            exp = oracle.robust_norm_f32(a, low_perc=lo, top_perc=hi)
            assert np.array_equal(np.isnan(out), np.isnan(exp)), (name, lo, hi)
            assert np.array_equal(out[~np.isnan(out)], exp[~np.isnan(exp)]), (name, lo, hi)
