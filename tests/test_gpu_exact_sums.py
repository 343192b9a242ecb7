"""Every fixed-point carry path, the packed storage layout and the host pipelines BIT FOR BIT, on exactly summable streams
(tests/edge_cases.py exact_streams): every tap is a multiple of 2^-g and no partial sum any summation order, quantisation,
flush or carry can form exceeds 2^(24-g), so each output cell must equal the f64 sum of its taps exactly
(exact_bounds.assert_exact).  The hot cells carry most of the events with their signs in one + run and one - run, so
the shared-memory tables of the voxel hot path (F = 22), the image hot kernel (nearest F = 10, bilinear F = 22) and the
cmax on-chip image (F = 22) wrap and carry upward and downward; a lost, doubled, misplaced, mis-signed or biased carry,
tap or flush shows in the cell it belongs to, whatever its size."""
import ctypes
import functools

import numpy as np
import pytest
import torch

from edge_cases import EXACT_SIZES, exact_streams, packed_of
from exact_bounds import assert_exact, assert_tables_wrap, check_exactly_summable, select_events
from test_gpu_adversarial import _lib, _p, _voxel_variants, dev

pytestmark = pytest.mark.gpu

# past AUTO's thresholds (voxel hot table at 2^20 events, image hot kernel at 2^18, cmax on-chip image at 4 * 2^20)
VOXEL_N, IMAGE_N, CMAX_N = EXACT_SIZES["voxel"], EXACT_SIZES["nearest"], EXACT_SIZES["cmax"]
CHUNK = 4096                        # host pipelines: small chunks, so that a 4 M-event call makes ~1000 of them
FILL = 0.25


@functools.lru_cache(maxsize=None)
def _stream(kind, n, seed=7):
    return exact_streams(seed, kind, n)


@functools.lru_cache(maxsize=None)
def _voxel_ref(which):
    """(stream dict, oracle grid Exact, oob) of the voxel stream: 'f32' or its packed form 'packed'."""
    from oracle import evk_oracle as oracle
    c = _stream("voxel", VOXEL_N)
    if which == "packed":
        c = dict(c, **packed_of(c)[6])
    pl, = check_exactly_summable(oracle, c)
    return c, pl.ex, pl.oob


def _ws(L, B, H, W, flags=0):
    return torch.empty(max(L.evk_voxel_workspace_bytes(B, H, W, flags), 256) * 2 + 4096, dtype=torch.uint8, device="cuda")


def test_tables_wrap_on_this_gpu():
    """At this GPU's SM count, every CTA's hot table slot in every table launch below wraps upward and back
    downward (exact_bounds.table_launches sizes the launches as the launch code does)."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    for kind in ("voxel", "nearest", "bilinear", "cmax"):
        assert_tables_wrap(_stream(kind, EXACT_SIZES[kind]), sms, what=kind)


# ---- evk_voxel_f32 / aos / negpos / trilinear ----------------------------------------------------------------------------
def test_voxel_f32_exact(oracle):
    _l, L = _lib()
    c, ex, o_oob = _voxel_ref("f32")
    B, H, W, n = c["B"], c["H"], c["W"], c["x"].shape[0]
    t0, dt = float(c["t0"]), float(c["dt"])
    ws = _ws(L, B, H, W)
    oob = torch.zeros(1, dtype=torch.int64, device="cuda")
    out = torch.empty((B, H, W), device="cuda")
    for off in (0, 1):                                  # SoA 16-byte aligned and misaligned
        X, Y, T, P = (dev(c[k], off) for k in "xytp")
        for name, var in _voxel_variants():
            for accum in (False, True):
                what = "voxel off=%d %s accum=%d" % (off, name, accum)
                out.fill_(FILL if accum else 0.0)
                oob.zero_()
                _l.check(L.evk_voxel_f32(_p(X), _p(Y), _p(T), _p(P), n, t0, dt, B, H, W,
                                         var | (_l.ACCUMULATE if accum else 0), _p(out), _p(ws), ws.numel(), _p(oob), None))
                torch.cuda.synchronize()
                assert int(oob.item()) == o_oob, what
                assert_exact(out.cpu().numpy(), ex, offset=FILL if accum else 0.0, what=what)
    ev = dev(np.stack([c[k] for k in "xytp"], axis=1))
    for name, var in _voxel_variants():
        oob.zero_()
        _l.check(L.evk_voxel_aos_f32(_p(ev), n, t0, dt, B, H, W, var, _p(out), _p(ws), ws.numel(), _p(oob), None))
        torch.cuda.synchronize()
        assert int(oob.item()) == o_oob
        assert_exact(out.cpu().numpy(), ex, what="voxel aos %s" % name)


def test_voxel_negpos_exact(oracle):
    _l, L = _lib()
    c = _stream("voxel", VOXEL_N)
    B, H, W, n = c["B"], c["H"], c["W"], c["x"].shape[0]
    X, Y, T, P = (dev(c[k]) for k in "xytp")
    ws = _ws(L, B, H, W)
    oob = torch.zeros(1, dtype=torch.int64, device="cuda")
    out = torch.empty((2, B, H, W), device="cuda")
    p = c["p"]
    for truthy in (False, True):
        split = ((p != 0), (p == 0)) if truthy else ((p > 0), (p <= 0))
        refs = [check_exactly_summable(oracle, dict(c, p=s.astype(np.float32)))[0] for s in split]
        for name, var in _voxel_variants():
            oob.zero_()
            _l.check(L.evk_voxel_negpos_f32(_p(X), _p(Y), _p(T), _p(P), n, float(c["t0"]), float(c["dt"]), B, H, W,
                                            var | (_l.NEGPOS_TRUTHY if truthy else 0), _p(out), _p(ws), ws.numel(),
                                            _p(oob), None))
            torch.cuda.synchronize()
            assert int(oob.item()) == refs[0].oob
            o = out.cpu().numpy()
            for s in range(2):
                assert_exact(o[s], refs[s].ex, what="negpos %s truthy=%d grid %d" % (name, truthy, s))


def test_voxel_trilinear_exact(oracle):
    _l, L = _lib()
    c = _stream("voxel", VOXEL_N)
    B, H, W, n = c["B"], c["H"], c["W"], c["x"].shape[0]
    Hc, Wc = H + 1, W + 1
    X, Y, T, P = (dev(c[k]) for k in "xytp")
    ws = torch.empty(L.evk_voxel_workspace_bytes(B, Hc, Wc, _l.BILINEAR) + 4096, dtype=torch.uint8, device="cuda")
    oob = torch.zeros(1, dtype=torch.int64, device="cuda")
    out = torch.empty((B, Hc, Wc), device="cuda")
    for clip in (False, True):
        refs = check_exactly_summable(oracle, c, bilinear=True, clip=clip)
        for name, var in (("global_red", _l.VARIANT_GLOBAL_RED), ("vector_red", _l.VARIANT_VECTOR_RED),
                          ("auto", _l.VARIANT_AUTO)):
            oob.zero_()
            _l.check(L.evk_voxel_f32(_p(X), _p(Y), _p(T), _p(P), n, float(c["t0"]), float(c["dt"]), B, Hc, Wc,
                                     var | _l.BILINEAR | (_l.CLIP if clip else 0), _p(out), _p(ws), ws.numel(),
                                     _p(oob), None))
            torch.cuda.synchronize()
            assert int(oob.item()) == refs[0].oob, (name, clip)
            o = out.cpu().numpy()
            for b in range(B):
                assert_exact(o[b], refs[b].ex, what="trilinear %s clip=%d bin %d" % (name, clip, b))


# ---- the storage layout: int16 / int16 / f64 / uint8 -----------------------------------------------------------------------
def test_voxel_packed_exact(oracle):
    _l, L = _lib()
    c0 = _stream("voxel", VOXEL_N)
    c, ex, o_oob = _voxel_ref("packed")
    x16, y16, T, p8, t_first, t_last, _ = packed_of(c0)
    assert (x16 < 0).any() and (x16 >= c["W"]).any() and abs(T[0] - 1.7e9) < 10
    B, H, W, n = c["B"], c["H"], c["W"], x16.shape[0]
    X, Y, TT = dev(x16), dev(y16), dev(T)
    ws = _ws(L, B, H, W)
    oob = torch.zeros(1, dtype=torch.int64, device="cuda")
    out = torch.empty((B, H, W), device="cuda")
    for pdt in (np.uint8, np.bool_):
        P = dev(p8.astype(pdt))
        for span in ("explicit", "auto"):
            # AUTO_SPAN reads T[0] / T[n-1], which the stream pins to t_first / t_last; the arguments are then ignored
            tf, tl = (t_first, t_last) if span == "explicit" else (123.0, -5.0)
            for name, var in _voxel_variants():
                what = "packed %s span=%s %s" % (np.dtype(pdt).name, span, name)
                oob.zero_()
                _l.check(L.evk_voxel_packed_f32(_p(X), _p(Y), _p(TT), _p(P), n, tf, tl, B, H, W,
                                                var | (_l.AUTO_SPAN if span == "auto" else 0), _p(out), _p(ws),
                                                ws.numel(), _p(oob), None))
                torch.cuda.synchronize()
                assert int(oob.item()) == o_oob, what
                assert_exact(out.cpu().numpy(), ex, what=what)


# ---- host pipelines --------------------------------------------------------------------------------------------------------
@pytest.fixture
def pipeline():
    """A host pipeline with CHUNK-event chunks, destroyed after the test."""
    _l, L = _lib()
    h = ctypes.c_void_p()
    _l.check(L.evk_pipeline_create(ctypes.byref(h), CHUNK))
    yield h
    torch.cuda.synchronize()
    L.evk_pipeline_destroy(h)


def _pinned(a):
    t = torch.empty(a.shape, dtype=torch.from_numpy(a[:0]).dtype, pin_memory=True)
    t.numpy()[...] = a
    return t.numpy(), t          # keep the tensor alive with the view


def _host_call(L, pipe, arrays, packed, n, span, B, H, W, flags):
    out = np.full((B, H, W), np.nan, np.float32)
    oob = ctypes.c_ulonglong(12345)
    fn = L.evk_voxel_host_packed_f32 if packed else L.evk_voxel_host_f32
    rc = fn(pipe, *(a.ctypes.data for a in arrays), n, span[0], span[1], B, H, W, flags, out.ctypes.data,
            ctypes.byref(oob))
    return rc, out, int(oob.value)


# n = 0, below a quarter chunk (the pageable path's first chunk), one chunk, k chunks +- 1, not a multiple of 4, all
HOST_NS = (0, 1000, CHUNK, 3 * CHUNK - 1, 3 * CHUNK + 1, 5 * CHUNK + 2, VOXEL_N)


@pytest.mark.parametrize("packed", [False, True])
def test_host_pipelines_exact(oracle, pipeline, packed):
    _l, L = _lib()
    c0 = _stream("voxel", VOXEL_N)
    B, H, W = c0["B"], c0["H"], c0["W"]
    if packed:
        x16, y16, T, p8, t_first, t_last, f32 = packed_of(c0)
        src, span, ref_ev = (x16, y16, T, p8), (t_first, t_last), dict(c0, **f32)
    else:
        src, span, ref_ev = tuple(c0[k] for k in "xytp"), (float(c0["t0"]), float(c0["dt"])), c0
    for mem in ("pageable", "pinned"):
        keep = [_pinned(a) for a in src] if mem == "pinned" else [(a, None) for a in src]
        arrays = [k[0] for k in keep]
        for n in HOST_NS:
            sub = select_events(ref_ev, slice(0, n))
            if n:
                pl, = check_exactly_summable(oracle, sub)
                ex, o_oob = pl.ex, pl.oob
            for call in range(2):                       # two calls in a row on one pipeline
                what = "host packed=%d %s n=%d call %d" % (packed, mem, n, call)
                rc, out, oob = _host_call(L, pipeline, arrays, packed, n, span, B, H, W, _l.VARIANT_AUTO)
                _l.check(rc)
                if n == 0:
                    assert oob == 0 and not out.any(), what
                    continue
                assert oob == o_oob, what
                assert_exact(out, ex, what=what)


@pytest.mark.parametrize("packed", [False, True])
def test_host_auto_span(oracle, pipeline, packed):
    """EVK_AUTO_SPAN through the chunked host pipelines: every chunk gets the span of the WHOLE stream (t[0], t[n-1]),
    whatever the t0 / dt (t_first / t_last) arguments say -- the same grid as the explicit call, bit for bit."""
    _l, L = _lib()
    c0 = _stream("voxel", VOXEL_N)
    B, H, W = c0["B"], c0["H"], c0["W"]
    n = 7 * CHUNK + 3
    c = select_events(c0, slice(0, n))
    # a sub-stream whose first and last stamps are the span ends: the explicit call uses the same span
    c["t"] = c["t"].copy()
    c["t"][0], c["t"][-1] = c0["t0"], c0["t0"] + c0["dt"]
    if packed:
        x16, y16, T, p8, t_first, t_last, f32 = packed_of(c)
        src, span, ref_ev = (x16, y16, T, p8), (t_first, t_last), dict(c, **f32)
    else:
        src, span, ref_ev = tuple(c[k] for k in "xytp"), (float(c["t0"]), float(c["dt"])), c
    pl, = check_exactly_summable(oracle, ref_ev)
    ex, o_oob = pl.ex, pl.oob
    rc, explicit, oob_e = _host_call(L, pipeline, src, packed, n, span, B, H, W, 0)
    _l.check(rc)
    rc, auto, oob_a = _host_call(L, pipeline, src, packed, n, (3.0, 0.125), B, H, W, _l.AUTO_SPAN)
    _l.check(rc)
    assert oob_e == oob_a == o_oob
    assert_exact(explicit, ex, what="explicit span")
    assert_exact(auto, ex, what="EVK_AUTO_SPAN")
    assert np.array_equal(auto, explicit)


# ---- event images ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("interp", [None, "bilinear"])
def test_image_exact(oracle, interp):
    from event_utils_b200.representations.image import _canvas_and_clip
    _l, L = _lib()
    c = _stream("bilinear" if interp else "nearest", IMAGE_N)
    n = c["x"].shape[0]
    X, Y, P = dev(c["x"]), dev(c["y"]), dev(c["p"])
    oob = torch.zeros(1, dtype=torch.int64, device="cuda")
    # a dyadic background: the nearest hot sums are multiples of 2^19 up to ~2^37, which no non-zero fill on the fine
    # cells' grid can join exactly, so the nearest image takes fill 0
    fill = FILL if interp else 0.0
    for clip, padding in ((False, False), (True, True), (True, False), (False, True)):
        (Hi, Wi), clipx, clipy = _canvas_and_clip((c["H"], c["W"]), interp, padding)
        pl, = check_exactly_summable(oracle, c, clip=clip, padding=padding)
        ex, o_oob = pl.ex, pl.oob
        ws = torch.empty(L.evk_image_workspace_bytes(Hi, Wi, _l.BILINEAR) + 256, dtype=torch.uint8, device="cuda")
        out = torch.empty((Hi, Wi), device="cuda")
        for name, var in (("auto", _l.VARIANT_AUTO), ("global_red", _l.VARIANT_GLOBAL_RED),
                          ("vector_red", _l.VARIANT_VECTOR_RED), ("warp_agg", _l.VARIANT_WARP_AGG),
                          ("smem_tile", _l.VARIANT_SMEM_TILE)):
            for accum in (False, True):
                flags = var | (_l.BILINEAR if interp else 0) | (_l.CLIP if clip else 0)
                if accum:
                    out.fill_(fill)
                    flags |= _l.ACCUMULATE
                oob.zero_()
                _l.check(L.evk_image_f32(_p(X), _p(Y), _p(P), n, Hi, Wi, clipx, clipy, flags, 0.0 if accum else fill,
                                         _p(out), _p(ws), ws.numel(), _p(oob), None))
                torch.cuda.synchronize()
                what = "image %s clip=%d pad=%d %s accum=%d" % (interp, clip, padding, name, accum)
                assert int(oob.item()) == o_oob, what
                assert_exact(out.cpu().numpy(), ex, offset=fill, what=what)


def test_timestamp_raw_exact(oracle):
    """EVK_TS_RAW: the weight is the dyadic stamp itself, so the sum and count images are exact, and each output is the
    correctly rounded f32 quotient np.float32(T / C) (f64 has 53 >= 2 * 24 + 2 bits, so rounding the f64 quotient to
    f32 rounds correctly)."""
    from exact_bounds import Exact_of, assert_exactly_summable
    _l, L = _lib()
    c = exact_streams(11, "bilinear", 50001)         # plain reductions: stamp taps on a 2^-9 grid, S <= 2^15 per cell
    n = c["x"].shape[0]
    X, Y, T, P = (dev(c[k]) for k in "xytp")
    for clip, padding in ((False, True), (True, True), (True, False)):
        H, W = c["H"] + padding, c["W"] + padding
        kw = dict(sensor_size=(c["H"], c["W"]), clip_out_of_range=clip, padding=padding, normalize_timestamps=False,
                  exact=True)
        _, _, ex, o_oob = oracle.timestamp_image_f32(c["x"], c["y"], c["t"], c["p"], **kw)
        for k in range(4):
            assert_exactly_summable(lambda m: Exact_of(oracle.timestamp_image_f32(
                c["x"][m], c["y"][m], c["t"][m], c["p"][m], **kw)[2], k), c["hot"], 9, None, what="tsimg plane %d" % k)
        clipx, clipy = float(W - 1), float(H - 1)
        ws = torch.empty(L.evk_timestamp_image_workspace_bytes(H, W) + 256, dtype=torch.uint8, device="cuda")
        wsa = ws[(-ws.data_ptr()) % 16:]
        oob = torch.zeros(1, dtype=torch.int64, device="cuda")
        imgs = [torch.empty((H, W), device="cuda") for _ in range(4)]
        _l.check(L.evk_timestamp_image_counts_f32(_p(X), _p(Y), _p(T), _p(P), n, 0.0, 0.0, H, W, clipx, clipy,
                                                  _l.TS_RAW | (_l.CLIP if clip else 0), *(_p(i) for i in imgs),
                                                  _p(wsa), wsa.numel(), _p(oob), None))
        torch.cuda.synchronize()
        assert int(oob.item()) == o_oob
        pos, neg, cpos, cneg = (i.cpu().numpy() for i in imgs)
        for s, (img, cnt) in enumerate(((pos, cpos), (neg, cneg))):
            what = "tsimg raw clip=%d pad=%d %s" % (clip, padding, ("pos", "neg")[s])
            Tex, Cex = Exact_of(ex, 2 * s), Exact_of(ex, 2 * s + 1)
            assert_exact(cnt, Cex, offset=1.0, what=what + " count")
            Cn = Cex.sum + 1.0
            Cn[Cn == 0] = 1.0
            assert np.array_equal(img, (Tex.sum / Cn).astype(np.float32)), what


# ---- contrast maximisation: IWE and dIWE ------------------------------------------------------------------------------------
def test_cmax_iwe_exact(oracle):
    _l, L = _lib()
    c = _stream("cmax", CMAX_N)
    Hs, Ws, n = c["Hs"], c["Ws"], c["x"].shape[0]
    X, Y, T, P = (dev(c[k]) for k in "xytp")
    ws = torch.empty(L.evk_cmax_workspace_bytes(Hs, Ws) + 256, dtype=torch.uint8, device="cuda")
    wsa = ws[(-ws.data_ptr()) % 256:]
    res = torch.zeros(12, dtype=torch.float64, device="cuda")
    iwe = torch.empty((Hs + 1, Ws + 1), device="cuda")
    diwe = torch.empty((2, Hs + 1, Ws + 1), device="cuda")
    for absp in (False, True):
        refs = check_exactly_summable(oracle, c, abs_polarity=absp)
        for name, var in (("l2_block", _l.VARIANT_VECTOR_RED), ("onchip", _l.VARIANT_SMEM_TILE),
                          ("global_red", _l.VARIANT_GLOBAL_RED), ("auto", _l.VARIANT_AUTO)):
            flags = var | _l.CMAX_WANT_GRAD | (_l.CMAX_ABS_POLARITY if absp else 0)
            _l.check(L.evk_cmax_linvel_variance_f64(_p(X), _p(Y), _p(T), _p(P), n, 1.0, c["vx"], c["vy"], c["t_ref"],
                                                    Hs, Ws, Hs, Ws, 1.0, flags, _p(res), _p(iwe), _p(diwe), _p(wsa),
                                                    wsa.numel(), None))
            torch.cuda.synchronize()
            what = "cmax abs=%d %s" % (absp, name)
            assert int(res[4].item()) == refs[0].oob, what
            planes = [iwe.cpu().numpy()] + list(diwe.cpu().numpy())
            for pl, img in zip(refs, planes):
                assert_exact(img, pl.ex, what=what + " " + pl.name)
