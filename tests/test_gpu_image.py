"""Parity of the CUDA event-image / flow-warp / helper paths with the oracle and the goldens."""
import numpy as np
import pytest
import torch

from conftest import assert_close_to_max, golden, make_events
from test_oracle_golden import IMG_VARIANTS

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _reset_variant():
    import event_utils_b200 as eu
    yield
    eu.config.variant = None


def dev(*arrs):
    return [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in arrs]


@pytest.mark.parametrize("variant", [None, "global_red", "vector_red", "warp_agg", "smem_cache"])
def test_golden_variants(variant):
    import event_utils_b200 as eu
    from event_utils_b200.representations.image import events_to_image_torch
    eu.config.variant = variant
    g = golden("image")
    hw = tuple(int(v) for v in g["ev_HW"])
    x, y, p = dev(g["ev_x"], g["ev_y"], g["ev_p"])
    for tag, kw in IMG_VARIANTS.items():
        out = events_to_image_torch(x, y, p, sensor_size=hw, **kw)
        assert out.shape == g["img_" + tag].shape
        assert_close_to_max(out.cpu().numpy(), g["img_" + tag], 1e-5, tag)
    x, y, p = dev(g["in_x"], g["in_y"], g["in_p"])
    out = events_to_image_torch(x, y, p, sensor_size=hw, clip_out_of_range=False)
    assert np.array_equal(out.cpu().numpy(), g["img_noclip_nearest"])  # +-1 weights: bit exact
    out = events_to_image_torch(x, y, p, sensor_size=hw, clip_out_of_range=False, interpolation='bilinear')
    assert_close_to_max(out.cpu().numpy(), g["img_noclip_bilinear"], 1e-5)


def test_known_answers():
    from event_utils_b200.representations.image import events_to_image_torch
    g = golden("image")
    x, y, p = dev(g["k1_x"], g["k1_y"], g["k1_p"])
    assert np.array_equal(events_to_image_torch(x, y, p, sensor_size=(4, 6)).cpu().numpy(), g["k1_default"])
    assert np.array_equal(events_to_image_torch(x, y, p, sensor_size=(4, 6), padding=False).cpu().numpy(), g["k1_nopad"])
    assert np.array_equal(events_to_image_torch(x, y, p, sensor_size=(4, 6), clip_out_of_range=False).cpu().numpy(), g["k1_noclip"])
    x, y, p = dev(g["k2_x"], g["k2_y"], g["k2_p"])
    assert np.array_equal(events_to_image_torch(x, y, p, sensor_size=(4, 6), clip_out_of_range=False).cpu().numpy(), g["k2_noclip"])
    with pytest.raises(IndexError):
        events_to_image_torch(*dev(np.float32([6.0]), np.float32([0.0]), np.float32([1.0])), sensor_size=(4, 6), clip_out_of_range=False)
    x, y, p = dev(g["k4_x"], g["k4_y"], g["k4_p"])
    for variant in (None, "vector_red"):
        import event_utils_b200 as eu
        eu.config.variant = variant
        out = events_to_image_torch(x, y, p, sensor_size=(4, 6), interpolation='bilinear').cpu().numpy()
        assert_close_to_max(out, g["k4_bilinear"], 1e-6)
    # CPU in -> CPU out, device= honoured
    out = events_to_image_torch(torch.from_numpy(g["k1_x"]), torch.from_numpy(g["k1_y"]), torch.from_numpy(g["k1_p"]), sensor_size=(4, 6))
    assert not out.is_cuda and np.array_equal(out.numpy(), g["k1_default"])


@pytest.mark.parametrize("variant", [None, "global_red", "vector_red", "warp_agg", "smem_cache"])
@pytest.mark.parametrize("bil", [False, True])
def test_vs_oracle_large(oracle, variant, bil):
    import event_utils_b200 as eu
    from event_utils_b200.representations.image import events_to_image_torch
    eu.config.variant = variant
    H, W = 720, 1280
    x, y, t, p = make_events(3, 1000003, H, W, pol="real")
    x[::13] += 3
    kw = dict(interpolation='bilinear') if bil else dict()
    out = events_to_image_torch(*dev(x, y, p), sensor_size=(H, W), **kw).cpu().numpy()
    assert_close_to_max(out, oracle.image_torch_f32(x, y, p, sensor_size=(H, W), **kw), 1e-5)


def zipf_events(seed, n, H, W, s=1.0):
    rng = np.random.default_rng(seed)
    npx = H * W
    w = 1.0 / np.arange(1, npx + 1) ** s
    cdf = np.cumsum(w) / w.sum()
    ranks = np.searchsorted(cdf, rng.random(n))
    perm = rng.permutation(npx)
    pix = perm[np.minimum(ranks, npx - 1)]
    return (pix % W).astype(np.float32), (pix // W).astype(np.float32)


@pytest.mark.parametrize("variant", [None, "global_red", "warp_agg", "smem_cache"])
def test_hot_spot_counts_bit_exact(oracle, variant):
    """Zipf-distributed pixels (BASELINE config 4, reduced N): count image must be bit exact."""
    import event_utils_b200 as eu
    from event_utils_b200 import _lib
    from event_utils_b200.representations.image import events_to_image_torch
    eu.config.variant = variant
    H, W, n = 720, 1280, 4_000_000
    x, y = zipf_events(99, n, H, W)
    p = np.ones(n, np.float32)
    ref = oracle.image_torch_f32(x, y, p, sensor_size=(H, W), clip_out_of_range=False)
    X, Y, P = dev(x, y, p)
    out = events_to_image_torch(X, Y, P, sensor_size=(H, W), clip_out_of_range=False).cpu().numpy()
    assert np.array_equal(out, ref)
    # integer entry point
    L = _lib.lib()
    cnt = torch.empty((H, W), dtype=torch.int32, device="cuda")
    oob = torch.zeros(1, dtype=torch.int64, device="cuda")
    for v in (_lib.VARIANT_AUTO, _lib.VARIANT_GLOBAL_RED, _lib.VARIANT_WARP_AGG, _lib.VARIANT_SMEM_TILE):
        _lib.check(L.evk_count_u32(X.data_ptr(), Y.data_ptr(), n, H, W, 0.0, 0.0, v, cnt.data_ptr(), oob.data_ptr(), None))
        torch.cuda.synchronize()
        assert np.array_equal(cnt.cpu().numpy().astype(np.float32), ref)
        assert int(cnt.sum()) == n


def test_hot_spot_bilinear_and_signed(oracle):
    """Zipf stream with +-1 polarities and sub-pixel jitter through the bilinear paths.
    The hottest pixel receives ~10^5 taps: f32 accumulation is then order dependent beyond 1e-5
    (the sequential f32 oracle itself is ~sqrt(n) eps away from the exact sum), so every variant --
    and the oracle -- is compared with an f64 accumulation of the same f32 tap weights, within the
    random-walk bound 2 sqrt(n_max) eps32 * max|image| (n_max = taps on the hottest pixel)."""
    import event_utils_b200 as eu
    from event_utils_b200.representations.image import events_to_image_torch
    H, W, n = 720, 1280, 2_000_000
    x, y = zipf_events(7, n, H, W, s=1.2)
    rng = np.random.default_rng(8)
    x = x + rng.random(n).astype(np.float32) * np.float32(0.999)
    y = y + rng.random(n).astype(np.float32) * np.float32(0.999)
    p = (rng.integers(0, 2, n) * 2 - 1).astype(np.float32)
    # the oracle's f32 taps (image.py:79-86,111-114) accumulated in f64, and the number of taps per cell
    ref, ex, oob = oracle.image_torch_f32(x, y, p, sensor_size=(H, W), interpolation='bilinear', exact=True)
    assert oob == 0
    exact, cnt = ex.sum, ex.cnt
    bound = 2.0 * np.sqrt(cnt.max()) * np.finfo(np.float32).eps * np.abs(exact).max()
    assert np.abs(ref - exact).max() <= bound
    for variant in ("smem_cache", "vector_red", "global_red", None):
        eu.config.variant = variant
        out = events_to_image_torch(*dev(x, y, p), sensor_size=(H, W), interpolation='bilinear').cpu().numpy()
        assert np.abs(out - exact).max() <= bound, (variant, np.abs(out - exact).max(), bound)
        # away from the hot pixels the 1e-5 bar holds as usual
        cold = cnt < 2000
        assert np.abs(out - ref)[cold].max() <= 1e-5 * np.abs(ref).max()


def test_timestamp_images(oracle):
    from event_utils_b200.representations.image import events_to_timestamp_image, events_to_timestamp_image_torch
    g = golden("tsimg")
    x, y, t, p = dev(g["x"], g["y"], g["t"], g["p"])
    for tag, kw in {"default": dict(), "reverse": dict(timestamp_reverse=True), "nopad": dict(padding=False)}.items():
        pos, neg = events_to_timestamp_image_torch(x, y, t, p, sensor_size=(40, 56), **kw)
        assert pos.shape == g[tag + "_pos"].shape and pos.is_cuda
        assert_close_to_max(pos.cpu().numpy(), g[tag + "_pos"], 1e-5, tag)
        assert_close_to_max(neg.cpu().numpy(), g[tag + "_neg"], 1e-5, tag)
    pos, neg = events_to_timestamp_image(g["x"].astype(np.float64), g["y"].astype(np.float64), g["np_t"], g["p"].astype(np.float64),
                                         sensor_size=(40, 56))
    assert pos.dtype == np.float32
    assert_close_to_max(pos, g["np_pos"], 1e-5)
    assert_close_to_max(neg, g["np_neg"], 1e-5)
    pos, neg = events_to_timestamp_image(g["x"].astype(np.float64), g["y"].astype(np.float64), g["np_t"], g["p"].astype(np.float64),
                                         sensor_size=(40, 56), normalize_timestamps=False)        # image.py:261
    assert_close_to_max(pos, g["np_raw_pos"], 1e-5)
    assert_close_to_max(neg, g["np_raw_neg"], 1e-5)
    # larger random case against the oracle
    xe, ye, te, pe = make_events(17, 700000, 180, 240)
    pos, neg = events_to_timestamp_image_torch(*dev(xe, ye, te, pe))
    po, no = oracle.timestamp_image_f32(xe, ye, te, pe)
    assert_close_to_max(pos.cpu().numpy(), po, 1e-5)
    assert_close_to_max(neg.cpu().numpy(), no, 1e-5)


def test_numpy_flavour():
    from event_utils_b200.representations.image import events_to_image
    g = golden("image")
    out = events_to_image(g["np_x"], g["np_y"], g["np_p"], sensor_size=(40, 56))
    assert out.dtype == np.float64 and out.shape == (40, 56)
    assert_close_to_max(out, g["np_nearest"], 1e-5)
    out = events_to_image(g["np_x"], g["np_y"], g["np_p"], sensor_size=(40, 56), meanval=True, default=-1)
    assert_close_to_max(out, g["np_meanval"], 1e-5)
    with pytest.raises(TypeError):
        events_to_image(np.float64([1.5]), np.float64([1.0]), np.float64([1.0]))


def test_flow_warp(oracle):
    from event_utils_b200.transforms.optic_flow import warp_events_flow_torch
    g = golden("flow")
    x, y, t, p, flow = dev(g["x"], g["y"], g["t"], g["p"], g["flow"])
    x_before = x.clone()
    xw, yw = warp_events_flow_torch(x, y, t, p, flow)
    assert torch.equal(x, x_before)  # inputs not mutated
    assert_close_to_max(xw.cpu().numpy(), g["xw"], 1e-5)
    assert_close_to_max(yw.cpu().numpy(), g["yw"], 1e-5)
    xw, yw = warp_events_flow_torch(x.unsqueeze(1), y.unsqueeze(1), t.unsqueeze(1), p.unsqueeze(1), flow.unsqueeze(0), t0=0.02)
    assert xw.shape == (x.shape[0],)
    assert_close_to_max(xw.cpu().numpy(), g["xw_t0"], 1e-5)
    assert_close_to_max(yw.cpu().numpy(), g["yw_t0"], 1e-5)
    xw, yw = warp_events_flow_torch(*dev(g["k_x"], g["k_y"], g["k_t"], g["k_t"], g["k_flow"]))
    assert_close_to_max(xw.cpu().numpy(), g["k_xw"], 1e-6)
    assert_close_to_max(yw.cpu().numpy(), g["k_yw"], 1e-6)
    # large random case against the oracle
    xe, ye, te, pe = make_events(8, 500000, 180, 240)
    fl = (np.random.default_rng(1).standard_normal((2, 180, 240)) * 30).astype(np.float32)
    xw, yw = warp_events_flow_torch(*dev(xe, ye, te, pe, fl))
    xo, yo = oracle.warp_flow_f32(xe, ye, te, fl)
    assert_close_to_max(xw.cpu().numpy(), xo, 1e-5)
    assert_close_to_max(yw.cpu().numpy(), yo, 1e-5)
    # sub-pixel and out-of-image coordinates, odd width, views that are not 16-byte aligned, few events
    rng = np.random.default_rng(2)
    for (H, W, n, off) in ((180, 240, 300001, 1), (181, 241, 200003, 0), (64, 34, 1000, 3), (33, 47, 90000, 2)):
        xe = rng.uniform(-3, W + 2, n + off).astype(np.float32)
        ye = rng.uniform(-3, H + 2, n + off).astype(np.float32)
        te = np.sort(rng.uniform(0, 0.1, n + off)).astype(np.float32)
        fl = (rng.standard_normal((2, H, W)) * 30).astype(np.float32)
        xd, yd, td, fd = dev(xe, ye, te, fl)
        xw, yw = warp_events_flow_torch(xd[off:], yd[off:], td[off:], td[off:], fd)
        xo, yo = oracle.warp_flow_f32(xe[off:], ye[off:], te[off:], fl)
        assert_close_to_max(xw.cpu().numpy(), xo, 1e-5)
        assert_close_to_max(yw.cpu().numpy(), yo, 1e-5)


def test_tap_helpers():
    from event_utils_b200.representations.image import (events_to_image_drv, image_to_event_weights,
                                                        interpolate_to_derivative_img, interpolate_to_image)
    from event_utils_b200.util.event_util import events_bounds_mask
    g = golden("taps")
    img = torch.zeros(16, 22, device="cuda")
    interpolate_to_image(*dev(g["px"], g["py"], g["dx"], g["dy"], g["w"]), img)
    assert_close_to_max(img.cpu().numpy(), g["img"], 1e-5)
    img_cpu = torch.zeros(16, 22)
    interpolate_to_image(*(torch.from_numpy(g[k]) for k in ("px", "py", "dx", "dy", "w")), img_cpu)
    assert_close_to_max(img_cpu.numpy(), g["img"], 1e-5)
    dimg = torch.zeros(2, 16, 22, device="cuda")
    px, py, dx, dy, w1, w2 = dev(g["px"], g["py"], g["dx"], g["dy"], g["w1"], g["w2"])
    interpolate_to_derivative_img(px, py, dx, dy, dimg, w1, w2)
    assert_close_to_max(dimg.cpu().numpy(), g["dimg"], 1e-5)
    out = image_to_event_weights(g["g_x"], g["g_y"], g["g_img"])
    assert out.dtype == np.float64
    assert_close_to_max(out, g["g_out"], 1e-12)
    assert np.array_equal(events_bounds_mask(g["m_x"], g["m_y"], 0, 240, 0, 180), g["m_out"])
    i0, d0 = events_to_image_drv(g["drv_x"], g["drv_y"], g["drv_p"], g["drv_jx"], g["drv_jy"], compute_gradient=True)
    assert i0.dtype == np.float32 and i0.shape == (181, 241) and d0.shape == (2, 181, 241)
    assert_close_to_max(i0, g["drv_img"], 1e-5)
    assert_close_to_max(d0, g["drv_dimg"], 1e-5)
    i1, d1 = events_to_image_drv(g["drv_x"], g["drv_y"], g["drv_p"], None, None)
    assert d1 is None
    assert_close_to_max(i1, g["drv_img"], 1e-5)


def test_robust_norm(oracle):
    from event_utils_b200.data_loaders.data_augmentation import RobustNorm
    g = golden("robust_norm")
    for tag, kw in (("voxel", {}), ("normal", dict(low_perc=10, top_perc=90)), ("sparse", {})):
        x = torch.from_numpy(g[tag + "_in"])
        out = RobustNorm(**kw)(x.cuda())
        assert out.is_cuda and out.shape == x.shape
        assert_close_to_max(out.cpu().numpy(), g[tag + "_out"], 1e-6, tag)
        assert not RobustNorm(**kw)(x).is_cuda                       # host tensor in -> host tensor out
        got = [RobustNorm.percentile(x.cuda(), q) for q in (0, 5, 50, 95, 100)]
        assert np.array_equal(np.float32(got), np.float32(g[tag + "_p"])), tag    # order statistics are exact
    # a voxel-sized random tensor against the oracle, ranks straddling bin boundaries of all three passes
    rng = np.random.default_rng(5)
    x = (rng.standard_normal((5, 480, 640)) * rng.choice([1e-3, 1.0, 300.0], size=(5, 480, 640))).astype(np.float32)
    for kw in (dict(), dict(low_perc=1, top_perc=99.9), dict(low_perc=50, top_perc=50)):
        out = RobustNorm(**kw)(torch.from_numpy(x).cuda()).cpu().numpy()
        assert_close_to_max(out, oracle.robust_norm_f32(x, **kw), 1e-6, str(kw))

