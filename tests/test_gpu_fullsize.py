"""Parity at the BASELINE sizes, CELL BY CELL against the C oracle (VERDICT r1 "what's weak" #1): the quoted
configurations themselves, not only size-independent properties.

  config 2: 50 M uniform events -> 5 x 480 x 640 voxel grid     (voxel_grid.py:129-153), every kernel variant
  config 3: 50 M events, linvel warp + IWE + variance f and g   (objectives.py:211-264), both event passes
  config 4: 50 M Zipf(1.0) events -> 1280 x 720 count image     (image.py:88-95), bit exact

The oracle (oracle/evk_oracle.c, sequential C) needs 1-3 s per 50 M-event call; event generation is numpy.
"""
import numpy as np
import pytest

from conftest import assert_close_to_max

torch = pytest.importorskip("torch")
pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")]

N = 50_000_000


@pytest.fixture(autouse=True)
def _reset():
    import event_utils_b200 as eu
    from event_utils_b200.contrast_max import objectives
    yield
    eu.config.variant = None
    eu.config.check_index_errors = True
    objectives.event_pass = None
    objectives.precision = "f64"
    objectives.clear_cache()


@pytest.fixture(scope="module")
def voxel_stream():
    rng = np.random.default_rng(2024)
    x = (rng.random(N, dtype=np.float32) * np.float32(639))
    y = (rng.random(N, dtype=np.float32) * np.float32(479))
    t = np.sort(rng.random(N, dtype=np.float32))
    p = (rng.integers(0, 2, N, dtype=np.int8) * 2 - 1).astype(np.float32)
    return x, y, t, p


def test_config2_voxel_50m_every_variant_cell_by_cell(oracle, voxel_stream):
    import event_utils_b200 as eu
    from event_utils_b200.representations.voxel_grid import events_to_voxel_torch
    x, y, t, p = voxel_stream
    ref = oracle.voxel_f32(x, y, t, p, 5, (480, 640))
    assert ref.shape == (5, 480, 640) and abs(float(ref.astype(np.float64).sum()) - float(p.astype(np.float64).sum())) <= 2.0
    X, Y, T, P = (torch.from_numpy(a).cuda() for a in (x, y, t, p))
    worst = {}
    for variant in (None, "global_red", "vector_red", "smem_cache"):
        eu.config.variant = variant
        out = events_to_voxel_torch(X, Y, T, P, 5, sensor_size=(480, 640)).cpu().numpy()
        assert_close_to_max(out, ref, 1e-5, "voxel 50M variant=%s" % variant)
        worst[variant] = float(np.abs(out - ref).max() / np.abs(ref).max())
    print("config 2 max rel err vs oracle:", worst)


def test_config3_cmax_50m_f_and_g_vs_oracle(oracle):
    from event_utils_b200.contrast_max import objectives as O
    from event_utils_b200.contrast_max.warps import linvel_warp
    rng = np.random.default_rng(7)
    x = rng.random(N) * 238.0 + 0.5
    y = rng.random(N) * 178.0 + 0.5
    t = np.sort(rng.random(N)) * 0.05
    p = rng.integers(0, 2, N) * 2.0 - 1.0
    params = (30.0, -20.0)
    fo, go = oracle.cmax_variance(params, x, y, t, p, blur_sigma=1.0)
    iwe, d = oracle.iwe_linvel(params, x, y, t, p, (180, 240), True)
    scale = np.sqrt(np.mean((2 * (iwe.astype(np.float64) - iwe.mean())) ** 2) * np.mean(d.astype(np.float64) ** 2))
    warp = linvel_warp()
    for event_pass in ("onchip", "l2", None):
        O.event_pass = event_pass
        obj = O.variance_objective()
        f = obj.evaluate_function(params, x, y, t, p, warp, (180, 240), 1.0)
        g = obj.evaluate_gradient(params, x, y, t, p, warp, (180, 240), 1.0)
        assert abs(f - fo) <= 1e-5 * abs(fo), (event_pass, f, fo)
        assert np.abs(g - go).max() <= 1e-5 * scale, (event_pass, g, go, scale)
        img, dimg = O.get_iwe(params, x, y, t, p, warp, (180, 240), compute_gradient=True)
        assert_close_to_max(img, iwe, 1e-5, "IWE 50M event_pass=%s" % event_pass)
        assert_close_to_max(dimg, d, 1e-5, "dIWE 50M event_pass=%s" % event_pass)
        print("config 3 event_pass=%s: f rel err %.2e, g err/scale %.2e" % (event_pass, abs(f - fo) / abs(fo), np.abs(g - go).max() / scale))


def _zipf(seed, n, H, W, s):
    rng = np.random.default_rng(seed)
    npx = H * W
    w = 1.0 / np.arange(1, npx + 1) ** s
    cdf = np.cumsum(w) / w.sum()
    ranks = np.searchsorted(cdf, rng.random(n))
    perm = rng.permutation(npx)
    pix = perm[np.minimum(ranks, npx - 1)]
    return (pix % W).astype(np.float32), (pix // W).astype(np.float32)


@pytest.mark.parametrize("s", [1.0, 1.2])
def test_config4_zipf_50m_counts_bit_exact(oracle, s):
    import event_utils_b200 as eu
    from event_utils_b200 import _lib
    from event_utils_b200.representations.image import events_to_image_torch
    H, W = 720, 1280
    x, y = _zipf(99, N, H, W, s)
    p = np.ones(N, np.float32)
    ref = oracle.image_torch_f32(x, y, p, sensor_size=(H, W), clip_out_of_range=False)
    assert float(ref.astype(np.float64).sum()) == N and ref.max() < 2 ** 24      # f32 holds every count exactly
    X, Y, P = (torch.from_numpy(a).cuda() for a in (x, y, p))
    for variant in (None, "smem_cache", "warp_agg"):
        eu.config.variant = variant
        out = events_to_image_torch(X, Y, P, sensor_size=(H, W), clip_out_of_range=False).cpu().numpy()
        assert np.array_equal(out, ref), "Zipf(%.1f) 50M nearest image, variant=%s" % (s, variant)
    L = _lib.lib()
    cnt = torch.empty((H, W), dtype=torch.int32, device="cuda")
    oob = torch.zeros(1, dtype=torch.int64, device="cuda")
    _lib.check(L.evk_count_u32(X.data_ptr(), Y.data_ptr(), N, H, W, 0.0, 0.0, _lib.VARIANT_AUTO, cnt.data_ptr(), oob.data_ptr(), None))
    torch.cuda.synchronize()
    assert np.array_equal(cnt.cpu().numpy().astype(np.float32), ref) and int(cnt.sum()) == N
