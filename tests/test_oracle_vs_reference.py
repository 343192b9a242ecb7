"""The oracle against the UNMODIFIED reference on larger, randomised companions of the other golden vectors.  The
inputs are regenerated here from their seeds; the reference's outputs were stored by tests/golden/make_golden_random.py
(large outputs at a fixed sample of their cells)."""
import numpy as np
import pytest

from conftest import assert_close_to_max, golden, make_events


@pytest.fixture(scope="module")
def ref():
    return golden("reference_random")


def assert_matches_sample(ours, ref, key, rel):
    ours = np.asarray(ours)
    assert ours.shape == tuple(ref[key + "_shape"]), (key, ours.shape)
    assert_close_to_max(ours.ravel()[ref[key + "_idx"]], ref[key], rel, key)


@pytest.mark.parametrize("seed,n,B,H,W", [(1, 200000, 5, 260, 346), (2, 50000, 7, 180, 240), (3, 1000, 2, 10, 12)])
def test_voxel_torch_bit_exact(ref, oracle, seed, n, B, H, W):
    x, y, t, p = make_events(seed, n, H, W)
    assert_matches_sample(oracle.voxel_f32(x, y, t, p, B, (H, W)), ref, "voxel_torch_%d" % seed, 1e-6)


def test_voxel_numpy(ref, oracle):
    rng = np.random.default_rng(1234)
    n = 100000
    xs, ys = rng.integers(0, 346, n), rng.integers(0, 260, n)
    ts = np.sort(rng.random(n))
    ps = rng.integers(0, 2, n) * 2 - 1.0
    assert_matches_sample(oracle.voxel_f64(xs, ys, ts, ps, 5, (260, 346)), ref, "voxel_numpy", 1e-12)


IMAGE_KW = [dict(), dict(interpolation='bilinear'), dict(padding=False), dict(interpolation='bilinear', padding=False),
            dict(clip_out_of_range=False)]


@pytest.mark.parametrize("kw", IMAGE_KW)
def test_image_torch(ref, oracle, kw):
    k = IMAGE_KW.index(kw)
    x, y, t, p = make_events(5, 100000, 180, 240, pol="real")
    if kw.get("clip_out_of_range", True):
        x[::7] += 4
    assert_matches_sample(oracle.image_torch_f32(x, y, p, **kw), ref, "image_%d" % k, 2e-6)


def test_flow(ref, oracle):
    x, y, t, p = make_events(6, 50000, 180, 240)
    flow = (np.random.default_rng(6).standard_normal((2, 180, 240)) * 30).astype(np.float32)
    xo, yo = oracle.warp_flow_f32(x, y, t, flow)
    assert_matches_sample(xo, ref, "flow_x", 1e-6)
    assert_matches_sample(yo, ref, "flow_y", 1e-6)


@pytest.mark.parametrize("sigma", [1.0, 0.0, 3.0])
def test_cmax(ref, oracle, sigma):
    x, y, t, p = make_events(7, 100000, 180, 240, dtype=np.float64)
    rows = [r for r in ref["cmax"] if r[0] == sigma]
    assert len(rows) == 2
    for _, vx, vy, f, g0, g1, scale in rows:
        fo, go = oracle.cmax_variance((vx, vy), x, y, t, p, blur_sigma=sigma)
        assert abs(fo - f) <= 1e-6 * abs(f), (sigma, vx, vy)
        assert np.abs(go - np.array([g0, g1])).max() <= 1e-5 * scale, (sigma, vx, vy)


def test_find_new_range_matches_reference(ref):
    """the grid-search driver's interval update (events_cmax.py:160-182), host logic only"""
    from event_utils_b200.contrast_max.events_cmax import find_new_range
    rng = np.random.default_rng(0)
    expect = ref["find_new_range"]
    assert expect.shape == (500, 2)
    for i in range(500):
        axis = np.sort(rng.uniform(-200, 200, rng.integers(3, 9)))
        value = rng.choice(axis) if rng.random() < 0.7 else rng.uniform(-250, 250)
        assert np.array_equal(expect[i], np.asarray(find_new_range(axis, value), dtype=np.float64)), i


def test_window_tables_match_reference_loader(ref):
    """k_events / t_seconds / fixed_frames / between_frames tables of BaseVoxelDataset
    (base_dataset.py:322-417), built here vectorised"""
    from event_utils_b200.data_loaders import windows as Wn
    rng = np.random.default_rng(3)
    ts = np.sort(rng.uniform(5.0, 7.5, 20000))
    ts[100:110] = ts[100]                                   # repeated stamps
    for k, w in ((1000, 0), (1500, 500), (333, 33)):
        assert np.array_equal(ref["windows_k_%d_%d" % (k, w)], Wn.k_event_indices(len(ts), k, w))
    for t, w in ((0.1, 0.0), (0.25, 0.05), (0.013, 0.0)):
        assert np.array_equal(ref["windows_t_%g_%g" % (t, w)], Wn.timeblock_indices(ts, t, w))
    for nf in (1, 7, 40):
        assert np.array_equal(ref["windows_f_%d" % nf], Wn.fixed_frames_indices(ts, nf))
    frame_ts = np.concatenate((np.sort(rng.uniform(5.0, 7.5, 30)), [9.0]))
    assert np.array_equal(frame_ts, ref["windows_frame_ts"])
    assert np.array_equal(ref["windows_between"], Wn.between_frame_indices(ts, frame_ts))
    with pytest.raises(Exception):
        Wn.check_event_indices(Wn.k_event_indices(1000, 300, 0).tolist() + [[900, 1200]], 1000)


NAMES = ["rms", "sos", "soe", "moa", "isoa", "sosa", "r1"]


@pytest.mark.parametrize("name", NAMES)
def test_other_objectives_random_scene(ref, oracle, name):
    x, y, t, p = make_events(17, 60000, 180, 240, dtype=np.float64)
    rows = [r for r in ref["objectives"] if int(r[0]) == NAMES.index(name)]
    assert len(rows) == 6
    for _, vx, vy, sigma, f, g0, g1 in rows:
        sigma = None if np.isnan(sigma) else sigma
        fo, go = oracle.cmax_objective(name, (vx, vy), x, y, t, p, blur_sigma=sigma)
        assert abs(fo - f) <= 1e-6 * max(abs(f), 1e-12), (name, vx, vy, sigma)
        if name in ("rms", "soe", "isoa", "sosa"):
            g = np.array([g0, g1])
            assert np.abs(go - g).max() <= 1e-5 * max(np.abs(g).max(), 1e-9), (name, vx, vy, sigma)
