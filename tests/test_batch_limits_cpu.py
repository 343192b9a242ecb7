"""No-GPU checks of the premises of tests/test_gpu_batch_limits.py: the skewed streams of tests/batch_limit_streams.py are
exactly summable in every window (the giant one included) under every velocity the GPU tests use, their window sizes
have the intended skew, and the batch sizes the GPU tests pick cross the Python window chunks of the candidate passes
and the fits."""
import numpy as np

import batch_limit_streams as S


def _lib():
    from event_utils_b200 import _lib
    return _lib.load()


def test_exact_stream_is_exactly_summable_in_every_window():
    s = S.exact_stream(S.MOTION_CAP, giant_at=S.MOTION_CAP // 2, seed=1)
    vel = S.exact_velocities()
    assert any((v == S.V).all() for v in vel)
    S.assert_exactly_summable(s, vel)
    # the giant window keeps most of its events under V, and its busiest pixel is far above any other window's
    mag, _ = S.tap_magnitudes(s, S.V)
    g = S.MOTION_CAP // 2
    assert mag[g].sum() > 0.5 * S.GIANT
    others = np.delete(mag, g, axis=0)
    assert mag[g].max() > 1000 * others.max()
    # the images are f32 values, the images of the same windows in reverse order are the same images
    iwe = S.linvel_iwe(s, S.V)
    assert (iwe.astype(np.float32) == iwe).all()
    r = S.reversed_stream(s)
    assert np.array_equal(S.linvel_iwe(r, S.V), iwe[::-1])


def test_timestamp_images_are_exact():
    s = S.exact_stream(S.TIMESTAMP_CAP, giant_at=S.TIMESTAMP_CAP - 1, seed=2)
    S.assert_exactly_summable(s, S.exact_velocities())
    Si, Ci = S.linvel_ts_images(s, S.V)
    assert (Si.astype(np.float32) == Si).all() and (Ci.astype(np.float32) == Ci).all()
    f, T = S.timestamp_f(Si, Ci)
    empty = s["sizes"] == 0
    assert (f[empty] == 0).all() and (f[~empty] >= 0).all()


def test_window_sizes_are_skewed():
    B = S.MOTION_CAP
    for giant_at in (0, B // 2, B - 1):
        sizes = S.window_sizes(B, giant_at, seed=3)
        assert sizes[giant_at] == S.GIANT and (np.delete(sizes, giant_at) <= 7).all()
        small = np.delete(sizes, giant_at)
        assert 0.18 < (small == 0).mean() < 0.22
        assert 0.08 < (small == 1).mean() < 0.12
        assert ((small >= 2) & (small <= 7)).mean() > 0.65 and set(np.unique(small)) == set(range(8))
        # the mean window the event grid is sized from is a few dozen events: one CTA per window
        assert sizes.sum() / B < 2048
    s = S.random_stream(1000, giant_at=10, seed=4)
    assert s["off"][-1] == s["x"].shape[0] and s["sizes"][10] == S.GIANT
    assert (s["d"] < 0).all() and (s["x"] >= 0).all() and (s["x"] < S.W).all()


def test_batch_sizes_cross_the_python_chunks():
    """the chunks the GPU tests rely on, from the rule of _candidates / _ts_candidates with the real caps and budgets"""
    from event_utils_b200.contrast_max import motion_objective as MO
    from event_utils_b200.contrast_max import motion_timestamp_objective as MT
    L = _lib()
    H, W = S.H, S.W

    def contrast(B, J):
        return S.window_chunk(B, J, 65535, L.evk_cmax_motion_candidates_workspace_bytes(1, min(J, 32), H, W),
                              MO.CANDIDATES_WORKSPACE_BYTES)

    def timestamp(B, J):
        return S.window_chunk(B, J, 32767, L.evk_motion_timestamp_candidates_workspace_bytes(1, min(J, 32), H, W),
                              MT.TIMESTAMP_CANDIDATES_WORKSPACE_BYTES)
    # the torch candidate functions: B = 4095 (contrast) / 2047 (timestamp) with J = 70
    assert S.chunk_sizes(4095, contrast(4095, 70)) == [2047, 2047, 1]
    assert S.chunk_sizes(2047, timestamp(2047, 70)) == [1023, 1023, 1]
    assert [min(32, 70 - j) for j in range(0, 70, 32)] == [32, 32, 6]
    # the fits' 5x5 linvel grid (J = 25): one chunk plus one window
    assert contrast(2621, 25) == 2621 and S.chunk_sizes(2622, contrast(2622, 25)) == [2621, 1]
    assert timestamp(1310, 25) == 1310 and S.chunk_sizes(1311, timestamp(1311, 25)) == [1310, 1]
    # at this canvas no budget binds: only the caps do
    for jc in (1, 8, 25, 32):
        assert MO.CANDIDATES_WORKSPACE_BYTES // L.evk_cmax_motion_candidates_workspace_bytes(1, jc, H, W) > 65535 // jc
        assert (MT.TIMESTAMP_CANDIDATES_WORKSPACE_BYTES // L.evk_motion_timestamp_candidates_workspace_bytes(1, jc, H, W)
                > 32767 // jc)
    # the entries' caps: one candidate per window fills them exactly
    assert contrast(65535, 1) == 65535 and timestamp(32767, 1) == 32767
    assert contrast(65536, 1) == 65535 and timestamp(32768, 1) == 32767


def test_fit_chunks_of_the_forward_and_gradient_calls():
    from event_utils_b200.contrast_max import motion_fit as MF
    from event_utils_b200.contrast_max import motion_timestamp_fit as MTF
    L = _lib()
    per = L.evk_cmax_motion_objective_workspace_bytes(1, S.H, S.W) + 4 * S.HC * S.WC
    assert MF.fit_window_chunk(65536, per, MF.FIT_WORKSPACE_BYTES, MF.FIT_MAX_WINDOWS) == 65535
    assert MF.fit_window_chunk(65535, per, MF.FIT_WORKSPACE_BYTES, MF.FIT_MAX_WINDOWS) == 65535
    assert MF.fit_window_chunk(32768, per, MF.FIT_WORKSPACE_BYTES, MTF.TIMESTAMP_FIT_MAX_WINDOWS) == 32767
    assert MF.fit_window_chunk(0, per, MF.FIT_WORKSPACE_BYTES, MF.FIT_MAX_WINDOWS) == 1
    # the budget binds at 180x240: about 2 MB per window
    per_big = L.evk_cmax_motion_objective_workspace_bytes(1, 180, 240) + 4 * 181 * 241
    wb = MF.fit_window_chunk(65535, per_big, MF.FIT_WORKSPACE_BYTES, MF.FIT_MAX_WINDOWS)
    assert 1000 < wb < 4096 and wb * per_big <= MF.FIT_WORKSPACE_BYTES
    # the workspace of a chunk is no more than the chunk's windows' workspaces
    assert L.evk_cmax_motion_objective_workspace_bytes(wb, 180, 240) + 4 * wb * 181 * 241 <= MF.FIT_WORKSPACE_BYTES + 4096


def test_voxel_stream_is_exact_in_every_window():
    """each window's own t0 = t[first] and dt = t[last] - t0 are its t0_w and dt_w, tn = k / 16 exactly in f32, every
    cell sum of |weight| is below 2^20 (so every partial sum is an f32 value) and the backward's f64 window sums of a
    voxel_incoming gradient are exact"""
    f32 = np.float32
    nw = 100000
    s = S.voxel_stream(nw, giant_at=nw // 2, seed=5)
    off, sizes = s["off"], s["sizes"]
    two = np.flatnonzero(sizes >= 2)
    first, last = off[two], off[two + 1] - 1
    t0 = s["t"][first]
    dt = (s["t"][last] - t0).astype(f32)
    assert (t0 == two % 64).all() and (dt == 2.0 ** (two % 4 - 1)).all()
    w = S.window_ids(off)
    m = sizes[w] >= 2
    t0e = np.zeros(nw, f32)
    dte = np.ones(nw, f32)
    t0e[two], dte[two] = t0, dt
    tn = (((s["t"] - t0e[w]).astype(f32) / dte[w]).astype(f32) * f32(S.VOXEL_BINS - 1)).astype(f32)
    assert (tn[m] == s["k"][m] / 16.0).all()
    assert ((s["x"] >= 0) & (s["x"] < S.W) & (s["y"] >= 0) & (s["y"] < S.H)).all()
    grids = S.voxel_grids(s)
    assert (grids.astype(f32) == grids).all() and (grids * 16 == np.round(grids * 16)).all()
    mag = S.voxel_grids(dict(s, p=np.abs(s["p"])))
    assert mag.max() <= 2.0 ** 20 and mag[nw // 2].max() > 1000 * np.delete(mag, nw // 2, axis=0).max()
    # the backward's f64 window sums: G = p sum_b g[b] s_b (s_b in 0, +-1/2, +-1) on the 1/32 grid with |G| <= 16, G tn on
    # the 1/512 grid: a sum of 2^21 such terms stays far below 2^53
    g = S.voxel_incoming(nw, 6)
    assert (g * 16 == np.round(g * 16)).all() and np.abs(g).max() <= 8
    assert S.GIANT * 16 * (S.VOXEL_BINS - 1) * 512 < 2.0 ** 53
    gp = S.voxel_grad_p(s, g)
    assert np.isfinite(gp[m]).all() and (gp[m].astype(f32) == gp[m]).all()
    # reversing the windows reverses the grids
    assert np.array_equal(S.voxel_grids(S.reversed_stream(s)), grids[::-1])
