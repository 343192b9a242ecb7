"""No-GPU checks of the premises of tests/test_gpu_batch_limits_models.py: the exact embeddings of
tests/batch_limit_streams.py reproduce the linvel warp bit for bit in every family's f32 arithmetic, the streams stay
exactly summable, the random variant's safety filter works, and the batch sizes and candidate counts the GPU tests pick
cross the window chunks and candidate passes of every family's candidates function and fit."""
import itertools

import numpy as np
import pytest

import batch_limit_streams as S
import depth_grid_reference as DR
import grid_flow_reference as GR
import model_grad_bounds as MB
import planar_motion_reference as P

f32 = np.float32


def _lib():
    from event_utils_b200 import _lib
    return _lib.load()


def _all_events():
    """every (x, y, d) sensor_stream can draw: x and y on the quarter grid of the sensor, d on the 2^-6 grid in
    [-1/16, 0]"""
    xs = np.arange(0, 4 * (S.W - 1) + 1) / 4.0
    ys = np.arange(0, 4 * (S.H - 1) + 1) / 4.0
    ds = -np.arange(0, 5) / 64.0
    x, y, d = (a.ravel().astype(f32) for a in np.meshgrid(xs, ys, ds, indexing="ij"))
    return x, y, d


def _linvel(x, y, d, v):
    return (x.astype(np.float64) - d.astype(np.float64) * v[0], y.astype(np.float64) - d.astype(np.float64) * v[1])


@pytest.mark.parametrize("family", S.EXACT_FAMILIES)
def test_exact_embedding_is_the_linvel_warp_bit_for_bit(family):
    """For every event the stream can hold, every velocity of EXACT_VELOCITIES and every window rho, the family's f32
    warp at exact_rows equals x - d vx, y - d vy exactly: the planar models through warp_f32, the camera motion and
    depth grid through camera_warp_jac's f32 restatement of cam_rotate / cam_project (w = 0 takes the Rodrigues series
    branch; b + A c + B e is b exactly), the grid flow through event_flow_f32 and the depth grid's rho through
    event_rho_f32 on the full-resolution grid"""
    x, y, d = _all_events()
    for v, rho in itertools.product(S.exact_velocities(), S.EXACT_RHOS):
        want = _linvel(x, y, d, v)
        vel, r = v[None], np.array([rho])
        if family in ("affine", "homography", "segmentation"):
            kind = "affine" if family == "segmentation" else family
            got = P.warp_f32(kind, x, y, d, S.exact_rows(family, vel)[0], S.CENTRE)
        elif family == "grid_flow":
            u, w = GR.event_flow_f32(x, y, S.exact_rows(family, vel)[0], S.H, S.W)
            assert (u == -v[0]).all() and (w == -v[1]).all()
            got = (x + u * d).astype(f32), (y + w * d).astype(f32)
        else:
            if family == "camera_motion":
                rows, re = S.exact_rows(family, vel, r)[0], np.full(x.shape, rho, f32)
            else:
                rows, nodes = S.exact_rows(family, vel, r)
                rows, re = rows[0], DR.event_rho_f32(x, y, nodes[0], S.H, S.W)
                assert (re == f32(rho)).all()
            got = MB.camera_warp_jac(x, y, d, rows[:3], tuple(rows[6:8]) + S.INTR[2:], v=rows[3:6], rho=re, kind="f32")[:2]
        for a, b in zip(got, want):
            assert a.dtype == f32 and np.array_equal(a.astype(np.float64), b), (family, v, rho)
        if family not in ("camera_motion", "depth_grid"):
            break                                   # rho plays no part


def test_depth_grid_candidate_embedding_is_exact():
    """the depth grid's candidates-entry test: motion rows built for rho 1 and uniform full-resolution nodes of a rho r of
    DEPTH_CANDIDATE_RHOS warp every event exactly to x - d (r vx), y - d (r vy), and the stream stays exactly summable
    under every such velocity"""
    x, y, d = _all_events()
    vels = []
    for v, r in itertools.product(S.exact_velocities(), S.DEPTH_CANDIDATE_RHOS):
        rows = S.exact_rows("camera_motion", v[None], np.ones(1))[0]
        re = DR.event_rho_f32(x, y, np.full((S.H, S.W), r, f32), S.H, S.W)
        assert (re == f32(r)).all()
        got = MB.camera_warp_jac(x, y, d, rows[:3], tuple(rows[6:8]) + S.INTR[2:], v=rows[3:6], rho=re, kind="f32")[:2]
        for a, b in zip(got, _linvel(x, y, d, r * v)):
            assert np.array_equal(a.astype(np.float64), b), (v, r)
        vels.append(r * v)
    S.assert_exactly_summable(S.sensor_stream(S.MOTION_CAP, None, seed=5), vels)


def test_camera_rotation_has_no_exact_embedding():
    """the camera rotation cannot translate: at w = 0 it is the identity, so only linvel's v = 0 embeds, and no window
    could get its own velocity; its tests use the random variant only"""
    x, y, d = _all_events()
    xw, yw = MB.camera_warp_jac(x, y, d, (0.0, 0.0, 0.0), S.INTR, kind="f32")[:2]
    assert np.array_equal(xw, x) and np.array_equal(yw, y)
    assert "camera_rotation" not in S.EXACT_FAMILIES


@pytest.mark.parametrize("flow", [False, True])
def test_sensor_stream_is_exactly_summable(flow):
    """at the entries' cap with the giant window, under every velocity; memberships on the 1/4 grid keep it so"""
    s = S.sensor_stream(S.MOTION_CAP, giant_at=S.MOTION_CAP // 2, seed=1, M=4)
    S.assert_exactly_summable(s, S.exact_velocities(), flow)
    assert (s["x"] >= 0).all() and (s["x"] <= S.W - 1).all() and (s["y"] >= 0).all() and (s["y"] <= S.H - 1).all()
    w = s["w"].astype(np.float64)
    assert (w * 4 == np.round(w * 4)).all() and w.min() == 0.25 and w.max() == 1.0
    # the giant window is the same window wherever it sits, and keeps most of its events
    t = S.sensor_stream(4095, giant_at=0, seed=1)
    g = slice(s["off"][S.MOTION_CAP // 2], s["off"][S.MOTION_CAP // 2 + 1])
    assert np.array_equal(t["x"][:S.GIANT], s["x"][g]) and np.array_equal(t["d"][:S.GIANT], s["d"][g])
    mag, _ = S.tap_magnitudes(s, S.V, flow)
    assert mag[S.MOTION_CAP // 2].sum() > 0.5 * S.GIANT
    # every window has one rho
    rho = S.window_rhos(S.MOTION_CAP, 1)
    assert np.array_equal(s["r"], rho[S.window_ids(s["off"])].astype(f32))


def test_flow_keep_rule_differs_at_zero():
    """x' = 0 is kept by the flow entries (0 <= x') and not by the motion entries (0 < x'): the stream has such events"""
    s = S.sensor_stream(4095, giant_at=7, seed=2)
    _, _, _, _, km = S.linvel_taps(s, S.V)
    _, _, _, _, kf = S.linvel_taps(s, S.V, flow=True)
    assert (km <= kf).all() and (kf & ~km).sum() > 1000


@pytest.mark.parametrize("family", S.FAMILIES)
def test_random_variant_is_safe_after_the_drop(family):
    """drop_unsafe leaves no event of the sampled windows within 1e-3 px of an integer, and keeps most of them"""
    M = 2 if family == "segmentation" else None
    B = 300
    s = S.random_stream_models(B, giant_at=150, seed=3, M=M)
    rows = S.random_rows(family, B, 4, M)
    idx = S.sampled_windows(s["sizes"], 150, 1, count=12)

    def params(b):
        if family == "segmentation":
            return list(rows[b])
        if family == "depth_grid":
            return [(rows[0][b], rows[1][b])]
        return [rows[b]]
    frac = S.drop_unsafe(s, family, idx, params, 0.0)
    assert frac < 0.05
    off = s["off"]
    for b in idx:
        sl = slice(off[b], off[b + 1])
        keep = s["p"][sl] != 0
        for prm in params(b):
            xw, yw = S.family_warp(family, s["x"][sl], s["y"][sl], s["d"][sl], s["r"][sl], prm)
            with np.errstate(invalid="ignore"):
                near = np.isfinite(xw) & np.isfinite(yw) & ((np.abs(xw - np.round(xw)) < 1e-3) |
                                                            (np.abs(yw - np.round(yw)) < 1e-3))
            assert not (near & keep).any()
    if family in ("homography", "camera_rotation", "camera_motion", "depth_grid"):
        # every term in play: a perspective, a rotation, a forward velocity, a non-uniform grid
        r = rows[0] if family == "depth_grid" else rows
        col = {"homography": 6, "camera_rotation": 0, "camera_motion": 5, "depth_grid": 5}[family]
        assert (np.abs(r[:, col]) > 0).all()


# ---- the chunk rules the GPU tests cross ----------------------------------------------------------------------------
def candidates_chunks(stem, B, J, cap, budget, M=None, grid=None):
    """_chunked_candidates' rule: (window chunk sizes, candidate pass sizes) from the entry's workspace query"""
    from event_utils_b200.contrast_max._batched import MAX_CANDIDATES, MAX_GRID_CANDIDATE_NODES
    L = _lib()
    jc = min(J, MAX_CANDIDATES // (M or 1))
    if grid:
        jc = max(1, min(jc, MAX_GRID_CANDIDATE_NODES // (grid[0] * grid[1])))
    ms = () if M is None else (M,)
    query = tuple(grid) if grid else ()
    per = getattr(L, stem + "_workspace_bytes")(1, *ms, jc, *query, S.H, S.W)
    wb = max(1, min(B, budget // per, cap // ((M or 1) * jc)))
    return S.chunk_sizes(B, wb), [min(jc, J - j) for j in range(0, J, jc)]


# (family, loss) -> (entry stem, cap, M, grid) of the candidates functions, with the B the GPU tests run at J = 70
CANDIDATE_CASES = {
    ("affine", "contrast"): ("evk_cmax_motion_candidates", 65535, None, None, 4095),
    ("affine", "timestamp"): ("evk_motion_timestamp_candidates", 32767, None, None, 2047),
    ("camera_motion", "contrast"): ("evk_cmax_motion_depth_candidates", 65535, None, None, 4095),
    ("camera_motion", "timestamp"): ("evk_motion_timestamp_depth_candidates", 32767, None, None, 2047),
    ("grid_flow", "contrast"): ("evk_cmax_grid_flow_candidates", 65535, None, S.RANDOM_GRID, 4095),
    ("grid_flow", "timestamp"): ("evk_grid_flow_timestamp_candidates", 32767, None, S.RANDOM_GRID, 2047),
    ("depth_grid", "contrast"): ("evk_cmax_depth_grid_candidates", 65535, None, S.RANDOM_GRID, 4095),
    ("depth_grid", "timestamp"): ("evk_depth_grid_timestamp_candidates", 32767, None, S.RANDOM_GRID, 2047),
    ("segmentation", 2): ("evk_cmax_motion_segment_candidates", 65535, 2, None, 4095),
    ("segmentation", 3): ("evk_cmax_motion_segment_candidates", 65535, 3, None, 4369),
    ("segmentation", 4): ("evk_cmax_motion_segment_candidates", 65535, 4, None, 4095),
}


def test_candidates_cross_three_window_chunks_and_three_passes():
    """J = 70 at the GPU tests' B: three window chunks, the last of one window, and at least three candidate passes,
    under the real budgets (which do not bind at this canvas: only the caps do)"""
    from event_utils_b200.contrast_max import motion_objective as MO
    from event_utils_b200.contrast_max import motion_segmentation as MS
    from event_utils_b200.contrast_max import motion_timestamp_objective as MT
    for (family, loss), (stem, cap, M, grid, B) in CANDIDATE_CASES.items():
        budget = (MS.SEGMENT_CANDIDATES_WORKSPACE_BYTES if M else
                  MT.TIMESTAMP_CANDIDATES_WORKSPACE_BYTES if cap == 32767 else MO.CANDIDATES_WORKSPACE_BYTES)
        chunks, passes = candidates_chunks(stem, B, 70, cap, budget, M, grid)
        jc = passes[0]
        assert len(chunks) == 3 and chunks[-1] == 1 and chunks[0] == cap // ((M or 1) * jc), (family, loss, chunks)
        assert len(passes) >= 3 and sum(passes) == 70, (family, loss, passes)
        # a window cap left without M would take M times the windows: past the entry's canvas cap
        assert M is None or (cap // jc) * M * jc > cap
    # the pass maxima the entry tests use: 32 for the parametric and grid losses (12288 // (gh gw) >= 32 for every grid
    # of the 6x10 sensor), 32 // M for the segmentation
    from event_utils_b200.contrast_max._batched import MAX_CANDIDATES, MAX_GRID_CANDIDATE_NODES
    assert MAX_CANDIDATES == 32 and MAX_GRID_CANDIDATE_NODES // (S.H * S.W) >= MAX_CANDIDATES
    for M in (2, 3, 4):
        assert candidates_chunks("evk_cmax_motion_segment_candidates", 10 ** 6, 70, 65535, 4 << 30, M)[1][0] == 32 // M


def test_segment_chunk_and_the_fits_cross_the_entry_caps():
    """cap + 1 windows run in two chunks: the forward and gradient of every fit, the segmentation's forward, gradient
    and assignment (65535 // M), and a line search's candidates pass (8 steps) in more"""
    from event_utils_b200.contrast_max import motion_fit as MF
    from event_utils_b200.contrast_max import motion_segmentation as MS
    from event_utils_b200.contrast_max import motion_timestamp_fit as MTF
    L = _lib()
    H, W = S.H, S.W
    for M in (2, 3, 4):
        cap = MS.MAX_CANVASES // M
        # _segment_chunk's rule
        per_window = L.evk_cmax_motion_segment_workspace_bytes(1, M, H, W) + 4 * M * S.HC * S.WC
        assert MF.fit_window_chunk(cap + 1, per_window, MF.FIT_WORKSPACE_BYTES, cap) == cap
        chunks, passes = candidates_chunks("evk_cmax_motion_segment_candidates", cap + 1, 8, 65535, 4 << 30, M)
        assert passes == [min(8, 32 // M)] and len(chunks) == -(-(cap + 1) // (65535 // (M * passes[0]))) >= 2
    gh, gw = 2, 2
    per = {"motion": L.evk_cmax_motion_objective_workspace_bytes(1, H, W) + 4 * S.HC * S.WC,
           "motion_ts": L.evk_motion_timestamp_objective_workspace_bytes(1, H, W) + 4 * 2 * 2 * S.HC * S.WC,
           "grid": L.evk_cmax_grid_flow_objective_workspace_bytes(1, gh, gw, H, W) + 4 * S.HC * S.WC,
           "grid_ts": L.evk_grid_flow_timestamp_objective_workspace_bytes(1, gh, gw, H, W) + 4 * 2 * 2 * S.HC * S.WC,
           "depth": L.evk_cmax_depth_grid_objective_workspace_bytes(1, gh, gw, H, W) + 4 * S.HC * S.WC,
           "depth_ts": L.evk_depth_grid_timestamp_objective_workspace_bytes(1, gh, gw, H, W) + 4 * 2 * 2 * S.HC * S.WC}
    for name, b in per.items():
        cap = MTF.TIMESTAMP_FIT_MAX_WINDOWS if name.endswith("_ts") else MF.FIT_MAX_WINDOWS
        assert MF.fit_window_chunk(cap + 1, b, MF.FIT_WORKSPACE_BYTES, cap) == cap, name
