"""Family-independent pieces of the candidates-pass tests of the planar and camera models (test_gpu_planar_motion.py,
test_gpu_camera_rotation.py, test_gpu_camera_motion.py) -- TEST INFRASTRUCTURE ONLY.

A candidate set gives every window J parameter vectors that share no component (distinct_sets), so that a pass which
scores candidate j with another candidate's parameters, or mixes up a segmentation's (m, j), changes f.  Candidate
GONE keeps no event, candidate PARTIAL keeps part of them, and for J >= 32 candidate NAN of window 0 has a NaN
component.  The streams (candidate_stream) keep only events whose reference warp under every candidate of their window
lies at least 1e-3 px from the integers or is not kept at all, so f32 rounding moves no tap or keep decision; the
sparse streams (sparse_pick) keep events whose footprints lie `gap` px apart under every candidate, so every image
pixel sums at most one tap.  The assertions compare a pass with its per-candidate forwards."""
import numpy as np

from motion_objective_reference import contributes

JS = (1, 7, 32, 70)
GONE, PARTIAL, NAN = 1, 2, 3


def no_event_value(name, H, W):
    """f of a window whose image is zero: the contrast objectives of tests/flow_objective_reference.py, and 0 for the
    timestamp loss (name None)"""
    return {None: 0.0, "variance": 0.0, "sos": 0.0, "soe": -1.0, "sosa": -float((H + 1) * (W + 1))}[name]


def distinct_sets(base, J, rng, spread, gone=None, partial=None, rel=0.2):
    """(B,J,K) f64: window b's base[b] perturbed independently per candidate and component, by up to `rel` of its
    value plus up to `spread` (K,); candidate 0 is the base itself and, when given, GONE the vector `gone` and PARTIAL
    `partial`, each moved by 1e-3 of that, so that no two candidates of a window share a component"""
    base = np.asarray(base, np.float64)
    B, K = base.shape
    spread = np.asarray(spread, np.float64)
    c = base[:, None, :] * (1 + rng.uniform(-rel, rel, (B, J, K))) + rng.uniform(-1, 1, (B, J, K)) * spread
    c[:, 0] = base
    for j, v in ((GONE, gone), (PARTIAL, partial)):
        if v is not None and J > j:
            c[:, j] = np.asarray(v, np.float64) + rng.uniform(-1e-3, 1e-3, (B, K)) * (np.abs(v) + spread)
    return c


def with_nan(cand):
    """a copy of cand whose candidate NAN of window 0 has a NaN third component (J >= 32)"""
    c = cand.copy()
    if c.shape[1] >= 32:
        c[0, NAN, 2] = np.nan
    return c


def assert_distinct(cand):
    """no two candidates of a window (of a window's models too, for (B,M,J,K)) share a finite component"""
    c = np.asarray(cand).reshape(cand.shape[0], -1, cand.shape[-1])
    for b in range(c.shape[0]):
        for k in range(c.shape[2]):
            v = c[b, :, k][np.isfinite(c[b, :, k])]
            assert np.unique(v).size == v.size, (b, k)


def safe(warped):
    """events whose warp (xw, yw) under every candidate of `warped` lies at least 1e-3 px from every integer or is not
    finite (an event that is not kept): f32 rounding can move neither its taps nor its keep decision"""
    ok = np.ones(warped[0][0].shape, bool)
    with np.errstate(invalid="ignore"):
        for xw, yw in warped:
            for c in (xw, yw):
                ok &= ~np.isfinite(c) | (np.abs(c - np.round(c)) >= 1e-3)
    return ok


def draw(rng, n, H, W, d_range=(-0.1, -0.05)):
    """n random events in the sensor, sorted d = t - t0 in d_range on a 2^-12 grid, rho in [1/8, 1]"""
    x = (rng.random(n) * (W - 1)).astype(np.float32)
    y = (rng.random(n) * (H - 1)).astype(np.float32)
    lo, hi = (int(round(-v * 4096)) for v in d_range)
    d = (-np.sort(rng.integers(hi, lo + 1, n))[::-1] / 4096.0).astype(np.float32)
    p = (rng.integers(0, 2, n) * 2 - 1).astype(np.float32)
    rho = rng.uniform(0.125, 1.0, n).astype(np.float32)
    return x, y, d, p, rho


def candidate_stream(seed, sizes, cands, warp, H, W):
    """Windows of exactly sizes[b] events, safe (above) under every finite candidate of cands[b] ((J,K) or (M,J,K)):
    x, y, d, p, rho (f32) and the offsets.  d lies in [-0.1, -0.05], away from 0, where every motion is the identity.
    warp(x, y, d, rho, prm) -> (xw, yw), NaN where an event is not kept."""
    rng = np.random.default_rng(seed)
    parts = []
    for b, n in enumerate(sizes):
        ev = draw(rng, 2 * n + 16, H, W)
        prms = [q for q in np.asarray(cands[b]).reshape(-1, np.shape(cands)[-1]) if np.isfinite(q).all()]
        ok = np.flatnonzero(safe([warp(ev[0], ev[1], ev[2], ev[4], q) for q in prms]))
        assert ok.size >= n, (b, ok.size, n)
        pick = np.sort(rng.choice(ok, n, replace=False))
        parts.append([a[pick] for a in ev])
    off = np.concatenate(([0], np.cumsum(sizes))).astype(np.int64)
    return [np.concatenate(a) for a in zip(*parts)] + [off]


def kept(warped, H, W):
    """(J, n) mask of the events each candidate's warp keeps"""
    return np.array([contributes(xw, yw, H, W) for xw, yw in warped])


def sparse_pick(warped, H, W, gap=3):
    """indices of the events that every candidate keeps, 1e-3 px from the integers, whose footprints' corners lie at
    least `gap` px apart under every candidate: every image pixel then sums at most one tap"""
    ok = kept(warped, H, W).all(0) & safe(warped)
    taken = np.zeros((len(warped), H + 1 + 2 * gap, W + 1 + 2 * gap), bool)
    pick = []
    for i in np.flatnonzero(ok):
        cells = [(int(np.floor(xw[i])) + gap, int(np.floor(yw[i])) + gap) for xw, yw in warped]
        if any(taken[j, cy - gap:cy + gap + 1, cx - gap:cx + gap + 1].any() for j, (cx, cy) in enumerate(cells)):
            continue
        for j, (cx, cy) in enumerate(cells):
            taken[j, cy, cx] = True
        pick.append(i)
    return np.array(pick, np.int64)


def taps_per_pixel(xw, yw, H, W):
    """the most bilinear taps any pixel of the (H+1, W+1) canvas receives from the kept events of one warp"""
    k = contributes(xw, yw, H, W)
    px, py = np.floor(xw[k]).astype(np.int64), np.floor(yw[k]).astype(np.int64)
    n = np.zeros((H + 1, W + 1), np.int64)
    for dy in (0, 1):
        for dx in (0, 1):
            np.add.at(n, (py + dy, px + dx), 1)
    return int(n.max())


def assert_forwards(f, ref, rtol=1e-6, what=""):
    """every entry of a (B,J) or (B,M,J) pass equals the per-candidate forward"""
    assert f.shape == ref.shape and f.dtype == np.float64, (what, f.shape, ref.shape)
    assert np.isfinite(f).all(), what
    np.testing.assert_allclose(f, ref, rtol=rtol, atol=0, err_msg=what)


def assert_edges(f, none, empty=(), what=""):
    """the entries of the empty windows and of the candidate GONE are the no-event value"""
    for b in empty:
        np.testing.assert_allclose(f[b], none, rtol=1e-12, atol=0, err_msg="%s: empty window %d" % (what, b))
    if f.shape[-1] > GONE:
        np.testing.assert_allclose(f[..., GONE], none, rtol=1e-12, atol=0, err_msg="%s: no event kept" % what)


def check_sets(master, run, forwards, reference, none, empty=(), what=""):
    """The pass run(cand) -> (B,J) f64 over the sets master[:, :J] for J in JS (with_nan): every entry against the
    per-candidate forwards(cand) to 1e-6, the edges and the NaN candidate's isolation, and at J = 7 against
    reference(cand) -> ((B,J) f64, rtol), the family's f64 reference"""
    for J in JS:
        cand = with_nan(master[:, :J])
        w = "%s J=%d" % (what, J)
        f = run(cand)
        assert_forwards(f, forwards(cand), what=w)
        assert_edges(f, none, empty, w)
        assert_nan_isolated(run, cand, f, none, w)
        if J == 7:
            fr, rtol = reference(cand)
            np.testing.assert_allclose(f, fr, rtol=rtol, atol=1e-30, err_msg=w + " against the reference")


SEG_JS = (0, 1, 5, 36)


def check_segmentation(f, forward, cand, reference, monkeypatch, module, budget, run):
    """A segmentation candidates pass f (B,M,J) of cand (B,M,J,K), J = 37: the columns SEG_JS against forward(cand[:, :,
    j]) -> (B,M) to 1e-6, column 1 against reference(cand[:, :, 1]) -> ((B,M), rtol), and run() again with the
    module's SEGMENT_CANDIDATES_WORKSPACE_BYTES at `budget` changes no value"""
    assert f.shape == cand.shape[:3] and f.dtype == np.float64
    for j in SEG_JS:
        assert_forwards(f[:, :, j], forward(np.ascontiguousarray(cand[:, :, j])), what="j=%d" % j)
    fr, rtol = reference(np.ascontiguousarray(cand[:, :, 1]))
    np.testing.assert_allclose(f[:, :, 1], fr, rtol=rtol, atol=1e-30, err_msg="against the reference")
    with monkeypatch.context() as m:
        m.setattr(module, "SEGMENT_CANDIDATES_WORKSPACE_BYTES", budget)
        many = run()
    np.testing.assert_allclose(many, f, rtol=1e-6, atol=0, err_msg="window chunks")


def check_chunks(monkeypatch, budgets, run, forwards, cand, what=""):
    """run(cand) whole and again with every (module, attribute, bytes) of budgets set: each entry equals the whole run
    and the per-candidate forwards(cand)"""
    one = run(cand)
    with monkeypatch.context() as m:
        for module, attr, v in budgets:
            m.setattr(module, attr, v)
        many = run(cand)
    np.testing.assert_allclose(many, one, rtol=1e-6, atol=0, err_msg=what + ": chunked against whole")
    assert_forwards(many, forwards(cand), what=what)


def assert_nan_isolated(run, cand, f, none, what=""):
    """cand[0, NAN] has a NaN component: its entry is the no-event value, and a finite candidate in its place changes
    no other entry.  run(cand) -> f of the pass."""
    if cand.shape[1] < 32:
        return
    np.testing.assert_allclose(f[0, NAN], none, rtol=1e-12, atol=0, err_msg="%s: NaN candidate" % what)
    c2 = cand.copy()
    c2[0, NAN] = cand[0, 0]
    f2 = run(c2)
    others = np.ones(f.shape, bool)
    others[0, NAN] = False
    np.testing.assert_allclose(f2[others], f[others], rtol=1e-6, atol=0, err_msg="%s: NaN isolation" % what)
