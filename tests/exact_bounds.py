"""Per-cell error bounds for kernels whose output cells are sums of f32 taps, against the oracle's exact mode
(oracle/evk_oracle.py, exact=True: per cell the f64 sum of the f32 taps, the f64 sum of |tap| and the tap count).
A kernel may add the taps of a cell in any order and grouping; the bound below holds for all of them, so it needs no
tuning, and a tap that is lost, doubled or sent to another cell shows up in the cell it belongs to whenever its weight
exceeds that cell's bound -- however hot the rest of the image is."""
import collections

import numpy as np

U32 = 2.0 ** -24          # unit roundoff of f32
Q22 = 2.0 ** -23          # per-tap quantisation of the 2^22 fixed-point tables (voxel / bilinear image / on-chip IWE)


def gamma(m):
    """gamma(m) = m u / (1 - m u): the classic bound on the relative error of m f32 additions in any order."""
    mu = np.asarray(m, np.float64) * U32
    return mu / (1.0 - mu)


def exact_error_bound(ex, q=0.0, offset=0.0):
    """Per-cell bound on |kernel - exact| for an output whose cells are sums of the f32 taps in `ex` (an oracle Exact:
    f64 tap sum, f64 |tap| sum, tap count k), added in any order and grouping: gamma(k+4) S + k q.  The +4 covers the
    partial sums a kernel folds together (quad / block / replica partials); q is the per-tap quantisation of the
    fixed-point path (0 where it is exact).  `offset`: a background the sums start from (`fill`)."""
    k = ex.cnt + (1.0 if offset != 0 else 0.0)
    return gamma(k + 4) * (ex.abs + abs(offset)) + k * q


def assert_within_exact(out, ex, q=0.0, offset=0.0, what=""):
    """Every cell of `out` within exact_error_bound of the exact sum (offset + sum of taps).  Cells whose exact sum is
    not finite must match it exactly (NaN where NaN, the same infinity)."""
    out = np.asarray(out, np.float64)
    ref = ex.sum + offset
    assert out.shape == ref.shape, (what, out.shape, ref.shape)
    fin = np.isfinite(ref)
    nr, no = np.isnan(ref), np.isnan(out)
    assert (nr == no).all(), "%s: NaN pattern differs at %s" % (what, np.argwhere(nr != no)[:5].tolist())
    inf = ~fin & ~nr
    assert (out[inf] == ref[inf]).all(), "%s: infinities differ" % what
    err = np.abs(out[fin] - ref[fin])
    bound = exact_error_bound(ex, q, offset)[fin]
    bad = err > bound
    if bad.any():
        idx = np.argwhere(fin)[np.flatnonzero(bad)[:5]]
        raise AssertionError("%s: %d cells outside the exact bound, e.g. %s: out %r exact %r bound %r (k %r)" % (
            what, int(bad.sum()), idx.tolist(), out[tuple(idx.T)].tolist(), ref[tuple(idx.T)].tolist(),
            bound[np.flatnonzero(bad)[:5]].tolist(), ex.cnt[tuple(idx.T)].tolist()))


def assert_ratio_within_exact(out, num, den, q=0.0, den_offset=1.0, what=""):
    """Timestamp images: out = fl(T / C) with T, C two sums of taps (num, den: oracle Exact) and C starting at
    `den_offset` (the count images start at one).  The bounds of T and C are carried through the division:
    |T'/C' - T/C| <= (eT C + |T| eC) / (C (C - eC)), plus one rounding of the quotient."""
    out = np.asarray(out, np.float64)
    T, C = num.sum, den.sum + den_offset
    eT = exact_error_bound(num, q)
    eC = exact_error_bound(den, q, den_offset)
    ref = T / C
    fin = np.isfinite(ref)
    assert (np.isnan(ref) == np.isnan(out)).all(), what + ": NaN pattern differs"
    assert (out[~fin & ~np.isnan(ref)] == ref[~fin & ~np.isnan(ref)]).all(), what + ": infinities differ"
    assert (C[fin] - eC[fin] > 0).all(), what + ": count image too close to zero for the bound"
    Cm = C - eC
    bound = (eT * C + np.abs(T) * eC) / (C * Cm) + U32 * (np.abs(T) + eT) / Cm
    err = np.abs(out - ref)
    bad = fin & (err > bound)
    assert not bad.any(), "%s: %d cells outside the bound, e.g. %s: out %r exact %r bound %r" % (
        what, int(bad.sum()), np.argwhere(bad)[:3].tolist(), out[bad][:3].tolist(), ref[bad][:3].tolist(), bound[bad][:3].tolist())


def assert_within_grad_bound(out, g, what=""):
    """A backward kernel's per-event output against its f64 reference g (tests/grad_reference.py Grad): every event
    within (gamma(m) + gamma64(m)) M + extra of the reference value, m being the roundings on the longest path of the
    kernel's expression.  Where the reference value is not finite the output must match it exactly (NaN where NaN, the
    same infinity)."""
    from grad_reference import bound_of
    out = np.asarray(out, np.float64).reshape(-1)
    ref = np.asarray(g.v, np.float64).reshape(-1)
    assert out.shape == ref.shape, (what, out.shape, ref.shape)
    nr, no = np.isnan(ref), np.isnan(out)
    assert (nr == no).all(), "%s: NaN pattern differs at %s" % (what, np.flatnonzero(nr != no)[:5].tolist())
    fin = np.isfinite(ref)
    inf = ~fin & ~nr
    assert (out[inf] == ref[inf]).all(), "%s: infinities differ at %s" % (what, np.flatnonzero(inf & (out != ref))[:5].tolist())
    bound = np.broadcast_to(bound_of(g), ref.shape)
    assert np.isfinite(bound[fin]).all(), what + ": bound not finite where the reference is"
    with np.errstate(invalid="ignore"):
        err = np.abs(out - ref)
    bad = fin & ~(err <= bound)
    if bad.any():
        i = np.flatnonzero(bad)[:5]
        raise AssertionError("%s: %d events outside the bound, e.g. %s: out %r ref %r bound %r" % (
            what, int(bad.sum()), i.tolist(), out[i].tolist(), ref[i].tolist(), bound[i].tolist()))


def assert_scalar_within(out, ref, bound, what=""):
    """One f64 sum (value, bound) of a kernel against its reference; a non-finite reference must match exactly."""
    out, ref = float(out), float(ref)
    if not np.isfinite(ref):
        assert (np.isnan(ref) and np.isnan(out)) or out == ref, (what, out, ref)
        return
    assert abs(out - ref) <= bound, "%s: %r vs %r (bound %r)" % (what, out, ref, bound)


# ---- exactly summable streams (tests/edge_cases.py exact_streams) ----------------------------------------------------
EXACT_C = 2048            # CTAs that may share a cell in the image and cmax table paths (at most one wave: 4 per SM)
# The voxel hot-table kernel holds 40 KB of static shared memory, so at most 5 of its CTAs fit on an SM; its launches
# cover 4 waves: 20 CTAs per SM, 4096 up to 204 SMs.
VOXEL_C = 4096


def Exact_of(ex, k):
    """Plane k of an oracle Exact whose arrays have a leading plane axis."""
    return type(ex)(*(a[k] for a in ex))


def _grid_ok(a, g):
    s = np.asarray(a, np.float64) * 2.0 ** g
    return bool((s == np.round(s)).all())


def assert_exactly_summable(exact_of, group, g_hot, F=None, g_fine=12, offset=0.0, C=EXACT_C, what=""):
    """The argument that makes every summation order of a stream exact, checked on the oracle's exact mode run on each
    class of events separately (`exact_of(mask)` -> Exact of the events selected by `mask`).  `group`: per event, 0 =
    fine, 1, 2, ... = hot classes (a bool array: one hot class); `g_hot`: the hot taps' grid exponent, or a dict
    {class: g} (each class is checked on its own grid):
      - the classes have pairwise disjoint supports;
      - fine cells: sums on the 2^-g_fine grid, sum |tap| + |offset| <= 2^(30-F) (half the wrap threshold of the
        table, 256 for F = 22) and <= 2^(24-g_fine);
      - hot cells: sums on the 2^-g grid and 2^g (S + |offset| + 1.5 * 2^(32-F) * C) <= 2^24, S = sum |tap|:
        per CTA the carries of one sign total at most S_c + 2^(32-F) and the residual flushed at the end at most
        2^(31-F), so no partial sum of a table path (F = its fixed-point bits) exceeds that; F = None: plain
        reductions, 2^g (S + |offset|) <= 2^24;
      - float32(sum + offset) == sum + offset in every cell."""
    group = np.asarray(group).astype(int)
    classes = [int(k) for k in np.unique(group)]
    exs = {k: exact_of(group == k) for k in classes}
    for i, a in enumerate(classes):
        for b in classes[i + 1:]:
            both = (exs[a].cnt > 0) & (exs[b].cnt > 0)
            assert not both.any(), "%s: cells with taps of classes %d and %d at %s" % (
                what, a, b, np.argwhere(both)[:5].tolist())
    off = abs(float(offset))
    tot = offset + sum(e.sum for e in exs.values())
    for k, e in exs.items():
        if k == 0:
            assert _grid_ok(e.sum, g_fine) and _grid_ok(offset, g_fine), what + ": fine sums off the 2^-%d grid" % g_fine
            lim = min(2.0 ** (24 - g_fine), 2.0 ** (30 - F) if F is not None else np.inf)
            assert (e.abs + off <= lim).all(), "%s: fine cell |tap| sum %r > %r" % (what, float(e.abs.max()), lim)
            continue
        g = g_hot[k] if isinstance(g_hot, dict) else g_hot
        assert _grid_ok(e.sum, g) and _grid_ok(offset, g), what + ": hot class %d sums off the 2^-%d grid" % (k, g)
        carry = 0.0 if F is None else 1.5 * 2.0 ** (32 - F) * C
        worst = 2.0 ** g * (e.abs.max(initial=0.0) + off + carry)
        assert worst <= 2.0 ** 24, "%s: hot class %d not exactly summable (2^g (S + carries) = %r)" % (what, k, worst)
    assert (tot.astype(np.float32).astype(np.float64) == tot).all(), what + ": a cell sum is not an f32 value"
    return exs


# One output plane of the oracle on an exact stream: f32 result, Exact, out-of-range count, the hot taps' grid (int or
# {class: g}), the fixed-point bits F of the table path (None: plain reductions) and the CTA bound C of its launches
Plane = collections.namedtuple("Plane", "name out ex oob g F C")


def select_events(c, m):
    """The sub-stream of an exact_streams() stream selected by the index / mask m (per-event arrays only)."""
    return {k: (v[m] if k in ("x", "y", "t", "p", "hot", "group") else v) for k, v in c.items()}


def exact_outputs(oracle, c, **kw):
    """The oracle's f32 outputs and exact sums of an exact_streams() stream, one Plane per output plane.
    kw: clip / padding for the images, bilinear=True (+ clip) for the trilinear voxel, abs_polarity for cmax."""
    k = c["kind"]
    if k == "voxel" and not kw.get("bilinear"):
        v, ex, oob = oracle.voxel_f32(c["x"], c["y"], c["t"], c["p"], c["B"], (c["H"], c["W"]), t0=c["t0"], dt=c["dt"],
                                      exact=True)
        return [Plane("voxel", v, ex, oob, {1: 0, 2: 1}, 22, VOXEL_C)]
    if k == "voxel":
        # trilinear: per bin the bilinear image of p * max(0, 1 - |tau - b|) on the (H+1, W+1) canvas; plain reductions
        tn = ((c["t"] - c["t0"]) / c["dt"]) * np.float32(c["B"] - 1)
        res = []
        for b in range(c["B"]):
            wb = np.maximum(np.float32(1) - np.abs(tn - np.float32(b)), np.float32(0)).astype(np.float32)
            img, ex, oob = oracle.image_torch_f32(c["x"], c["y"], (c["p"] * wb).astype(np.float32),
                                                  sensor_size=(c["H"], c["W"]), clip_out_of_range=kw.get("clip", False),
                                                  interpolation="bilinear", exact=True)
            res.append(Plane("trilinear bin %d" % b, img, ex, oob, {1: 2, 2: 4}, None, None))
        return res
    if k in ("nearest", "bilinear"):
        img, ex, oob = oracle.image_torch_f32(c["x"], c["y"], c["p"], sensor_size=(c["H"], c["W"]),
                                              clip_out_of_range=kw.get("clip", False),
                                              interpolation="bilinear" if k == "bilinear" else None,
                                              padding=kw.get("padding", False), exact=True)
        return [Plane(k, img, ex, oob, -19 if k == "nearest" else 1, 10 if k == "nearest" else 22, EXACT_C)]
    iwe, d, ex, oob = oracle.iwe_linvel((c["vx"], c["vy"]), c["x"], c["y"], c["t"], c["p"], (c["Hs"], c["Ws"]), True,
                                        use_polarity=not kw.get("abs_polarity", False), sensor_size=(c["Hs"], c["Ws"]),
                                        t_ref=c["t_ref"], exact=True)
    return [Plane("iwe", iwe, Exact_of(ex, 0), oob, 2, 22, EXACT_C), Plane("diwe0", d[0], Exact_of(ex, 1), oob, 7, None, None),
            Plane("diwe1", d[1], Exact_of(ex, 2), oob, 7, None, None)]


def check_exactly_summable(oracle, c, **kw):
    """assert_exactly_summable for every output plane of an exact_streams() stream (the oracle runs once per event
    class); returns exact_outputs() of the whole stream."""
    outs = exact_outputs(oracle, c, **kw)
    per_class = {}
    for j, pl in enumerate(outs):
        def exact_of(m, j=j):
            key = m.tobytes()
            if key not in per_class:
                per_class[key] = exact_outputs(oracle, select_events(c, m), **kw)
            return per_class[key][j].ex
        # nearest taps are the polarities themselves: the fine ones lie on the 2^-2 grid
        assert_exactly_summable(exact_of, c["group"], pl.g, pl.F, g_fine=2 if pl.name == "nearest" else 12,
                                C=pl.C or EXACT_C, what="%s %s" % (pl.name, kw))
    return outs


# ---- do the tables wrap? -----------------------------------------------------------------------------------------------
def table_wraps(v, F, C, threads, vec=1):
    """Wraps of ONE shared-memory table slot in each CTA of a grid-stride launch (C CTAs of `threads` threads, `vec`
    events per thread and iteration), the CTA's events taken in index order.  v: per event, the value it adds to the
    slot (0 for the other events).  A slot holds (-2^(31-F), 2^(31-F)) and carries 2^(32-F) when it wraps.
    Returns (up, down, net): per CTA the number of upward and downward wraps and the net carry count."""
    v = np.asarray(v, np.float64)
    cta = ((np.arange(v.shape[0]) // vec) % (C * threads)) // threads
    P = np.bincount(cta, np.maximum(v, 0.0), minlength=C)
    M = np.bincount(cta, np.maximum(-v, 0.0), minlength=C)
    h = 2.0 ** (31 - F)
    up = np.floor((P + h) / (2 * h))
    r = P - 2 * h * up                                   # the slot after the + run, in [-h, h)
    down = np.where(M - r > h, np.floor((M - r - h) / (2 * h)) + 1, 0.0)
    return up, down, up - down


def table_launches(c, sms):
    """The table launches of the exact-sum tests on a GPU with `sms` SMs, as the launch code sizes them, and the value
    each event adds to the hottest slot: [(name, v, F, C, threads, vec)].
      voxel     grid_for: 4096 events per CTA (16-byte aligned SoA) / 1024 (misaligned SoA, AoS, packed), capped at 4
                waves of 4 or 5 resident CTAs per SM (both checked); slot = hot pixel A, bin 0
      images    one wave of 512-thread CTAs, 8192 events per CTA, 16-byte loads; slot = the hot point
      cmax      on-chip image: ceil(n / 8192) CTAs, at most one per SM, 1024 threads, two f64 events per 16-byte load"""
    n, k = c["x"].shape[0], c["kind"]
    g, p = c["group"], c["p"].astype(np.float64)
    if k == "voxel":
        v = np.where((g == 1) & (c["t"] == c["t0"]), p, 0.0)
        return [("voxel soa4", v, 22, min(-(-n // 4096), sms * 20), 256, 4)] + \
               [("voxel 1024/CTA r=%d" % r, v, 22, min(-(-n // 1024), sms * r * 4), 256, 1) for r in (4, 5)]
    if k == "nearest":
        return [("nearest", np.where(g == 1, p, 0.0), 10, -(-n // 8192), 512, 4)]
    if k == "bilinear":
        return [("bilinear", np.where(g == 1, 0.5 * p, 0.0), 22, -(-n // 8192), 512, 4)]
    return [("cmax onchip", np.where(g == 1, 0.25 * p, 0.0), 22, min(-(-n // 8192), sms), 1024, 2)]


def assert_tables_wrap(c, sms, what=""):
    """Every CTA's hot slot wraps upward and back downward in every table launch of the stream; the image and cmax
    cells also receive a non-zero net carry over all CTAs, which a carry sent to the wrong cell cannot hide behind."""
    for name, v, F, C, threads, vec in table_launches(c, sms):
        up, down, net = table_wraps(v, F, C, threads, vec)
        assert up.min() >= 1 and down.min() >= 1, "%s %s: a CTA's slot wraps %d up / %d down" % (
            what, name, up.min(), down.min())
        if not name.startswith("voxel"):
            assert net.sum() != 0, "%s %s: the carries cancel" % (what, name)


def assert_exact(out, ex, offset=0.0, what=""):
    """`out` equals the exact sum (offset + sum of taps) BIT FOR BIT in every cell; cells whose exact sum is not finite
    must match it as assert_within_exact requires (NaN where NaN, the same infinity)."""
    out = np.asarray(out, np.float64)
    ref = ex.sum + offset
    assert out.shape == ref.shape, (what, out.shape, ref.shape)
    nr, no = np.isnan(ref), np.isnan(out)
    assert (nr == no).all(), "%s: NaN pattern differs at %s" % (what, np.argwhere(nr != no)[:5].tolist())
    bad = ~nr & (out != ref)
    if bad.any():
        idx = np.argwhere(bad)[:5]
        raise AssertionError("%s: %d cells differ from the exact sum, e.g. %s: out %r exact %r (k %r)" % (
            what, int(bad.sum()), idx.tolist(), out[tuple(idx.T)].tolist(), ref[tuple(idx.T)].tolist(),
            ex.cnt[tuple(idx.T)].tolist()))
