"""The oracle's exact mode against its own f32 path on the hard edge cases (CPU only): the sequential f32 sums must lie
within the per-cell bound the GPU tests apply to the kernels, and the exact mode must not disturb the f32 results.
Also RobustNorm's order statistics and NaN behaviour against torch (the reference's own kthvalue / clamp / min / max)."""
import numpy as np
import pytest
import torch

from exact_bounds import Q22, assert_ratio_within_exact, assert_within_exact, exact_error_bound, gamma
from edge_cases import hard_cases, replicate


def _img_kw(c, interp):
    return dict(sensor_size=(c["H"], c["W"]), clip_out_of_range=c["clip"], interpolation=interp, padding=c["padding"])


def test_gamma():
    assert gamma(0) == 0.0
    assert gamma(1) == pytest.approx(2.0 ** -24, rel=1e-6)
    assert gamma(2 ** 23) == pytest.approx(1.0)


@pytest.mark.parametrize("big", [False, True])
def test_exact_mode_bounds_the_f32_oracle(oracle, big):
    for c in hard_cases(11, 40):
        if big:
            if c["k"] % 8:
                continue
            c = replicate(c, 20000)
        xyp = (c["x"], c["y"], c["p"])
        v, ex, oob = oracle.voxel_f32(c["x"], c["y"], c["t"], c["p"], c["B"], (c["H"], c["W"]), t0=c["t0"], dt=c["dt"],
                                      exact=True)
        v32, ex2, oob2 = oracle.voxel_f32(c["x"], c["y"], c["t"], c["p"], c["B"], (c["H"], c["W"]), t0=c["t0"],
                                          dt=c["dt"], exact=True)
        assert np.array_equal(v, v32, equal_nan=True) and oob == oob2
        if oob == 0:
            assert np.array_equal(v, oracle.voxel_f32(c["x"], c["y"], c["t"], c["p"], c["B"], (c["H"], c["W"]),
                                                      t0=c["t0"], dt=c["dt"]), equal_nan=True)
        assert_within_exact(v, ex, what="voxel %s" % c["k"])
        for interp in (None, "bilinear"):
            img, ex, oob = oracle.image_torch_f32(*xyp, default=c["fill"], exact=True, **_img_kw(c, interp))
            assert_within_exact(img, ex, offset=float(c["fill"]), what="image %s %s" % (c["k"], interp))
            if oob == 0:
                assert np.array_equal(img, oracle.image_torch_f32(*xyp, default=c["fill"], **_img_kw(c, interp)),
                                      equal_nan=True)
        for kw in (dict(), dict(timestamp_reverse=True), dict(normalize_timestamps=False), dict(padding=False)):
            kw2 = dict(sensor_size=(c["H"], c["W"]), clip_out_of_range=c["clip"])
            kw2.update(kw)
            pos, neg, ex, oob = oracle.timestamp_image_f32(c["x"], c["y"], c["t"], c["p"], exact=True, **kw2)
            for s, img in enumerate((pos, neg)):
                num = type(ex)(*(a[2 * s] for a in ex))
                den = type(ex)(*(a[2 * s + 1] for a in ex))
                assert_ratio_within_exact(img, num, den, what="tsimg %s %s %d" % (c["k"], kw, s))


def test_exact_mode_iwe_and_out_of_canvas_count(oracle):
    rng = np.random.default_rng(3)
    n = 5000
    Hs, Ws = 9, 13
    x = rng.uniform(-2, Ws + 2, n)
    y = rng.uniform(-2, Hs + 2, n)
    x[::7], y[::11] = np.float64(Ws), np.float64(Hs)          # on the (0, W] mask edge and the canvas clip line
    t = np.sort(rng.random(n)) * 0.1
    p = rng.choice([-1.0, 1.0, 0.5], n)
    for params in ((0.0, 0.0), (40.0, -25.0), (-90.0, 60.0)):
        iwe, d, ex, oob = oracle.iwe_linvel(params, x, y, t, p, (Hs + 3, Ws + 3), compute_gradient=True,
                                            sensor_size=(Hs, Ws), exact=True)
        planes = [iwe, d[0], d[1]]
        for k in range(3):
            assert_within_exact(planes[k], type(ex)(*(a[k] for a in ex)), what="iwe plane %d %s" % (k, params))
        if oob:
            with pytest.raises(oracle.OracleIndexError):
                oracle.iwe_linvel(params, x, y, t, p, (Hs + 3, Ws + 3), sensor_size=(Hs, Ws))
        else:
            i2, _ = oracle.iwe_linvel(params, x, y, t, p, (Hs + 3, Ws + 3), sensor_size=(Hs, Ws))
            assert np.array_equal(i2, iwe)
    # a NaN coordinate passes the bounds mask (NaN compares false) and indexes nowhere: counted, not raised
    x[[5, 9]] = np.nan
    _, _, _, oob = oracle.iwe_linvel((0.0, 0.0), x, y, t, p, (Hs + 3, Ws + 3), sensor_size=(Hs, Ws), exact=True)
    assert oob == 2


def test_bound_detects_a_lost_tap(oracle):
    """The bound is tight enough to see one tap of a cold cell go missing next to a hot one."""
    x = np.float32([0.5] * 100000 + [3.25, 3.25])
    y = np.float32([0.5] * 100000 + [1.5, 1.5])
    p = np.float32([1.0] * 100000 + [0.01, 0.01])
    img, ex, _ = oracle.image_torch_f32(x, y, p, sensor_size=(4, 6), interpolation="bilinear", exact=True)
    assert_within_exact(img, ex, q=Q22)
    lost = img.copy()
    lost[1, 3] -= np.float32(0.01 * 0.75 * 0.5)
    with pytest.raises(AssertionError):
        assert_within_exact(lost, ex, q=Q22)
    assert exact_error_bound(ex, Q22)[0, 0] > 0.01    # the hot cell's own bound hides such a tap, a cold cell's does not


# ---- RobustNorm order statistics and NaN handling against torch on CPU -------------------------------------------------
def reference_robust_norm(x, low_perc, top_perc):
    """data_augmentation.py:94-130 restated with the same torch calls (kthvalue, clamp, min, max)."""
    def pct(q):
        k = 1 + round(.01 * float(q) * (x.numel() - 1))
        return x.reshape(-1).kthvalue(k).values.item()
    t_max, t_min = pct(top_perc), pct(low_perc)
    if t_max == 0 and t_min == 0:
        return x, t_min, t_max
    normed = torch.clamp(x, min=t_min, max=t_max)
    return (normed - torch.min(normed)) / (torch.max(normed) + 1e-6), t_min, t_max


def robust_norm_cases():
    """(name, f32 array, [(low_perc, top_perc), ...])"""
    rng = np.random.default_rng(12)
    f = np.float32
    qs = [(0, 95), (0, 100), (100, 100), (0, 0), (10, 90), (50, 50), (90, 10)]
    sub = np.finfo(f).smallest_subnormal
    yield "all_equal", np.full(300, f(2.5)), qs
    yield "all_zero", np.zeros(257, f), qs
    ties = rng.choice(f([-1.0, 0.0, 3.0]), 1000).astype(f)
    yield "ties", ties, qs
    yield "signed_zeros", f([0.0, -0.0, 0.0, -0.0, 1.0, -1.0, -0.0]), qs
    yield "subnormals", (rng.integers(-20, 20, 513) * sub).astype(f), qs
    yield "infinities", f([np.inf, -np.inf, 1.0, 2.0, -3.0, np.inf, 0.5]), qs
    for n in (1, 2, 3, 255, 257, 1000):
        yield "random_%d" % n, rng.standard_normal(n).astype(f), qs
    # values that differ only in their last 10 bits: decided by the radix select's third pass
    base = np.full(700, f(1.75)).view(np.uint32) + rng.integers(0, 1024, 700).astype(np.uint32)
    yield "last_bits", base.view(f), qs
    neg_nan = np.array([0xffc00000], np.uint32).view(f)[0]
    pos_nan = np.float32(np.nan)
    yield "neg_nan_small", f([1.0, 2.0, -1.0, neg_nan]), qs
    for sign, nanv in (("neg", neg_nan), ("pos", pos_nan)):
        a = rng.standard_normal(301).astype(f)
        a[[7, 100]] = nanv
        yield "%s_nan_below_rank" % sign, a, [(0, 50), (0, 95), (10, 90)]
        yield "%s_nan_at_rank" % sign, a, [(0, 100), (0, 99.7), (100, 100)]
    z = np.zeros(200, f)
    z[5] = neg_nan
    yield "nan_identity", z, [(0, 95), (0, 100)]


def _kth(a, q):
    return 1 + round(.01 * float(q) * (a.size - 1))


def test_robust_norm_oracle_matches_torch_reference(oracle):
    for name, a, qs in robust_norm_cases():
        x = torch.from_numpy(a.copy())
        for lo, hi in qs:
            ref, t_min, t_max = reference_robust_norm(x, lo, hi)
            part = np.sort(a.astype(np.float64))                    # numpy sorts every NaN last, like kthvalue
            assert np.array_equal([part[_kth(a, lo) - 1], part[_kth(a, hi) - 1]], [t_min, t_max], equal_nan=True), name
            out = oracle.robust_norm_f32(a, low_perc=lo, top_perc=hi)
            assert np.array_equal(out, ref.numpy(), equal_nan=True), (name, lo, hi)


def test_kthvalue_ranks_every_nan_last():
    neg_nan = np.array([0xffc00000], np.uint32).view(np.float32)
    x = torch.from_numpy(np.concatenate([np.float32([1, 2, -1]), neg_nan]))
    assert x.kthvalue(1).values.item() == -1.0
    assert np.isnan(x.kthvalue(4).values.item())


# ---- exactly summable streams: the oracle's own f32 sums must equal the exact sums bit for bit ---------------------------
@pytest.mark.parametrize("kind", ["voxel", "trilinear", "nearest", "bilinear", "cmax"])
def test_exact_streams_are_exactly_summable(oracle, kind):
    """exact_streams(): the oracle's sequential f32 sums equal the f64 sums bit for bit, for the stream as generated,
    reversed and shuffled -- the streams are exactly summable in practice, not only by the argument of
    exact_bounds.assert_exactly_summable (which is checked as well)."""
    from edge_cases import exact_streams
    from exact_bounds import assert_exact, check_exactly_summable, exact_outputs, select_events
    for seed in (1, 2, 3):
        c = exact_streams(seed, "voxel" if kind == "trilinear" else kind, 200003)
        kws = [dict(bilinear=True, clip=False), dict(bilinear=True, clip=True)] if kind == "trilinear" else \
            [dict(clip=False, padding=False), dict(clip=True, padding=True)] if kind in ("nearest", "bilinear") else \
            [dict(), dict(abs_polarity=True)] if kind == "cmax" else [dict()]
        for kw in kws:
            outs = check_exactly_summable(oracle, c, **kw)
            n = c["hot"].shape[0]
            for order in (np.arange(n), np.arange(n)[::-1], np.random.default_rng(seed).permutation(n)):
                for pl in exact_outputs(oracle, select_events(c, order), **kw):
                    assert_exact(pl.out, pl.ex, what="%s %s seed %d" % (pl.name, kw, seed))
            if kind != "cmax" and not kw.get("clip"):
                assert all(pl.oob > 0 for pl in outs), "the stream has out-of-range events"
            assert max((pl.ex.abs > 2 ** 14).sum() for pl in outs) > 0, "no hot cell"


@pytest.mark.parametrize("kind", ["voxel", "nearest", "bilinear", "cmax"])
def test_exact_streams_wrap_every_table_slot(kind):
    """At the sizes of tests/test_gpu_exact_sums.py and the launch geometry of an H100 SXM (132 SMs), every CTA's hot
    table slot wraps upward and back downward (exact_bounds.assert_tables_wrap), so the carries of both signs run."""
    from edge_cases import EXACT_SIZES, exact_streams
    from exact_bounds import assert_tables_wrap
    assert_tables_wrap(exact_streams(7, kind, EXACT_SIZES[kind]), 132, what=kind)


def test_table_wraps_model():
    """The slot model of table_wraps on hand-counted runs (F = 22: the slot holds +-512, a wrap carries 1024)."""
    from exact_bounds import table_wraps
    for P, M, up, down in ((800, 200, 1, 0), (511, 1000, 0, 0), (512, 0, 1, 0), (600, 900, 1, 1), (1600, 400, 2, 1),
                           (0, 513, 0, 1)):
        v = np.concatenate([np.ones(P), -np.ones(M)])
        u, d, net = table_wraps(v, 22, 1, 1)
        assert (u[0], d[0], net[0]) == (up, down, up - down), (P, M)
