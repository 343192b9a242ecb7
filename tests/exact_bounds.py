"""Per-cell error bounds for kernels whose output cells are sums of f32 taps, against the oracle's exact mode
(oracle/evk_oracle.py, exact=True: per cell the f64 sum of the f32 taps, the f64 sum of |tap| and the tap count).
A kernel may add the taps of a cell in any order and grouping; the bound below holds for all of them, so it needs no
tuning, and a tap that is lost, doubled or sent to another cell shows up in the cell it belongs to whenever its weight
exceeds that cell's bound -- however hot the rest of the image is."""
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
