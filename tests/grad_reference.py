"""f64 references of the backward kernels of csrc/evk_grad.cu, in plain numpy -- TEST INFRASTRUCTURE ONLY.

Each function evaluates the kernel's own expression for every per-event output, term by term as evk_grad.cu writes
it, but in f64.  Every DISCRETE decision is taken from the forward's f32 arithmetic (floor, clip mask, trunc + wrap of
the index, |tn| < 1e9, the tie v == 0 and the sign of d of the voxel bins, the neg/pos split), so the taps are exactly
the kernel's taps; only the continuous part is computed in f64.

A value is carried as an `R`: v, the f64 value; M, the magnitude (the same expression with every term replaced by its
absolute value); m, the number of f32 roundings on the longest path of the kernel's expression, counted as
    a +- b: max(m_a, m_b) + 1   (M = |a +- b| when both are exact f32 inputs: one rounding of an exact value)
    a * b:  m_a + m_b + 1       a / d (d an exact f32 value): m_a + 1
    a * s, s in {0, +-1/2, +-1}: m_a (exact)
Then |kernel - v| <= gamma(m) M (Higham, Accuracy and Stability of Numerical Algorithms, 2nd ed., section 3.1 and
lemma 3.3), and v itself is within gamma64(m) M of the exact value; exact_bounds.assert_within_grad_bound checks the
sum of the two.  Each function states the m of its outputs next to the kernel expression and asserts it.

Where an output also takes other inputs that carry an error bound (the timestamp images' forward `out` and count
images, the f64 sums behind the end-stamp and t0 terms), that bound is carried through and returned as `extra`.
"""
import collections

import numpy as np

from exact_bounds import U32, exact_error_bound

F32 = np.float32
U64 = 2.0 ** -53
FLT_MAX = float(np.finfo(np.float32).max)

# one per-event output: f64 value v, magnitude M, roundings m, and an absolute error `extra` from inexact inputs
Grad = collections.namedtuple("Grad", "v M m extra")
Exact = collections.namedtuple("Exact", "sum abs cnt")


def gamma64(m):
    mu = np.asarray(m, np.float64) * U64
    return mu / (1.0 - mu)


def gamma32(m):
    mu = np.asarray(m, np.float64) * U32
    return mu / (1.0 - mu)


def bound_of(g):
    """|kernel - v| <= (gamma(m) + gamma64(m)) M + extra."""
    return (gamma32(g.m) + gamma64(g.m)) * g.M + g.extra


class R:
    __slots__ = ("v", "M", "m")

    def __init__(self, v, M, m):
        self.v, self.M, self.m = v, M, m


def ex(a):
    """An exact f32 input of the expression."""
    a = np.asarray(a, np.float64)
    return R(a, np.abs(a), np.zeros(a.shape, np.int64))


ZERO = ex(0.0)


def add(a, b):
    v = a.v + b.v
    both = (a.m == 0) & (b.m == 0)
    return R(v, np.where(both, np.abs(v), a.M + b.M), np.maximum(a.m, b.m) + 1)


def neg(a):
    return R(-a.v, a.M, a.m)


def sub(a, b):
    return add(a, neg(b))


def mul(a, b):
    return R(a.v * b.v, a.M * b.M, a.m + b.m + 1)


def scale(a, s):
    """a * s with s exact and the product exact (0, +-1/2, +-1)."""
    s = np.asarray(s, np.float64)
    return R(a.v * s, a.M * np.abs(s), a.m + np.zeros(s.shape, np.int64))


def div(a, d):
    d = np.asarray(d, np.float64)
    return R(a.v / d, a.M / np.abs(d), a.m + 1)


def rabs(a):
    return R(np.abs(a.v), a.M, a.m)


def pick(mask, a, b):
    return R(np.where(mask, a.v, b.v), np.where(mask, a.M, b.M), np.where(mask, a.m, b.m))


def acc(total, started, term, mask):
    """total += term where mask, as the kernel's running f32 sum that starts from 0 (its first add is exact)."""
    first = mask & ~started
    out = pick(mask & started, add(total, term), total)
    return pick(first, term, out), started | mask


def grad(r, extra=0.0, m_expect=None, valid=None):
    if m_expect is not None:
        sel = r.m if valid is None else r.m[valid]
        assert sel.size == 0 or sel.max() <= m_expect, (int(sel.max()), m_expect)
    return Grad(r.v, r.M, np.asarray(r.m), np.asarray(extra, np.float64) + np.zeros(np.shape(r.v)))


def _f32(*a):
    return tuple(np.asarray(v, np.float32).reshape(-1) for v in a)


def _trunc(v):
    """trunc_checked: |v| < 2e9, then truncation toward zero."""
    ok = np.abs(v) < F32(2.0e9)
    return ok, np.trunc(np.where(ok, v, 0)).astype(np.int64)


def _wrap(i, size):
    """wrap_int_index: [-size, -1] wraps once; valid iff the result is in [0, size)."""
    j = np.where(i < 0, i + size, i)
    return (j >= 0) & (j < size), np.clip(j, 0, size - 1)


# ---- event image: image_grad_event -----------------------------------------------------------------------------------
def image_grad(x, y, p, g, clip=False, clipx=0.0, clipy=0.0, bilinear=True):
    """{gx, gy, gp} of evk_image_grad_f32; nearest: {gp} only (the coordinates get nothing).
      nearest   gp = G[yi, xi]                                          m = 0 (exact)
      bilinear  gp = m * (ox*oy*g00 + dx*oy*g01 + ox*dy*g10 + dx*dy*g11)  m = 9
                gx = w * (oy*(g01 - g00) + dy*(g11 - g10))               m = 6  (likewise gy)
                with dx = x - floor(x) (1), ox = 1 - dx (2), w = p*m exact."""
    x, y, p = _f32(x, y, p)
    g = np.asarray(g, np.float32)
    H, W = g.shape
    with np.errstate(all="ignore"):
        if not bilinear:
            keep = ~np.bool_(clip) | (~(x >= F32(clipx)) & ~(y >= F32(clipy)))
            okx, ux = _trunc(x)
            oky, uy = _trunc(y)
            ux, uy = np.where(keep, ux, 0), np.where(keep, uy, 0)
            okw, xi = _wrap(ux, W)
            okh, yi = _wrap(uy, H)
            ok = okx & oky & okw & okh
            return dict(gp=grad(pick(ok, ex(g[yi, xi]), ZERO), m_expect=0))
        m = np.ones_like(x)
        if clip:
            m = np.where(x >= F32(clipx), F32(0), F32(1)) * np.where(y >= F32(clipy), F32(0), F32(1))
        pxf, pyf = np.floor(x), np.floor(y)
        okx, upx = _trunc(pxf * m)
        oky, upy = _trunc(pyf * m)
        v0, x0 = _wrap(upx, W)
        v1, x1 = _wrap(upx + 1, W)
        v2, y0 = _wrap(upy, H)
        v3, y1 = _wrap(upy + 1, H)
        ok = okx & oky & v0 & v1 & v2 & v3
        dx, dy = sub(ex(x), ex(pxf)), sub(ex(y), ex(pyf))
        ox, oy = sub(ex(1.0), dx), sub(ex(1.0), dy)
        g00, g01, g10, g11 = ex(g[y0, x0]), ex(g[y0, x1]), ex(g[y1, x0]), ex(g[y1, x1])
        w = ex(p * m)
        gp = scale(add(add(add(mul(mul(ox, oy), g00), mul(mul(dx, oy), g01)), mul(mul(ox, dy), g10)),
                       mul(mul(dx, dy), g11)), m)
        gx = mul(w, add(mul(oy, sub(g01, g00)), mul(dy, sub(g11, g10))))
        gy = mul(w, add(mul(ox, sub(g10, g00)), mul(dx, sub(g11, g01))))
        return dict(gx=grad(pick(ok, gx, ZERO), m_expect=6), gy=grad(pick(ok, gy, ZERO), m_expect=6),
                    gp=grad(pick(ok, gp, ZERO), m_expect=9))


# ---- timestamp images: tsimg_grad_prep_kernel + tsimg_grad_kernel + autograd.py's end terms ---------------------------
def ts_denom(t_first, t_last):
    """The forward's f32 denominator (t_last - t_first) + 1e-6."""
    return F32(F32(F32(t_last) - F32(t_first)) + F32(1e-6))


def _ts_geometry(x, y, t, p, t_first, t_last, H, W, clip, clipx, clipy, reverse):
    m = np.ones_like(x)
    if clip:
        m = np.where(x >= F32(clipx), F32(0), F32(1)) * np.where(y >= F32(clipy), F32(0), F32(1))
    pxf, pyf = np.floor(x), np.floor(y)
    okx, upx = _trunc(pxf * m)
    oky, upy = _trunc(pyf * m)
    v0, x0 = _wrap(upx, W)
    v1, x1 = _wrap(upx + 1, W)
    v2, y0 = _wrap(upy, H)
    v3, y1 = _wrap(upy + 1, H)
    pos, negm = p > 0, p <= 0
    ok = okx & oky & v0 & v1 & v2 & v3 & (pos | negm)
    D = ts_denom(t_first, t_last)
    tn32 = (F32(t_last) - t if reverse else t - F32(t_first)) / D
    return ok, negm, (x0, x1, y0, y1), pxf, pyf, D, tn32


def tsimg_forward_exact(x, y, t, p, t_first, t_last, H, W, clip=False, clipx=0.0, clipy=0.0, reverse=False):
    """Per cell the f64 sum, |sum| and count of the f32 taps of tsimg_scatter_kernel, planes [Tpos, Cpos, Tneg, Cneg]
    (the count images without their initial one), as the oracle's exact mode gives them."""
    x, y, t, p = _f32(x, y, t, p)
    with np.errstate(all="ignore"):
        ok, negm, (x0, x1, y0, y1), pxf, pyf, _, tn = _ts_geometry(x, y, t, p, t_first, t_last, H, W, clip, clipx,
                                                                    clipy, reverse)
        dx, dy = x - pxf, y - pyf
        ox, oy = F32(1) - dx, F32(1) - dy
        tl, tr = tn * ox, tn * dx
        tt = (tl * oy, tr * oy, tl * dy, tr * dy)
        cc = (ox * oy, dx * oy, ox * dy, dx * dy)
    S, A, K = (np.zeros((4, H, W)) for _ in range(3))
    plane = np.where(negm, 2, 0)[ok]
    for k, (yy, xx) in enumerate(((y0, x0), (y0, x1), (y1, x0), (y1, x1))):
        for off, vals in ((0, tt[k]), (1, cc[k])):
            v = vals[ok].astype(np.float64)
            idx = (plane + off, yy[ok], xx[ok])
            np.add.at(S, idx, v)
            np.add.at(A, idx, np.abs(v))
            np.add.at(K, idx, 1.0)
    return Exact(S, A, K)


def ratio_bound(num, den, den_offset=1.0):
    """T / C and the bound on |fl(T'/C') - T/C| of assert_ratio_within_exact (T, C: Exact sums, C from den_offset)."""
    T, C = num.sum, den.sum + den_offset
    eT = exact_error_bound(num)
    eC = exact_error_bound(den, 0.0, den_offset)
    Cm = C - eC
    assert (Cm > 0).all(), "count image too close to zero for the bound"
    return T / C, C, eC, (eT * C + np.abs(T) * eC) / (C * Cm) + U32 * (np.abs(T) + eT) / Cm


def tsimg_grad(x, y, t, p, t_first, t_last, g_pos, g_neg, clip=False, clipx=0.0, clipy=0.0, reverse=False, reps=1):
    """{gx, gy, gt} of evk_timestamp_image_grad_f32 (gt WITHOUT autograd.py's ts[0] / ts[-1] terms) and the kernel's two
    f64 sums {s0: sum g_tn, s1: sum g_tn * tn} as (value, bound).  Per pixel the kernel reads a = G/C and b = a*out
    (tsimg_grad_prep_kernel) with its forward's f32 out and C; their error from the exact T/C and C is carried through
    (ratio_bound) into `extra`.
      tn = (t - t_first) / D  (reverse: (t_last - t) / D)          m = 2
      e  = tn*a - b                                               m = 4
      gx = oy*(e01 - e00) + dy*(e11 - e10)                        m = 9   (likewise gy)
      gtn = ox*oy*a00 + dx*oy*a01 + ox*dy*a10 + dx*dy*a11         m = 9
      gt = gtn * tscale, tscale = fl(+-1 / D)                     m = 11
    reps: the kernel ran on these events tiled `reps` times (the per-event values are those of one copy)."""
    x, y, t, p = _f32(x, y, t, p)
    G = np.stack([np.asarray(g_pos, np.float32), np.asarray(g_neg, np.float32)]).astype(np.float64)
    H, W = G.shape[1:]
    ex4 = Exact(*(a * reps for a in tsimg_forward_exact(x, y, t, p, t_first, t_last, H, W, clip, clipx, clipy, reverse)))
    a, da, b, db = (np.zeros((2, H, W)) for _ in range(4))
    for s in range(2):
        num, den = (Exact(*(arr[2 * s + k] for arr in ex4)) for k in (0, 1))
        o, C, eC, eo = ratio_bound(num, den)
        Gs = G[s]
        a[s] = Gs / C
        da[s] = np.abs(Gs) * (eC / C + U32) / (C - eC)
        Aa = np.abs(Gs) * (1 + U32) / (C - eC)
        b[s] = a[s] * o
        db[s] = Aa * eo + np.abs(o) * da[s] + U32 * Aa * (np.abs(o) + eo)
    with np.errstate(all="ignore"):
        ok, negm, (x0, x1, y0, y1), pxf, pyf, D, _ = _ts_geometry(x, y, t, p, t_first, t_last, H, W, clip, clipx,
                                                                   clipy, reverse)
        s = np.where(negm, 1, 0)
        taps = [(s, y0, x0), (s, y0, x1), (s, y1, x0), (s, y1, x1)]
        tn = div(sub(ex(t_last), ex(t)) if reverse else sub(ex(t), ex(t_first)), D)
        dx, dy = sub(ex(x), ex(pxf)), sub(ex(y), ex(pyf))
        ox, oy = sub(ex(1.0), dx), sub(ex(1.0), dy)
        A = [ex(a[i]) for i in taps]
        e = [sub(mul(tn, A[k]), ex(b[i])) for k, i in enumerate(taps)]
        # |tn (a' - a) - (b' - b)| per tap: the error the inexact a, b bring into e
        de = [np.abs(tn.v) * da[i] + db[i] for i in taps]
        dA = [da[i] for i in taps]
        gx = add(mul(oy, sub(e[1], e[0])), mul(dy, sub(e[3], e[2])))
        gy = add(mul(ox, sub(e[2], e[0])), mul(dx, sub(e[3], e[1])))
        w = [mul(ox, oy), mul(dx, oy), mul(ox, dy), mul(dx, dy)]
        gtn = add(add(add(mul(w[0], A[0]), mul(w[1], A[1])), mul(w[2], A[2])), mul(w[3], A[3]))
        tscale = R(np.float64((-1.0 if reverse else 1.0) / np.float64(D)), np.float64(1.0 / np.float64(D)), 1)
        gt = mul(gtn, tscale)
        xg = (1 + gamma32(gx.m)) * (oy.M * (de[1] + de[0]) + dy.M * (de[3] + de[2]))
        xy = (1 + gamma32(gy.m)) * (ox.M * (de[2] + de[0]) + dx.M * (de[3] + de[1]))
        xt = (1 + gamma32(gtn.m)) * sum(wk.M * d for wk, d in zip(w, dA))
        out = dict(gx=grad(pick(ok, gx, ZERO), np.where(ok, xg, 0), 9), gy=grad(pick(ok, gy, ZERO), np.where(ok, xy, 0), 9),
                   gtn=grad(pick(ok, gtn, ZERO), np.where(ok, xt, 0), 9),
                   gt=grad(pick(ok, gt, ZERO), np.where(ok, xt / np.float64(D), 0), 11))
        bt = bound_of(out["gtn"])
        etn = (gamma32(2) + gamma64(2)) * np.abs(tn.v)
        G_, T_ = out["gtn"].v, np.where(ok, tn.v, 0.0)
        n = x.shape[0] * reps
        s0 = (reps * G_.sum(), reps * (bt.sum() + 2 * gamma64(n) * np.abs(G_).sum()))
        s1 = (reps * (G_ * T_).sum(),
              reps * ((bt * (np.abs(T_) + etn) + np.abs(G_) * etn).sum() + 2 * gamma64(n) * np.abs(G_ * T_).sum()))
    out["s0"], out["s1"] = s0, s1
    out["D"] = D
    return out


def tsimg_grad_t(r, reverse=False):
    """autograd.py's ts gradient: the kernel's gt plus, on ts[0] and ts[-1], the f64 terms of D = ts[-1] - ts[0] + 1e-6
    (forward: (s1 - s0) / D, -s1 / D; reverse: s1 / D, (s0 - s1) / D), each cast to f32 and added in f32."""
    (s0, e0), (s1, e1), D = r["s0"], r["s1"], np.float64(r["D"])
    e64 = 2 * gamma64(2) * (abs(s0) + abs(s1)) / D          # the f64 subtraction and division
    if reverse:
        terms = [(0, s1 / D, e1 / D + e64), (-1, (s0 - s1) / D, (e0 + e1) / D + e64)]
    else:
        terms = [(0, (s1 - s0) / D, (e0 + e1) / D + e64), (-1, -s1 / D, e1 / D + e64)]
    return add_terms(r["gt"], terms)


def add_terms(g, terms):
    """g with f32 additions of f64 terms (index, value, bound of the f64 value) applied in order: each term is cast to f32
    (one rounding) and added in f32 (one more)."""
    v, b = g.v.copy(), bound_of(g).copy()
    for i, T, e in terms:
        v[i] += T
        b[i] += e + U32 * (abs(T) + e)
        b[i] += U32 * (abs(v[i]) + b[i])
    return Grad(v, g.M, g.m, b - (gamma32(g.m) + gamma64(g.m)) * g.M)


# ---- dense-flow warp: flow_grad_one ------------------------------------------------------------------------------------
def _warp_geometry(x, y, H, W):
    wm1, hm1 = F32(W - 1), F32(H - 1)
    ix32 = ((x / wm1) * F32(2) - F32(1) + F32(1)) / F32(2) * wm1
    iy32 = ((y / hm1) * F32(2) - F32(1) + F32(1)) / F32(2) * hm1
    ok = (np.abs(ix32) < F32(1e9)) & (np.abs(iy32) < F32(1e9))
    return ok, np.floor(np.where(ok, ix32, 0)), np.floor(np.where(ok, iy32, 0)), ix32, iy32


def _sample_pos(c, size):
    """ix = ((c / (S-1) * 2 - 1) + 1) / 2 * (S-1): the normalise round trip, = c exactly (m = 4, M = |c| + S-1)."""
    s1 = F32(size - 1)
    return mul(scale(add(sub(scale(div(ex(c), s1), 2.0), ex(1.0)), ex(1.0)), 0.5), ex(s1))


def warp_grad(x, y, t, flow, gxw, gyw, t0=0.0):
    """{gx, gy, gt} of evk_warp_flow_grad_f32 and {sum_gt: (value, bound)} of its f64 sum.
      ix (the normalise round trip of x)                        m = 4
      wx1 = (fx + 1) - ix, wx0 = ix - fx                          m = 5;  nw = wx1*wy1  m = 11
      u = top.x*nw + top.z*ne + bot.x*sw + bot.z*se               m = 15  (likewise v)
      gu = g_x * (t - t0)                                         m = 2
      c00 = gu*top.x + gv*top.y                                   m = 4
      gx = g_x + wy1*(c01 - c00) + wy0*(c11 - c10)                m = 13  (likewise gy)
      gt = g_x*u + g_y*v                                          m = 17"""
    x, y, t, gxw, gyw = _f32(x, y, t, gxw, gyw)
    flow = np.asarray(flow, np.float32)
    H, W = flow.shape[1:]
    with np.errstate(all="ignore"):
        ok, fx, fy, _, _ = _warp_geometry(x, y, H, W)
        x0, y0 = fx.astype(np.int64), fy.astype(np.int64)
        ix, iy = _sample_pos(x, W), _sample_pos(y, H)
        wx1, wx0 = sub(ex(fx + F32(1)), ix), sub(ix, ex(fx))
        wy1, wy0 = sub(ex(fy + F32(1)), iy), sub(iy, ex(fy))
        nw, ne, sw, se = mul(wx1, wy1), mul(wx0, wy1), mul(wx1, wy0), mul(wx0, wy0)

        def tap(c, yy, xx):
            inside = (xx >= 0) & (xx < W) & (yy >= 0) & (yy < H) & ok
            return ex(np.where(inside, flow[c, np.clip(yy, 0, H - 1), np.clip(xx, 0, W - 1)], 0))
        fu = [tap(0, y0, x0), tap(0, y0, x0 + 1), tap(0, y0 + 1, x0), tap(0, y0 + 1, x0 + 1)]
        fv = [tap(1, y0, x0), tap(1, y0, x0 + 1), tap(1, y0 + 1, x0), tap(1, y0 + 1, x0 + 1)]
        u = add(add(add(mul(fu[0], nw), mul(fu[1], ne)), mul(fu[2], sw)), mul(fu[3], se))
        v = add(add(add(mul(fv[0], nw), mul(fv[1], ne)), mul(fv[2], sw)), mul(fv[3], se))
        d = sub(ex(t), ex(t0))
        GX, GY = ex(gxw), ex(gyw)
        gu, gv = mul(GX, d), mul(GY, d)
        c = [add(mul(gu, fu[k]), mul(gv, fv[k])) for k in range(4)]
        gix = add(mul(wy1, sub(c[1], c[0])), mul(wy0, sub(c[3], c[2])))
        giy = add(mul(wx1, sub(c[2], c[0])), mul(wx0, sub(c[3], c[1])))
        gx = add(GX, pick(ok, gix, ZERO))
        gy = add(GY, pick(ok, giy, ZERO))
        gt = pick(ok, add(mul(GX, u), mul(GY, v)), ZERO)
        out = dict(gx=grad(gx, m_expect=13), gy=grad(gy, m_expect=13), gt=grad(gt, m_expect=17))
        n = x.shape[0]
        out["sum_gt"] = (gt.v.sum(), bound_of(out["gt"]).sum() + 2 * gamma64(n) * np.abs(gt.v).sum())
    return out


def flow_grad_exact(x, y, t_rel, gxw, gyw, H, W):
    """Per cell of the flow gradient: the f64 sum, |sum| and count of the f32 taps g*dt*w the kernel adds (the sample
    position and weights as flow_one forms them, in f32)."""
    x, y, t_rel, gxw, gyw = _f32(x, y, t_rel, gxw, gyw)
    with np.errstate(all="ignore"):
        ok, fx, fy, ix, iy = _warp_geometry(x, y, H, W)
        wx1, wx0, wy1, wy0 = (fx + F32(1)) - ix, ix - fx, (fy + F32(1)) - iy, iy - fy
        taps = [(0, 0, wx1 * wy1), (0, 1, wx0 * wy1), (1, 0, wx1 * wy0), (1, 1, wx0 * wy0)]
        S, A, K = (np.zeros((2, H, W)) for _ in range(3))
        for c, g in enumerate((gxw * t_rel, gyw * t_rel)):
            for oy, ox, w in taps:
                v = (g * w).astype(np.float32)
                xx, yy = fx.astype(np.int64) + ox, fy.astype(np.int64) + oy
                m = ok & (xx >= 0) & (xx < W) & (yy >= 0) & (yy < H) & (v != 0)
                np.add.at(S[c], (yy[m], xx[m]), v[m].astype(np.float64))
                np.add.at(A[c], (yy[m], xx[m]), np.abs(v[m]).astype(np.float64))
                np.add.at(K[c], (yy[m], xx[m]), 1.0)
    return Exact(S, A, K)


# ---- voxel grid: voxel_grad_event + voxel_grad_ends_kernel -------------------------------------------------------------
def _wrap_trunc(v, size):
    ok = np.abs(v) < F32(2.0e9)
    i = np.trunc(np.where(ok, v, 0)).astype(np.int64)
    i = np.where(i < 0, i + size, i)
    ok &= (i >= 0) & (i < size)
    return ok, np.clip(i, 0, size - 1)


def _bin(tn, tn32, b, g, p):
    """voxel_bin_grad: the terms g*bw (of gp) and -gv*sign(d) (of G) of bin b (an int array)."""
    d32 = tn32 - b.astype(np.float32)
    v32 = F32(1) - np.abs(d32)
    d = sub(tn, ex(b.astype(np.float64)))
    v = sub(ex(1.0), rabs(d))
    bw = pick(np.isnan(v32) | (v32 > 0), v, ZERO)
    gv = mul(ex(g), ex(p))
    gv = pick(v32 == 0, scale(gv, 0.5), gv)
    gv = pick(v32 < 0, ZERO, gv)
    sg = np.where(d32 > 0, 1.0, np.where(d32 < 0, -1.0, 0.0))
    return mul(ex(g), bw), scale(gv, -sg)


def _voxel_window(x, y, t, p, t0, dt, B, gw, negpos):
    """Per event of one window: (gp, G = dL/dtn, tn) as R.  gw: the window's incoming gradient [grids][B][H][W].
      tn = ((t - t0) / dt) * (B-1)                                  m = 3
      per bin: d = tn - b (4), v = 1 - |d| (5), g*bw (6), -g*p*sign(d) (1)
      G, gp: running sums over the bins visited (see voxel_grad)"""
    n = x.shape[0]
    H, W = gw.shape[2:]
    bm1 = F32(B - 1)
    tn32 = ((t - F32(t0)) / F32(dt)) * bm1
    tn = mul(div(sub(ex(t), ex(t0)), dt), ex(bm1))
    okx, xi = _wrap_trunc(x, W)
    oky, yi = _wrap_trunc(y, H)
    pix = okx & oky
    tfin = np.abs(tn32) < F32(1e9)
    zero_m = np.zeros(n, bool)
    f = np.floor(np.where(tfin, tn32, 0)).astype(np.int64)
    lo, hi = np.maximum(f - 1, 0), np.minimum(f + 2, B - 1)

    def row(grid, b):
        return gw[grid, np.clip(b, 0, B - 1), yi, xi]

    def run(seq):
        gp, G = ZERO, ZERO
        sp, sg = zero_m, zero_m
        for mask, grid, b, pv in seq:
            tp, tg = _bin(tn, tn32, b, row(grid, b), pv)
            gp, sp = acc(gp, sp, tp, mask)
            G, sg = acc(G, sg, tg, mask)
        return gp, G
    near_bins = lambda near, grid, pv: [(near & (f + k >= lo) & (f + k <= hi), grid, f + k, pv) for k in (-1, 0, 1, 2)]
    all_bins = lambda mask, grid, pv: [(mask, grid, np.full(n, b), pv) for b in range(B)]
    if negpos:
        wpos, wneg = np.where(p > 0, F32(1), F32(0)), np.where(p <= 0, F32(1), F32(0))
        near = pix & tfin & ((wpos != 0) | (wneg != 0))
        grid = np.where(wneg != 0, 1, 0)
        _, Gn = run(near_bins(near, grid, np.ones_like(p)))
        allp = pix & ~tfin
        _, Ga = run(all_bins(allp, np.zeros(n, np.int64), wpos))
        _, Gb = run(all_bins(allp, np.ones(n, np.int64), wneg))
        G = pick(allp, add(Ga, Gb), pick(near, Gn, ZERO))
        return None, G, tn
    near = pix & tfin & (np.abs(p) <= FLT_MAX)
    allp = pix & ~near
    z = np.zeros(n, np.int64)
    gp1, G1 = run(near_bins(near, z, p))
    gp2, G2 = run(all_bins(allp, z, p))
    return pick(allp, gp2, pick(near, gp1, ZERO)), pick(allp, G2, pick(near, G1, ZERO)), tn


def voxel_grad(x, y, t, p, B, g, pairs=None, negpos=False, want_gt=True):
    """{gp, gt} of evk_voxel_grad_f32 (gp None for neg/pos), the end-stamp terms included in gt, and {sums}: per window
    ((sum G, bound), (sum G tn, bound)).  g: incoming gradient [nw][grids][B][H][W]; pairs: [nw][2] (start, end) or None
    (one window [0, n)).  Each window's first stamp gets (S1 - (B-1) S0) / dt and its last -S1 / dt (f64, cast to f32,
    added in f32); an event in several windows (EVK_WINDOW_OVERLAP) gets each window's f32 value added in f32.
      per bin: g*bw m = 6, -g*p*sign(d) m = 1; the running sums add one rounding per bin after the first:
      G   m <= 4 (bins floor(tn)-1 .. floor(tn)+2), B (every bin, non-finite tn or p), B + 1 (neg/pos, non-finite tn)
      gp  m <= 9, 5 + B
      gt = (G * (B-1)) / dt                                           m <= m(G) + 2"""
    x, y, t, p = _f32(x, y, t, p)
    n = x.shape[0]
    g = np.asarray(g, np.float32)
    if pairs is None:
        pairs = np.array([[0, n]], np.int64)
    pairs = np.asarray(pairs, np.int64).reshape(-1, 2)
    bm1 = np.float64(B - 1)
    # per event: sum of values, magnitudes, max m, and the contributions' sum |v| + bound and count (f32 additions)
    acc_ = {k: dict(v=np.zeros(n), M=np.zeros(n), m=np.zeros(n, np.int64), absb=np.zeros(n), K=np.zeros(n, np.int64),
                    extra=np.zeros(n)) for k in ("gp", "gt")}

    def contribute(k, idx, v, M=0.0, m=0, extra=0.0):
        a = acc_[k]
        b = (gamma32(m) + gamma64(m)) * M + extra
        np.add.at(a["v"], idx, v)
        np.add.at(a["M"], idx, M)
        np.maximum.at(a["m"], idx, np.asarray(m, np.int64) + np.zeros(np.shape(idx), np.int64))
        np.add.at(a["extra"], idx, extra)
        np.add.at(a["absb"], idx, np.abs(v) + b)
        np.add.at(a["K"], idx, 1)
    sums = []
    with np.errstate(all="ignore"):
        for w, (first, last) in enumerate(pairs):
            if last <= first:
                sums.append(((0.0, 0.0), (0.0, 0.0)))
                continue
            sl = slice(first, last)
            t0, dt = t[first], F32(t[last - 1] - t[first])
            gp, G, tn = _voxel_window(x[sl], y[sl], t[sl], p[sl], t0, dt, B, g[w], negpos)
            idx = np.arange(first, last)
            if gp is not None:
                contribute("gp", idx, gp.v, gp.M, gp.m)
            gt = div(mul(G, ex(bm1)), dt)
            assert G.m.max(initial=0) <= max(4, B + 1) and gt.m.max(initial=0) <= max(4, B + 1) + 2
            if gp is not None:
                assert gp.m.max(initial=0) <= max(9, 5 + B)
            contribute("gt", idx, gt.v, gt.M, gt.m)
            bG = (gamma32(G.m) + gamma64(G.m)) * G.M
            btn = (gamma32(tn.m) + gamma64(tn.m)) * tn.M
            k = last - first
            S0 = (G.v.sum(), bG.sum() + 2 * gamma64(k) * np.abs(G.v).sum())
            S1 = ((G.v * tn.v).sum(), (bG * (np.abs(tn.v) + btn) + np.abs(G.v) * btn).sum()
                  + 2 * gamma64(k) * np.abs(G.v * tn.v).sum())
            sums.append((S0, S1))
            if want_gt:
                adt = abs(np.float64(dt))
                T0 = (S1[0] - bm1 * S0[0]) / np.float64(dt)
                e0 = (S1[1] + bm1 * S0[1]) / adt + 4 * gamma64(3) * (abs(S1[0]) + bm1 * abs(S0[0])) / adt
                T1 = -S1[0] / np.float64(dt)
                e1 = S1[1] / adt + 4 * gamma64(1) * abs(S1[0]) / adt
                for i, T, e in ((first, T0, e0), (last - 1, T1, e1)):
                    contribute("gt", np.array([i]), np.array([T]), extra=np.array([e + U32 * (abs(T) + e)]))
        out = {}
        for k in ("gp", "gt"):
            if k == "gp" and negpos:
                out[k] = None
                continue
            a = acc_[k]
            adds = np.maximum(a["K"] - 1, 0)
            out[k] = Grad(a["v"], a["M"], a["m"], a["extra"] + gamma32(adds) * a["absb"])
    out["sums"] = sums
    return out


# ---- the public torch functions: their options mapped to the kernel's arguments ----------------------------------------
def image_canvas(sensor_size, interpolation, padding):
    """events_to_image_torch's canvas and clip thresholds (image.py:64-74)."""
    if interpolation == 'bilinear' and padding:
        H, W = sensor_size[0] + 1, sensor_size[1] + 1
    else:
        H, W = sensor_size
    clipx = W if interpolation is None and padding is False else W - 1
    clipy = H if interpolation is None and padding is False else H - 1
    return int(H), int(W), float(clipx), float(clipy)


def public_grads(kind, a, weights, opts=None, B=None, negpos=False):
    """The f64 reference of the gradients that autograd gives each differentiable input of one public function, for
    the loss sum(out_k * weights_k).  kind: "image" (events_to_image_torch), "tsimg" (events_to_timestamp_image_torch),
    "warp" (warp_events_flow_torch; a["t0"] optional, else ts[-1]) or "voxel" (events_to_voxel_torch /
    events_to_neg_pos_voxel_torch).  a: numpy inputs.  Returns {input name: Grad} (the flow: an Exact of its cells)."""
    opts = opts or {}
    x, y = (np.asarray(a[k], np.float32).reshape(-1) for k in ("xs", "ys"))
    if kind == "image":
        interp, padding = opts.get("interpolation"), opts.get("padding", True)
        H, W, cx, cy = image_canvas(opts.get("sensor_size", (180, 240)), interp, padding)
        r = image_grad(x, y, a["ps"], weights[0], opts.get("clip_out_of_range", True), cx, cy, interp == 'bilinear')
        return {"xs": r.get("gx"), "ys": r.get("gy"), "ps": r["gp"]}
    if kind == "tsimg":
        sensor, padding = opts.get("sensor_size", (180, 240)), opts.get("padding", True)
        H, W = (sensor[0] + 1, sensor[1] + 1) if padding else tuple(sensor)
        cx, cy = (float(W - 1), float(H - 1)) if opts.get("interpolation", 'bilinear') is not None or padding else (W, H)
        t = np.asarray(a["ts"], np.float32).reshape(-1)
        rev = opts.get("timestamp_reverse", False)
        r = tsimg_grad(x, y, t, a["ps"], t[0], t[-1], weights[0], weights[1], opts.get("clip_out_of_range", True),
                       cx, cy, rev)
        return {"xs": r["gx"], "ys": r["gy"], "ts": tsimg_grad_t(r, rev)}
    if kind == "warp":
        t = np.asarray(a["ts"], np.float32).reshape(-1)
        has_t0 = a.get("t0") is not None
        t0 = F32(a["t0"]) if has_t0 else t[-1]
        r = warp_grad(x, y, t, a["flow"], weights[0], weights[1], t0)
        S, E = r["sum_gt"]
        tr = (t - t0).astype(np.float32)
        out = {"xs": r["gx"], "ys": r["gy"], "flow": flow_grad_exact(x, y, tr, weights[0], weights[1], *np.shape(a["flow"])[1:])}
        if has_t0:
            out["ts"] = r["gt"]
            out["t0"] = Grad(np.array([-S]), np.zeros(1), np.zeros(1, np.int64), np.array([E + U32 * (abs(S) + E)]))
        else:
            out["ts"] = add_terms(r["gt"], [(-1, -S, E)])
        return out
    assert kind == "voxel"
    g = np.stack([np.asarray(w, np.float32) for w in weights])[None]
    r = voxel_grad(x, y, a["ts"], a["ps"], B, g, negpos=negpos)
    return {"ts": r["gt"], "ps": r["gp"]}
