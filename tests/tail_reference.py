"""f64 reference of the contrast objectives' image-space tail (csrc/evk_cmax.cu) -- TEST INFRASTRUCTURE ONLY.

Every contrast objective ends in the same tail: G = a separable, reflect-mode Gaussian blur of the image (truncate 4),
f = a reduction of G and, for the gradient, a blur of a per-pixel weight image contracted with the derivative images.
Here the blur is scipy's (flow_objective_reference.blur_matrix, applied in f64) and every scalar comes with a bound
carried through its reduction from the per-cell bound of the kernel's blur:

    |G_kernel - blur64(I)| <= blur_bound(I) = 2^-23 (1 + 2^-20) blur64(|I|)

The kernel accumulates each axis in f64 and rounds it to f32 (axis 0, then axis 1): two f32 roundings of at most 2^-24
of a value no larger than blur64(|I|); the factor 1 + 2^-20 covers the f64 accumulation and second-order terms.  f64
sums of P terms add gamma64(P) of the sum of magnitudes.  No bound is a flat tolerance, so a wrong tap, reflection or
channel mix shows up as soon as it moves a value by more than the rounding the kernel is allowed.

The module also transcribes the kernel's blur rules (reflect_idx, make_taps, mix_coeffs) so that the CPU tests can tie
them to scipy, and emulates the kernel's f32 blur with a mutated rule to show that the bounds reject it."""
import numpy as np
import scipy.ndimage

from flow_objective_reference import blur_matrix

U32 = 2.0 ** -24
U64 = 2.0 ** -53
MAX_RADIUS = 64
FUSED_MAX_R = 8
f32 = np.float32


def gamma64(n):
    """n u / (1 - n u), u = 2^-53: the relative error of n f64 operations in any order"""
    mu = np.asarray(n, np.float64) * U64
    return mu / (1.0 - mu)


def radius(sigma):
    """the truncate-4 radius of make_taps (0 for sigma <= 0, no blur)"""
    return int(4.0 * sigma + 0.5) if sigma > 0 else 0


# ---- transcription of the kernel's rules -----------------------------------------------------------------------------
def reflect_idx(i, n, mode="reflect"):
    """reflect_idx of csrc/evk_cmax.cu (scipy's mode 'reflect', d c b a | a b c d | d c b a); 'mirror' and 'nearest'
    are the two wrong rules the sensitivity tests plant"""
    if n == 1:
        return 0
    if mode == "nearest":
        return min(max(i, 0), n - 1)
    period = 2 * n if mode == "reflect" else 2 * n - 2
    i %= period
    return i if i < n else (period - 1 - i if mode == "reflect" else period - i)


def taps(sigma, r=None):
    """make_taps: w[k], k = 0..r, exp(-k^2 / 2 sigma^2) normalised over [-r, r] (r defaults to the truncate-4 radius)"""
    r = radius(sigma) if r is None else r
    k = np.arange(-r, r + 1, dtype=np.float64)
    e = np.exp(-0.5 / (sigma * sigma) * k * k)
    return e[r:] / e.sum()


def mix_coeffs(w):
    """mix_coeffs: (a, b) of scipy's blur along the length-2 stack axis, from the reflected unit vector [1, 0]"""
    r = len(w) - 1
    a = b = 0.0
    for k in range(-r, r + 1):
        if k % 4 in (0, 3):
            a += w[abs(k)]
        else:
            b += w[abs(k)]
    return a, b


def kernel_blur_matrix(n, sigma, mode="reflect", dr=0, shift=0):
    """M with M @ a == the kernel's blur of a along one axis, built from the transcribed rules.  dr changes the radius
    (taps renormalised over [-(r + dr), r + dr]), shift moves every source index by that many pixels (a halo gathered one
    pixel off)."""
    if sigma <= 0:
        return np.eye(n)
    w = taps(sigma, radius(sigma) + dr)
    r = len(w) - 1
    M = np.zeros((n, n))
    for i in range(n):
        for k in range(-r, r + 1):
            M[i, reflect_idx(i + k + shift, n, mode)] += w[abs(k)]
    return M


def emulate_blur32(I, sigma, **mutation):
    """the kernel's two-pass f32 blur of a 2-D image with (possibly mutated) rules: each axis in f64, rounded to f32"""
    I = np.asarray(I, np.float64)
    My = kernel_blur_matrix(I.shape[0], sigma, **mutation)
    Mx = kernel_blur_matrix(I.shape[1], sigma, **mutation)
    T = (My @ I).astype(f32).astype(np.float64)
    return (T @ Mx.T).astype(f32)


# ---- f64 reference -----------------------------------------------------------------------------------------------------
def blur64(I, sigma):
    """scipy.ndimage.gaussian_filter(I, sigma) (mode reflect, truncate 4) of a 2-D image, in f64; sigma <= 0: I"""
    I = np.asarray(I, np.float64)
    return blur_matrix(I.shape[0], sigma) @ I @ blur_matrix(I.shape[1], sigma).T


def blur_bound(I, sigma):
    """per-cell bound of |kernel blur - blur64| (module docstring); 0 without a blur"""
    if sigma <= 0:
        return np.zeros(np.shape(I))
    return 2.0 ** -23 * (1.0 + 2.0 ** -20) * blur64(np.abs(np.asarray(I, np.float64)), sigma)


def mix64(sigma):
    """(a, b): scipy's blur of the 2-stack [1, 0] along its own axis -- how the reference's 3-D blur of the (2, H, W)
    derivative stack mixes its channels"""
    if sigma <= 0:
        return 1.0, 0.0
    a, b = scipy.ndimage.gaussian_filter1d(np.array([1.0, 0.0]), sigma, mode="reflect", truncate=4.0)
    return float(a), float(b)


def blur3d64(D, sigma):
    """the reference's literal G3d: scipy's 3-D blur of the (2, H, W) derivative stack"""
    D = np.asarray(D, np.float64)
    if sigma <= 0:
        return D.copy()
    return scipy.ndimage.gaussian_filter(D, sigma, mode="reflect", truncate=4.0)


def tail(I, D, sigma, name, param=0.0, mix=True):
    """The values of the legacy image-space tail and their bounds: {key: (value, bound)} with keys
    f, g0, g1 (mixed as the reference's G3d mixes them unless mix=False), u0, u1 (the un-mixed gradient), sumI,
    meanG, var, msq32 (mean of the f32 products G*G), msq64 (sum of the f64 products G*G / P), sosa (sum exp(-p G)),
    max, count (#(G > f32(param))).  I: (H, W) f32 image, D: (2, H, W) f32 derivative images or None.
    The gradient is the reference's form, -c sum(w * G3d(dIWE)_k); the kernel contracts the blurred w with dIWE instead,
    which is the same number because the reflect blur is self-adjoint."""
    I = np.asarray(I, np.float64)
    P = I.size
    r = radius(sigma)
    G = blur64(I, sigma)
    e = blur_bound(I, sigma)
    Ga = np.abs(G) + e                       # bound on |G_kernel|
    gP = gamma64(P + 8 * r + 16)            # f64 sums and blurs of the tail and of this reference
    out = {}
    out["sumI"] = (I.sum(), gP * np.abs(I).sum())
    E = e.sum() / P
    mG = G.mean()
    out["meanG"] = (mG, E + gP * Ga.sum() / P)
    var = ((G - mG) ** 2).mean()
    dvar = (2 * np.abs(G) * e + e * e).sum() / P + 2 * abs(mG) * E + E * E + 4 * gP * ((Ga * Ga).sum() / P + (abs(mG) + E) ** 2)
    out["var"] = (var, dvar)
    sq = (G * G).sum() / P
    dsq64 = (2 * np.abs(G) * e + e * e).sum() / P + gP * (Ga * Ga).sum() / P
    out["msq64"] = (sq, dsq64)
    out["msq32"] = (sq, dsq64 + U32 * (Ga * Ga).sum() / P)
    out["max"] = (G.max(), e.max())
    t32 = float(f32(param))
    flip = np.abs(G - t32) <= e
    out["count"] = (float((G > t32).sum()), float(flip.sum()))
    p = float(param)
    xs = np.exp(-p * G + abs(p) * e)         # bound on exp(-p G_kernel)
    out["sosa"] = (np.exp(-p * G).sum(), (xs * (abs(p) * e + 2 * U64)).sum() + gP * xs.sum())

    if name == "variance":
        f = (-var, dvar)
    elif name == "sos":
        f = (-sq, out["msq32"][1])
    elif name == "soe":
        xe = np.exp(G + e)
        f = (-np.exp(G).sum() / P, ((xe * (e + 2 * U64)).sum() + gP * xe.sum()) / P)
    elif name == "moa":
        f = (-G.max(), e.max())
    elif name == "isoa":
        f = out["count"]
    elif name == "sosa":
        f = (-out["sosa"][0], out["sosa"][1])
    else:
        raise ValueError(name)
    out["f"] = f

    # gradient: u_k = -c sum(w * G2(D_k)), w the objective's weight image, dw a per-cell bound of the kernel's w - w
    if D is None or name == "moa":
        for k in ("u0", "u1", "g0", "g1"):
            out[k] = (0.0, 0.0)
        return out
    D = np.asarray(D, np.float64)
    mu = I.mean()
    if name == "variance":
        w, dw, wa, c = 2 * (G - mu), 2 * e, 2 * (Ga + abs(mu)), 1.0 / P   # the kernel's form: 2 (G - mu) against dIWE
    elif name == "sos":
        w, dw, wa, c = 2 * I, np.zeros_like(I), 2 * np.abs(I), 1.0 / P
    elif name == "soe":
        xe = np.exp(G + e)
        w, dw, wa, c = np.exp(G), xe * (e + 2 * U64), xe, 1.0 / P
    elif name == "isoa":
        w, dw, wa, c = (G > t32).astype(np.float64), flip.astype(np.float64), np.ones_like(I), 1.0
    else:  # sosa: w = -p exp(f32(-p G))
        da = abs(p) * e + U32 * abs(p) * Ga + U64 * abs(p) * Ga
        xa = np.exp(-p * G + da)
        w, dw, wa, c = -p * np.exp(-p * G), abs(p) * xa * (da + 2 * U64), abs(p) * xa, 1.0
    # the variance's w multiplies the UN-blurred D in the kernel; in the reference's form (I - mu) multiplies G2(D)
    GD = np.stack([blur64(D[k], sigma) for k in range(2)])
    GDa = np.stack([blur64(np.abs(D[k]), sigma) for k in range(2)])
    G3 = blur3d64(D, sigma)
    a, b = mix64(sigma)
    if name == "variance":
        src, srcmix, mag = 2 * (I - mu), G3, [np.abs(D[k]) for k in range(2)]
    else:
        src, srcmix, mag = w, G3, list(GDa)
    u, du = [], []
    for k in range(2):
        u.append(-c * (src * GD[k]).sum())
        du.append(c * ((dw * mag[k]).sum() + gP * (wa * mag[k]).sum()))
    out["u0"], out["u1"] = (u[0], du[0]), (u[1], du[1])
    if mix:
        gm = [-c * (src * srcmix[k]).sum() for k in range(2)]
        dg = [a * du[0] + b * du[1], b * du[0] + a * du[1]]
        dg = [d + gP * (abs(gm[k]) + a * abs(u[0]) + b * abs(u[1])) for k, d in enumerate(dg)]
        out["g0"], out["g1"] = (gm[0], dg[0]), (gm[1], dg[1])
    else:
        out["g0"], out["g1"] = out["u0"], out["u1"]
    return out


# result layouts: index -> key of tail(); None = not compared
def legacy_layout(name, grad):
    """the 12 doubles of evk_iwe_objective_f32 / evk_cmax_linvel_objective_* (include/evk.h)"""
    lay = {0: "f", 3: "sumI", 5: "var" if name == "variance" else "meanG"}
    if grad:
        lay.update({1: "g0", 2: "g1", 6: "u0", 7: "u1"})
    if name != "variance":
        lay.update({8: "msq32", 10: "max"})
        if name == "sosa":
            lay[9] = "sosa"
        if name == "isoa":
            lay[11] = "count"
    return lay


def model_layout(name):
    """the 16 doubles of evk_cmax_warp_objective_* (f only)"""
    lay = {0: "f", 5: "sumI", 7: "meanG", 8: "msq32", 10: "max"}
    if name == "sosa":
        lay[9] = "sosa"
    if name == "isoa":
        lay[11] = "count"
    return lay


def violations(res, ref, layout, exact_zero=()):
    """[(index, key, got, want, bound)] of the entries of `res` outside their bound"""
    bad = []
    for i, key in layout.items():
        want, bound = ref[key]
        if not abs(res[i] - want) <= bound:
            bad.append((i, key, res[i], want, bound))
    for i in exact_zero:
        if res[i] != 0:
            bad.append((i, "zero", res[i], 0.0, 0.0))
    return bad


def batched_f(I, sigma, name, param=0.0):
    """(f, bound) of one sample of the batched losses (flow / motion contrast): f64 products throughout"""
    t = tail(I, None, sigma, "variance" if name == "variance" else ("sos" if name == "sos" else name), param)
    if name == "sos":
        return -t["msq64"][0], t["msq64"][1]
    return t["f"]


def timestamp_f(T, sigma):
    """(f, bound) of one sample of the flow-timestamp loss: sum over its two images of sum(G^2), f64 products"""
    f = b = 0.0
    for img in T:
        t = tail(img, None, sigma, "sos")
        P = np.asarray(img).size
        f += t["msq64"][0] * P
        b += t["msq64"][1] * P
    return f, b
