/*
 * evk_oracle.c -- CPU restatement of the event_utils hot path.  TEST INFRASTRUCTURE ONLY.
 *
 * This file is the parity oracle for the CUDA kernels in event_utils_b200/csrc.  It is never
 * part of the product path: only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
 * --impl reference legs may load it.  It is a plain, sequential, single-threaded restatement
 * of what the reference computes (which in the reference is spread over numpy / torch / scipy
 * library calls), with every rounding point of the reference kept (f32 vs f64, no FMA
 * contraction: build with -ffp-contract=off).
 *
 * Parity pin: tests/golden/ holds vectors generated from the real reference by
 * tests/golden/make_golden.py and make_golden_random.py; tests/test_oracle_golden.py and
 * tests/test_oracle_vs_reference.py compare this file against them.
 *
 * Reference citations (paths relative to the reference tree):
 *   voxel (torch, f32)      lib/representations/voxel_grid.py:129-153
 *   voxel (numpy, f64)      lib/representations/voxel_grid.py:198-217 + image.py:17,29-44
 *   image nearest/bilinear  lib/representations/image.py:62-100, 102-115
 *   derivative image        lib/representations/image.py:117-136, 179-217
 *   linear-velocity warp    lib/contrast_max/warps.py:51-61
 *   bounds mask             lib/util/event_util.py:26-27
 *   get_iwe                 lib/contrast_max/objectives.py:184-192
 *   variance objective      lib/contrast_max/objectives.py:231-236, 251-264
 *   dense-flow warp         lib/transforms/optic_flow.py:23-46 (+ torch grid_sample, bilinear,
 *                           align_corners=True, zero padding)
 *   gaussian_filter         scipy.ndimage (truncate=4, mode='reflect', axis 0 first, f64
 *                           line accumulation, result rounded to the f32 array after each axis)
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define EVO_API __attribute__((visibility("default")))

/* torch ``Tensor.long()`` on a float: C cast toward zero (NaN/inf -> INT64_MIN on x86) */
static inline int64_t trunc_to_long(float v)
{
    if (!(v == v) || v >= 9.2e18f || v <= -9.2e18f) return INT64_MIN;
    return (int64_t)v;
}

/* ------------------------------------------------------------------------------------------
 * Exact mode.  Every scatter function below sends each of its taps through add_tap(); with a
 * non-NULL `ex` (3 * cells doubles, cells = the size of all its output planes together) the tap
 * is also accumulated into ex[0*cells + j] (f64 sum of the f32 taps), ex[1*cells + j] (f64 sum
 * of |tap|) and ex[2*cells + j] (number of non-zero taps).  The f32 outputs are unchanged: tests
 * bound a kernel's per-cell error by these, independently of the order it adds the taps in.
 * `j` = plane offset + cell index inside the plane.
 * ------------------------------------------------------------------------------------------ */
typedef struct {
    double *sum, *abs, *cnt;
} evo_exact;

static inline evo_exact exact_of(double *ex, int64_t cells)
{
    evo_exact e = {ex, ex ? ex + cells : NULL, ex ? ex + 2 * cells : NULL};
    return e;
}

static inline void add_tap(float *out, const evo_exact *e, int64_t plane, int64_t i, float w)
{
    out[i] += w;
    if (e->sum && w != 0.0f) {
        e->sum[plane + i] += (double)w;
        e->abs[plane + i] += fabs((double)w);
        e->cnt[plane + i] += 1.0;
    }
}

/* python / torch advanced-index wrap: [-size,-1] wraps, anything else outside [0,size) is an error */
static inline int wrap_index(int64_t i, int64_t size, int64_t *out)
{
    if (i < 0) i += size;
    if (i < 0 || i >= size) return 0;
    *out = i;
    return 1;
}

/* ------------------------------------------------------------------------------------------
 * voxel_grid.py:129-153  events_to_voxel_torch, all arithmetic f32.
 * t_norm = (t - t0) / dt * (B-1); every one of the B bins receives p * max(0, 1-|t_norm-b|)
 * (zero adds included, NaN propagates like torch.max).  Spatial index = trunc toward zero,
 * negative indices wrap, anything else out of range is the reference's IndexError -> counted
 * in *oob and nothing is written for that event.
 * ------------------------------------------------------------------------------------------ */
EVO_API int64_t evo_voxel_f32(const float *x, const float *y, const float *t, const float *p,
                              int64_t n, float t0, float dt, int B, int H, int W, float *out, double *ex)
{
    int64_t oob = 0;
    const evo_exact e = exact_of(ex, (int64_t)B * H * W);
    const float bm1 = (float)(B - 1);
    for (int64_t i = 0; i < n; ++i) {
        int64_t xi, yi;
        if (!wrap_index(trunc_to_long(x[i]), W, &xi) || !wrap_index(trunc_to_long(y[i]), H, &yi)) {
            ++oob;
            continue;
        }
        float d = t[i] - t0;
        float q = d / dt;
        float tn = q * bm1;
        for (int b = 0; b < B; ++b) {
            float a = fabsf(tn - (float)b);
            float w = 1.0f - a;
            /* torch.max(zeros, w): NaN if w is NaN, else the larger */
            float wb = (w != w) ? w : (w > 0.0f ? w : 0.0f);
            float wt = p[i] * wb;
            add_tap(out, &e, 0, ((int64_t)b * H + yi) * W + xi, wt);
        }
    }
    return oob;
}

/* ------------------------------------------------------------------------------------------
 * voxel_grid.py:198-217  events_to_voxel (numpy): f64 maths, integer coordinates, scatter on an
 * (H+1, W+1) canvas (image.py:17) that is then cropped (image.py:44): an index equal to H or W
 * is silently dropped, anything negative or larger makes ravel_multi_index raise ValueError
 * (returned here as the count of such events; output is then meaningless, as in the reference).
 * ------------------------------------------------------------------------------------------ */
EVO_API int64_t evo_voxel_f64(const int64_t *x, const int64_t *y, const double *t, const double *p,
                              int64_t n, double t0, double dt, int B, int H, int W, double *out)
{
    int64_t bad = 0;
    const double bm1 = (double)(B - 1);
    for (int64_t i = 0; i < n; ++i) {
        int64_t xi = x[i], yi = y[i];
        if (xi < 0 || yi < 0 || xi > W || yi > H) { ++bad; continue; }
        if (xi == W || yi == H) continue; /* lands on the pad row/col, cropped away */
        double tn = (t[i] - t0) / dt * bm1;
        for (int b = 0; b < B; ++b) {
            double w = 1.0 - fabs(tn - (double)b);
            double wb = (w != w) ? w : (w > 0.0 ? w : 0.0); /* np.maximum propagates NaN */
            out[((int64_t)b * H + yi) * W + xi] += p[i] * wb;
        }
    }
    return bad;
}

/* ------------------------------------------------------------------------------------------
 * image.py:62-100 nearest branch.  ``out`` must be pre-filled with ``default`` by the caller.
 * clip != 0: mask = [x < clipx][y < clipy]; the INDEX is multiplied by the mask, the weight
 * is not (image.py:94-95): clipped events deposit their full weight at pixel (0,0).
 * ------------------------------------------------------------------------------------------ */
EVO_API int64_t evo_image_nearest_f32(const float *x, const float *y, const float *p, int64_t n,
                                      int Himg, int Wimg, int clip, float clipx, float clipy,
                                      float *out, double *ex)
{
    int64_t oob = 0;
    const evo_exact e = exact_of(ex, (int64_t)Himg * Wimg);
    for (int64_t i = 0; i < n; ++i) {
        int64_t m = 1;
        if (clip) m = (x[i] >= clipx ? 0 : 1) * (y[i] >= clipy ? 0 : 1);
        int64_t xl = trunc_to_long(x[i]), yl = trunc_to_long(y[i]);
        /* INT64_MIN * 0 == 0 in two's complement, same as torch */
        xl = (m ? xl : 0);
        yl = (m ? yl : 0);
        int64_t xi, yi;
        if (!wrap_index(xl, Wimg, &xi) || !wrap_index(yl, Himg, &yi)) { ++oob; continue; }
        add_tap(out, &e, 0, yi * Wimg + xi, p[i]);
    }
    return oob;
}

/* ------------------------------------------------------------------------------------------
 * image.py:78-86 + 102-115 bilinear branch.  floor / frac in f32, mask applied to the floored
 * coordinate (as a float multiply, then .long()) and to the weight, NOT to dx, dy.
 * Tap weights are evaluated left to right like torch: (w*(1-dx))*(1-dy) etc.
 * Any tap whose index is out of range (after the negative wrap) is the reference's IndexError.
 * ------------------------------------------------------------------------------------------ */
EVO_API int64_t evo_image_bilinear_f32(const float *x, const float *y, const float *p, int64_t n,
                                       int Himg, int Wimg, int clip, float clipx, float clipy,
                                       float *out, double *ex)
{
    int64_t oob = 0;
    const evo_exact e = exact_of(ex, (int64_t)Himg * Wimg);
    for (int64_t i = 0; i < n; ++i) {
        float m = 1.0f;
        if (clip) m = (x[i] >= clipx ? 0.0f : 1.0f) * (y[i] >= clipy ? 0.0f : 1.0f);
        float pxf = floorf(x[i]), pyf = floorf(y[i]);
        float dx = x[i] - pxf, dy = y[i] - pyf;
        int64_t px = trunc_to_long(pxf * m), py = trunc_to_long(pyf * m);
        float w = p[i] * m;
        int64_t x0, x1, y0, y1;
        if (!wrap_index(px, Wimg, &x0) || !wrap_index(px + 1, Wimg, &x1) ||
            !wrap_index(py, Himg, &y0) || !wrap_index(py + 1, Himg, &y1)) { ++oob; continue; }
        float ox = 1.0f - dx, oy = 1.0f - dy;
        add_tap(out, &e, 0, y0 * Wimg + x0, (w * ox) * oy);
        add_tap(out, &e, 0, y0 * Wimg + x1, (w * dx) * oy);
        add_tap(out, &e, 0, y1 * Wimg + x0, (w * ox) * dy);
        add_tap(out, &e, 0, y1 * Wimg + x1, (w * dx) * dy);
    }
    return oob;
}

/* ------------------------------------------------------------------------------------------
 * optic_flow.py:23-46.  flow is (2,H,W) f32.  The reference normalises the pixel coordinate to
 * [-1,1] (x/(W-1)*2-1, f32) and torch's grid_sample (align_corners=True) maps it back with
 * ((g+1)/2)*(W-1); both round trips are kept.  Bilinear, out-of-image taps contribute zero.
 * x' = x + u*(t-t0), y' = y + v*(t-t0).
 * ------------------------------------------------------------------------------------------ */
static inline float flow_tap(const float *f, int H, int W, int64_t yy, int64_t xx)
{
    if (xx < 0 || yy < 0 || xx >= W || yy >= H) return 0.0f;
    return f[yy * W + xx];
}

EVO_API void evo_warp_flow_f32(const float *x, const float *y, const float *t, int64_t n,
                               const float *flow, int H, int W, float t0, float *xw, float *yw)
{
    const float *fu = flow, *fv = flow + (int64_t)H * W;
    const float wm1 = (float)(W - 1), hm1 = (float)(H - 1);
    for (int64_t i = 0; i < n; ++i) {
        float gx = x[i] / wm1 * 2.0f - 1.0f;
        float gy = y[i] / hm1 * 2.0f - 1.0f;
        float ix = ((gx + 1.0f) / 2.0f) * wm1;
        float iy = ((gy + 1.0f) / 2.0f) * hm1;
        float fx = floorf(ix), fy = floorf(iy);
        int64_t x0 = (int64_t)fx, y0 = (int64_t)fy;
        /* ATen grid_sampler: nw = (ix_se-ix)*(iy_se-iy), ne = (ix-ix_sw)*(iy_sw-iy), ... */
        float xe = fx + 1.0f, ye = fy + 1.0f;
        float nw = (xe - ix) * (ye - iy);
        float ne = (ix - fx) * (ye - iy);
        float sw = (xe - ix) * (iy - fy);
        float se = (ix - fx) * (iy - fy);
        float u = 0.0f, v = 0.0f;
        u += flow_tap(fu, H, W, y0, x0) * nw;       v += flow_tap(fv, H, W, y0, x0) * nw;
        u += flow_tap(fu, H, W, y0, x0 + 1) * ne;   v += flow_tap(fv, H, W, y0, x0 + 1) * ne;
        u += flow_tap(fu, H, W, y0 + 1, x0) * sw;   v += flow_tap(fv, H, W, y0 + 1, x0) * sw;
        u += flow_tap(fu, H, W, y0 + 1, x0 + 1) * se; v += flow_tap(fv, H, W, y0 + 1, x0 + 1) * se;
        float d = t[i] - t0;
        xw[i] = x[i] + u * d;
        yw[i] = y[i] + v * d;
    }
}

/* ------------------------------------------------------------------------------------------
 * get_iwe with linvel_warp (objectives.py:184-192, warps.py:52-60, event_util.py:26-27,
 * image.py:179-217).  f64 warp + bounds mask, then the f64->f32 cast, then the bilinear splat on
 * the FIXED (Hs+1)x(Ws+1) canvas (the reference never forwards sensor_size: Hs=180, Ws=240).
 * iwe: (Hs+1)*(Ws+1) f32, zero-filled by caller.  diwe: 2*(Hs+1)*(Ws+1) f32 or NULL.
 * use_polarity == 0 -> p = |p| (objectives.py:184-185).
 * ------------------------------------------------------------------------------------------ */
EVO_API int64_t evo_iwe_linvel(const double *x, const double *y, const double *t, const double *p,
                               int64_t n, double vx, double vy, double t_ref,
                               int Hm, int Wm, int Hs, int Ws, int use_polarity,
                               float *iwe, float *diwe, double *ex)
{
    const int Hc = Hs + 1, Wc = Ws + 1;
    const float clipx = (float)(Wc - 1), clipy = (float)(Hc - 1);
    const int64_t plane = (int64_t)Hc * Wc;
    const evo_exact e = exact_of(ex, plane * 3);   /* planes: IWE, dIWE[0], dIWE[1] */
    int64_t oob = 0;
    for (int64_t i = 0; i < n; ++i) {
        double pp = use_polarity ? p[i] : fabs(p[i]);
        double d = t[i] - t_ref;
        double xw = x[i] - d * vx;
        double yw = y[i] - d * vy;
        double mk = ((xw <= 0.0 || xw > (double)Wm) ? 0.0 : 1.0);
        mk *= ((yw <= 0.0 || yw > (double)Hm) ? 0.0 : 1.0);
        float xf = (float)(xw * mk), yf = (float)(yw * mk), pf = (float)(pp * mk);
        float jf = (float)((-d) * mk);
        float m2 = (xf >= clipx ? 0.0f : 1.0f) * (yf >= clipy ? 0.0f : 1.0f);
        float pxf = floorf(xf), pyf = floorf(yf);
        float dx = xf - pxf, dy = yf - pyf;
        int64_t px = trunc_to_long(pxf * m2), py = trunc_to_long(pyf * m2);
        float w = pf * m2;
        int64_t x0, x1, y0, y1;
        if (!wrap_index(px, Wc, &x0) || !wrap_index(px + 1, Wc, &x1) ||
            !wrap_index(py, Hc, &y0) || !wrap_index(py + 1, Hc, &y1)) { ++oob; continue; }
        float ox = 1.0f - dx, oy = 1.0f - dy;
        add_tap(iwe, &e, 0, y0 * Wc + x0, (w * ox) * oy);
        add_tap(iwe, &e, 0, y0 * Wc + x1, (w * dx) * oy);
        add_tap(iwe, &e, 0, y1 * Wc + x0, (w * ox) * dy);
        add_tap(iwe, &e, 0, y1 * Wc + x1, (w * dx) * dy);
        if (diwe) {
            /* image.py:211-213: w1 = jacobian_x * masked_ps, w2 = jacobian_y * masked_ps with
             * jacobian_x = [-d; 0], jacobian_y = [0; -d] (warps.py:57-60). image.py:131-135. */
            float a = jf * w, z = 0.0f * w;
            float *d0 = diwe, *d1 = diwe + plane;
            add_tap(d0, &e, plane, y0 * Wc + x0, a * (-oy) + z * (-ox));
            add_tap(d0, &e, plane, y0 * Wc + x1, a * oy + z * (-dx));
            add_tap(d0, &e, plane, y1 * Wc + x0, a * (-dy) + z * ox);
            add_tap(d0, &e, plane, y1 * Wc + x1, a * dy + z * dx);
            add_tap(d1, &e, 2 * plane, y0 * Wc + x0, z * (-oy) + a * (-ox));
            add_tap(d1, &e, 2 * plane, y0 * Wc + x1, z * oy + a * (-dx));
            add_tap(d1, &e, 2 * plane, y1 * Wc + x0, z * (-dy) + a * ox);
            add_tap(d1, &e, 2 * plane, y1 * Wc + x1, z * dy + a * dx);
        }
    }
    return oob;
}

/* ------------------------------------------------------------------------------------------
 * scipy.ndimage.gaussian_filter restated: separable, radius = int(4*sigma+0.5), weights
 * exp(-k^2/(2 sigma^2)) normalised in f64, boundary 'reflect' (d c b a | a b c d | d c b a),
 * each line accumulated in f64 and written back to the f32 array before the next axis.
 * ------------------------------------------------------------------------------------------ */
static inline int reflect_idx(int i, int n)
{
    /* scipy 'reflect' = half-sample symmetric, any distance */
    if (n == 1) return 0;
    int period = 2 * n;
    i %= period;
    if (i < 0) i += period;
    return (i < n) ? i : period - 1 - i;
}

EVO_API int evo_gauss_taps(double sigma, double *taps, int max_taps)
{
    int r = (int)(4.0 * sigma + 0.5);
    if (2 * r + 1 > max_taps) return -1;
    double s = 0.0;
    for (int k = -r; k <= r; ++k) { taps[k + r] = exp(-0.5 / (sigma * sigma) * (double)k * (double)k); s += taps[k + r]; }
    for (int k = 0; k <= 2 * r; ++k) taps[k] /= s;
    return r;
}

/* filter along one axis of an array viewed as (outer, len, inner) */
static void gauss_axis_f32(float *a, int64_t outer, int len, int64_t inner, const double *taps, int r)
{
    double *line = (double *)malloc(sizeof(double) * (size_t)len);
    for (int64_t o = 0; o < outer; ++o)
        for (int64_t in = 0; in < inner; ++in) {
            float *base = a + o * len * inner + in;
            for (int i = 0; i < len; ++i) line[i] = (double)base[(int64_t)i * inner];
            for (int i = 0; i < len; ++i) {
                /* scipy correlate1d symmetric path: centre tap, then pairs outward */
                double acc = line[i] * taps[r];
                for (int k = 1; k <= r; ++k)
                    acc += (line[reflect_idx(i - k, len)] + line[reflect_idx(i + k, len)]) * taps[r - k];
                base[(int64_t)i * inner] = (float)acc;
            }
        }
    free(line);
}

/* in-place gaussian_filter over ALL axes of a C-contiguous f32 array of ``ndim`` <= 3 dims */
EVO_API int evo_gaussian_filter_f32(float *a, const int *shape, int ndim, double sigma)
{
    double taps[257];
    if (sigma <= 1e-15) return 0;
    int r = evo_gauss_taps(sigma, taps, 257);
    if (r < 0 || ndim < 1 || ndim > 3) return -1;
    int64_t total = 1;
    for (int d = 0; d < ndim; ++d) total *= shape[d];
    int64_t outer = 1;
    for (int d = 0; d < ndim; ++d) {
        int64_t inner = total / (outer * shape[d]);
        gauss_axis_f32(a, outer, shape[d], inner, taps, r);
        outer *= shape[d];
    }
    return 0;
}

/* ------------------------------------------------------------------------------------------
 * variance_objective (objectives.py:231-236, 251-264).
 *   f   = -var(G(iwe))                                   (G skipped when sigma <= 0)
 *   g_k = -mean( 2*(iwe - mean(iwe)) * G3d(diwe)[k] )    (iwe NOT blurred; G3d blurs axis 0 too)
 * iwe / diwe are not modified (copies are blurred).  Means in f64 (numpy uses pairwise f32;
 * the difference is ~1e-7 relative, inside every tolerance used).
 * ------------------------------------------------------------------------------------------ */
EVO_API double evo_variance_f(const float *iwe, int Hc, int Wc, double sigma)
{
    int64_t np_ = (int64_t)Hc * Wc;
    float *b = (float *)malloc(sizeof(float) * (size_t)np_);
    memcpy(b, iwe, sizeof(float) * (size_t)np_);
    int shape[2] = {Hc, Wc};
    if (sigma > 0) evo_gaussian_filter_f32(b, shape, 2, sigma);
    double s = 0.0;
    for (int64_t i = 0; i < np_; ++i) s += b[i];
    float mu = (float)(s / (double)np_);
    /* np.var(iwe - mean): subtract in f32, then population variance */
    double s1 = 0.0;
    for (int64_t i = 0; i < np_; ++i) { b[i] = b[i] - mu; s1 += b[i]; }
    double mu2 = s1 / (double)np_, s2 = 0.0;
    for (int64_t i = 0; i < np_; ++i) { double d = (double)b[i] - mu2; s2 += d * d; }
    free(b);
    return -(s2 / (double)np_);
}

EVO_API void evo_variance_g(const float *iwe, const float *diwe, int Hc, int Wc, double sigma,
                            double *g /* [2] */)
{
    int64_t np_ = (int64_t)Hc * Wc;
    float *d = (float *)malloc(sizeof(float) * (size_t)np_ * 2);
    memcpy(d, diwe, sizeof(float) * (size_t)np_ * 2);
    int shape[3] = {2, Hc, Wc};
    if (sigma > 0) evo_gaussian_filter_f32(d, shape, 3, sigma);
    double s = 0.0;
    for (int64_t i = 0; i < np_; ++i) s += iwe[i];
    float mu = (float)(s / (double)np_);
    for (int k = 0; k < 2; ++k) {
        double acc = 0.0;
        for (int64_t i = 0; i < np_; ++i) {
            float comp = 2.0f * (iwe[i] - mu);
            acc += (double)(comp * d[k * np_ + i]);
        }
        g[k] = -(acc / (double)np_);
    }
    free(d);
}

/* bounds mask restated on its own (event_util.py:26-27) for the known-answer fixture */
EVO_API void evo_bounds_mask_f64(const double *x, const double *y, int64_t n, double xmin, double xmax,
                                 double ymin, double ymax, double *mask)
{
    for (int64_t i = 0; i < n; ++i) {
        double m = (x[i] <= xmin || x[i] > xmax) ? 0.0 : 1.0;
        m *= (y[i] <= ymin || y[i] > ymax) ? 0.0 : 1.0;
        mask[i] = m;
    }
}

/* ------------------------------------------------------------------------------------------
 * image.py:286-353 events_to_timestamp_image_torch (and :219-284, same arithmetic after its
 * casts): average-timestamp images of the positive / negative events.
 *   tn = (t - t_first) / (t_last - t_first + 1e-6)        (reverse: (-t + t_last) / (...);
 *   reverse == 2: tn = t, the numpy flavour's normalize_timestamps=False, image.py:261)
 *   four bilinear accumulations: tn*[p>0], [p>0], tn*[p<=0], [p<=0]; the two count images
 *   start at ONE (image.py:333,335); the clip mask zeroes the INDEX only, never the weights
 *   (masked_ps is computed but unused, image.py:330); result = sum / count with count==0 -> 1.
 * out: pos then neg, each Himg*Wimg.  ex (exact mode): the four accumulation images Tpos, Cpos, Tneg,
 * Cneg, each without the count images' initial one.
 * ------------------------------------------------------------------------------------------ */
EVO_API int64_t evo_timestamp_image_f32(const float *x, const float *y, const float *t, const float *p, int64_t n,
                                        float t_first, float t_last, int reverse, int Himg, int Wimg, int clip,
                                        float clipx, float clipy, float *out, double *ex)
{
    const int64_t np_ = (int64_t)Himg * Wimg;
    float *acc = (float *)calloc((size_t)np_ * 4, sizeof(float)); /* Tpos, Cpos, Tneg, Cneg */
    const evo_exact e = exact_of(ex, np_ * 4);
    int64_t oob = 0;
    const float denom = (t_last - t_first) + 1e-6f;
    for (int64_t i = 0; i < np_; ++i) { acc[np_ + i] = 1.0f; acc[3 * np_ + i] = 1.0f; }
    for (int64_t i = 0; i < n; ++i) {
        float m = 1.0f;
        if (clip) m = (x[i] >= clipx ? 0.0f : 1.0f) * (y[i] >= clipy ? 0.0f : 1.0f);
        float pxf = floorf(x[i]), pyf = floorf(y[i]);
        float dx = x[i] - pxf, dy = y[i] - pyf;
        int64_t px = trunc_to_long(pxf * m), py = trunc_to_long(pyf * m);
        int64_t x0, x1, y0, y1;
        if (!wrap_index(px, Wimg, &x0) || !wrap_index(px + 1, Wimg, &x1) ||
            !wrap_index(py, Himg, &y0) || !wrap_index(py + 1, Himg, &y1)) { ++oob; continue; }
        float tn = (reverse == 2) ? t[i] : (reverse ? ((-t[i] + t_last) / denom) : ((t[i] - t_first) / denom));
        float pm = (p[i] > 0.0f) ? 1.0f : 0.0f, nm = (p[i] <= 0.0f) ? 1.0f : 0.0f;
        float w[4] = {tn * pm, pm, tn * nm, nm};
        float ox = 1.0f - dx, oy = 1.0f - dy;
        for (int k = 0; k < 4; ++k) {
            float *im = acc + k * np_;
            add_tap(im, &e, k * np_, y0 * Wimg + x0, (w[k] * ox) * oy);
            add_tap(im, &e, k * np_, y0 * Wimg + x1, (w[k] * dx) * oy);
            add_tap(im, &e, k * np_, y1 * Wimg + x0, (w[k] * ox) * dy);
            add_tap(im, &e, k * np_, y1 * Wimg + x1, (w[k] * dx) * dy);
        }
    }
    for (int s = 0; s < 2; ++s)
        for (int64_t i = 0; i < np_; ++i) {
            float c = acc[(2 * s + 1) * np_ + i];
            if (c == 0.0f) c = 1.0f;
            out[s * np_ + i] = acc[(2 * s) * np_ + i] / c;
        }
    free(acc);
    return oob;
}
