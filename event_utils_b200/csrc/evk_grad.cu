// evk_grad.cu -- backward passes of the differentiable torch functions on H100.
//
// The reference builds these outputs from plain torch ops, so autograd runs through them:
//   events_to_image_torch            image.py:46-100 (interpolate_to_image :102-115, index_put_ :95)
//   events_to_timestamp_image_torch  image.py:286-353
//   warp_events_flow_torch           optic_flow.py:5-46 (grid_sample bilinear, zeros, align_corners=True)
//   events_to_voxel_torch            voxel_grid.py:114-153, and its neg/pos and windowed callers :37-112, :155-182
// Each kernel here takes one pass over the events and recomputes the forward's per-event quantities (index,
// clip, wrap, fractions, weights) with the same arithmetic as the forward kernel, so that the taps it reads
// are the taps the forward wrote.  floor() has zero derivative: the gradient is one-sided at integer
// coordinates, as in torch.
//
// Image and timestamp images: the backward is a GATHER of the incoming gradient image(s) at the event's
// taps; the images are L2-resident, the event arrays stream (12-16 B in, 8-12 B out per event).
// Flow warp: the gradient of the flow field is a SCATTER of g*dt*w_tap.  Like the forward image scatter
// (DESIGN.md section 3) it goes through a 2x2-block workspace ws[2][H][W][4]: an event whose footprint lies
// inside the field is ONE red.global.add.v4.f32 per channel; a footprint on the border takes the scalar
// path and drops the taps outside the field (grid_sample's zero padding); image_fold sums the blocks.
#include "evk_common.cuh"

namespace evk {

constexpr int kGradThreads = 256;

// sum of a per-thread double over the CTA, added once per CTA into *dst (dst may be null)
__device__ __forceinline__ void block_red_add_f64(double v, double *dst)
{
    __shared__ double part[kGradThreads / 32];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    if (lane == 0) part[wid] = v;
    __syncthreads();
    if (wid == 0) {
        v = lane < kGradThreads / 32 ? part[lane] : 0.0;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
        if (lane == 0 && dst && v != 0.0) atomicAdd(dst, v);
    }
    __syncthreads();
}

// ---- event image (evk_image_f32) --------------------------------------------------------------
struct ImageGradArgs {
    const float *x, *y, *p;
    int64_t n;
    int H, W, clip;
    float clipx, clipy;
    const float *g;              // [H][W] incoming gradient
    float *gx, *gy, *gp;         // per event, each may be null
};

template <bool BIL>
__device__ __forceinline__ void image_grad_event(const ImageGradArgs &A, float x, float y, float p, float &gx, float &gy,
                                                 float &gp)
{
    gx = 0.0f; gy = 0.0f; gp = 0.0f;
    if (!BIL) {
        // image.py:88-95: out[trunc(y)*m, trunc(x)*m] += p  ->  d/dp = G at that cell, coordinates get nothing
        const bool keep = !A.clip || (!(x >= A.clipx) && !(y >= A.clipy));
        int ux, uy, xi, yi;
        if (!trunc_checked(x, ux) || !trunc_checked(y, uy)) return;
        if (!keep) { ux = 0; uy = 0; }
        if (!wrap_int_index(ux, A.W, xi) || !wrap_int_index(uy, A.H, yi)) return;
        gp = __ldg(A.g + (int64_t)yi * A.W + xi);
        return;
    }
    // image.py:79-86 + :111-114: taps w*(1-dx)(1-dy), w*dx(1-dy), w*(1-dx)dy, w*dx*dy with w = p*m
    float m = 1.0f;
    if (A.clip) m = (x >= A.clipx ? 0.0f : 1.0f) * (y >= A.clipy ? 0.0f : 1.0f);
    const float pxf = floorf(x), pyf = floorf(y);
    const float dx = __fsub_rn(x, pxf), dy = __fsub_rn(y, pyf);
    int upx, upy, x0, x1, y0, y1;
    if (!trunc_checked(__fmul_rn(pxf, m), upx) || !trunc_checked(__fmul_rn(pyf, m), upy) ||
        !wrap_int_index(upx, A.W, x0) || !wrap_int_index(upx + 1, A.W, x1) ||
        !wrap_int_index(upy, A.H, y0) || !wrap_int_index(upy + 1, A.H, y1)) return;
    const float g00 = __ldg(A.g + (int64_t)y0 * A.W + x0), g01 = __ldg(A.g + (int64_t)y0 * A.W + x1);
    const float g10 = __ldg(A.g + (int64_t)y1 * A.W + x0), g11 = __ldg(A.g + (int64_t)y1 * A.W + x1);
    const float ox = __fsub_rn(1.0f, dx), oy = __fsub_rn(1.0f, dy);
    const float w = __fmul_rn(p, m);
    gp = m * (ox * oy * g00 + dx * oy * g01 + ox * dy * g10 + dx * dy * g11);
    gx = w * (oy * (g01 - g00) + dy * (g11 - g10));
    gy = w * (ox * (g10 - g00) + dx * (g11 - g01));
}

template <bool BIL, bool VEC4>
__global__ void __launch_bounds__(kGradThreads) image_grad_kernel(const ImageGradArgs A)
{
    const int64_t tid = (int64_t)blockIdx.x * kGradThreads + threadIdx.x;
    const int64_t stride = (int64_t)gridDim.x * kGradThreads;
    int64_t scalar_from = 0;
    if (VEC4) {
        const int64_t n4 = A.n >> 2;
        for (int64_t q = tid; q < n4; q += stride) {
            const float4 X = ld_stream4(A.x + 4 * q), Y = ld_stream4(A.y + 4 * q), P = ld_stream4(A.p + 4 * q);
            float4 gx, gy, gp;
            image_grad_event<BIL>(A, X.x, Y.x, P.x, gx.x, gy.x, gp.x);
            image_grad_event<BIL>(A, X.y, Y.y, P.y, gx.y, gy.y, gp.y);
            image_grad_event<BIL>(A, X.z, Y.z, P.z, gx.z, gy.z, gp.z);
            image_grad_event<BIL>(A, X.w, Y.w, P.w, gx.w, gy.w, gp.w);
            if (A.gx) __stcs(reinterpret_cast<float4 *>(A.gx + 4 * q), gx);
            if (A.gy) __stcs(reinterpret_cast<float4 *>(A.gy + 4 * q), gy);
            if (A.gp) __stcs(reinterpret_cast<float4 *>(A.gp + 4 * q), gp);
        }
        scalar_from = n4 << 2;
    }
    for (int64_t i = scalar_from + tid; i < A.n; i += stride) {
        float gx, gy, gp;
        image_grad_event<BIL>(A, ld_stream(A.x + i), ld_stream(A.y + i), ld_stream(A.p + i), gx, gy, gp);
        if (A.gx) A.gx[i] = gx;
        if (A.gy) A.gy[i] = gy;
        if (A.gp) A.gp[i] = gp;
    }
}

// ---- timestamp images (evk_timestamp_image_counts_f32) ----------------------------------------
// out = S / C per pixel  ->  dL/dS = G/C, dL/dC = -G*out/C.  ab[s][y][x] = {G/C, G*out/C} for s = pos, neg.
__global__ void __launch_bounds__(256) tsimg_grad_prep_kernel(const float *__restrict__ g_pos, const float *__restrict__ g_neg,
                                                              const float *__restrict__ out_pos, const float *__restrict__ out_neg,
                                                              const float *__restrict__ c_pos, const float *__restrict__ c_neg,
                                                              int64_t npix, float2 *__restrict__ ab)
{
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < 2 * npix; j += stride) {
        const int s = j >= npix;
        const int64_t i = j - s * npix;
        const float g = (s ? g_neg : g_pos)[i], c = (s ? c_neg : c_pos)[i], o = (s ? out_neg : out_pos)[i];
        const float a = __fdiv_rn(g, c);
        ab[j] = make_float2(a, __fmul_rn(a, o));
    }
}

struct TsGradArgs {
    const float *x, *y, *t, *p;
    int64_t n;
    float t_first, t_last, denom, tscale;
    int reverse;
    int H, W, clip;
    float clipx, clipy;
    const float2 *ab;            // [2][H][W]
    float *gx, *gy, *gt;
    double *sums;                // [0] += sum g_tn, [1] += sum g_tn * tn
};

__global__ void __launch_bounds__(kGradThreads) tsimg_grad_kernel(const TsGradArgs A)
{
    const int64_t stride = (int64_t)gridDim.x * kGradThreads;
    const int64_t plane = (int64_t)A.H * A.W;
    double s_g = 0.0, s_gt = 0.0;
    for (int64_t i = (int64_t)blockIdx.x * kGradThreads + threadIdx.x; i < A.n; i += stride) {
        const float x = ld_stream(A.x + i), y = ld_stream(A.y + i), t = ld_stream(A.t + i), p = ld_stream(A.p + i);
        float gx = 0.0f, gy = 0.0f, gt = 0.0f;
        // index, clip and weights exactly as tsimg_scatter_kernel (evk_tsimg.cu)
        float m = 1.0f;
        if (A.clip) m = (x >= A.clipx ? 0.0f : 1.0f) * (y >= A.clipy ? 0.0f : 1.0f);
        const float pxf = floorf(x), pyf = floorf(y);
        const float dx = __fsub_rn(x, pxf), dy = __fsub_rn(y, pyf);
        int upx, upy, x0, x1, y0, y1;
        const bool pos = p > 0.0f, neg = p <= 0.0f;
        if (trunc_checked(__fmul_rn(pxf, m), upx) && trunc_checked(__fmul_rn(pyf, m), upy) &&
            wrap_int_index(upx, A.W, x0) && wrap_int_index(upx + 1, A.W, x1) &&
            wrap_int_index(upy, A.H, y0) && wrap_int_index(upy + 1, A.H, y1) && (pos || neg)) {
            const float tn = A.reverse ? __fdiv_rn(__fadd_rn(-t, A.t_last), A.denom) : __fdiv_rn(__fsub_rn(t, A.t_first), A.denom);
            const float2 *b = A.ab + (neg ? plane : 0);
            const float2 a00 = __ldg(b + (int64_t)y0 * A.W + x0), a01 = __ldg(b + (int64_t)y0 * A.W + x1);
            const float2 a10 = __ldg(b + (int64_t)y1 * A.W + x0), a11 = __ldg(b + (int64_t)y1 * A.W + x1);
            const float ox = __fsub_rn(1.0f, dx), oy = __fsub_rn(1.0f, dy);
            // a tap of weight w adds w*tn to S and w to C: dL/dw = tn*G/C - G*out/C
            const float e00 = tn * a00.x - a00.y, e01 = tn * a01.x - a01.y;
            const float e10 = tn * a10.x - a10.y, e11 = tn * a11.x - a11.y;
            gx = oy * (e01 - e00) + dy * (e11 - e10);
            gy = ox * (e10 - e00) + dx * (e11 - e01);
            const float gtn = ox * oy * a00.x + dx * oy * a01.x + ox * dy * a10.x + dx * dy * a11.x;
            gt = gtn * A.tscale;
            s_g += (double)gtn;
            s_gt += (double)gtn * (double)tn;
        }
        if (A.gx) A.gx[i] = gx;
        if (A.gy) A.gy[i] = gy;
        if (A.gt) A.gt[i] = gt;
    }
    block_red_add_f64(s_g, A.sums);
    block_red_add_f64(s_gt, A.sums ? A.sums + 1 : nullptr);
}

// ---- dense-flow warp (evk_warp_flow_f32) ------------------------------------------------------
struct FlowGradArgs {
    const float *x, *y, *t;
    int64_t n;
    const float *flow;           // [2][H][W]
    int H, W;
    float t0;
    const float *gxw, *gyw;      // incoming gradients of the warped coordinates
    float *gx, *gy, *gt;         // per event, each may be null
    float *ws;                   // [2][H][W][4] blocks {TL,TR,BL,BR}
    double *sum_gt;              // += sum (g_x u + g_y v)
};

__device__ __forceinline__ void flow_grad_one(const FlowGradArgs &A, float xe, float ye, float te, float gxo, float gyo,
                                              float wm1, float hm1, float &gx, float &gy, float &gt)
{
    // sample position, weights and flow exactly as flow_one (evk_image.cu)
    const float gxn = __fsub_rn(__fmul_rn(__fdiv_rn(xe, wm1), 2.0f), 1.0f);
    const float gyn = __fsub_rn(__fmul_rn(__fdiv_rn(ye, hm1), 2.0f), 1.0f);
    const float ix = __fmul_rn(__fdiv_rn(__fadd_rn(gxn, 1.0f), 2.0f), wm1);
    const float iy = __fmul_rn(__fdiv_rn(__fadd_rn(gyn, 1.0f), 2.0f), hm1);
    const float d = __fsub_rn(te, A.t0);
    float u = 0.0f, v = 0.0f, gix = 0.0f, giy = 0.0f;
    if (fabsf(ix) < 1.0e9f && fabsf(iy) < 1.0e9f) {
        const float fx = floorf(ix), fy = floorf(iy);
        const int x0 = (int)fx, y0 = (int)fy;
        const float xs = fx + 1.0f, ys = fy + 1.0f;
        const float wx1 = __fsub_rn(xs, ix), wx0 = __fsub_rn(ix, fx), wy1 = __fsub_rn(ys, iy), wy0 = __fsub_rn(iy, fy);
        const float nw = __fmul_rn(wx1, wy1), ne = __fmul_rn(wx0, wy1), sw = __fmul_rn(wx1, wy0), se = __fmul_rn(wx0, wy0);
        const float4 top = flow_row<false>(A.flow, nullptr, A.H, A.W, y0, x0), bot = flow_row<false>(A.flow, nullptr, A.H, A.W, y0 + 1, x0);
        u = __fadd_rn(u, __fmul_rn(top.x, nw)); v = __fadd_rn(v, __fmul_rn(top.y, nw));
        u = __fadd_rn(u, __fmul_rn(top.z, ne)); v = __fadd_rn(v, __fmul_rn(top.w, ne));
        u = __fadd_rn(u, __fmul_rn(bot.x, sw)); v = __fadd_rn(v, __fmul_rn(bot.y, sw));
        u = __fadd_rn(u, __fmul_rn(bot.z, se)); v = __fadd_rn(v, __fmul_rn(bot.w, se));
        // x' = x + u*d: the sampled flow sees g*d per channel
        const float gu = gxo * d, gv = gyo * d;
        // grid_sample backward w.r.t. the sample position (taps outside the field read 0); the normalise /
        // un-normalise round trip has derivative (W-1)/2 * 2/(W-1) = 1
        const float c00 = gu * top.x + gv * top.y, c01 = gu * top.z + gv * top.w;
        const float c10 = gu * bot.x + gv * bot.y, c11 = gu * bot.z + gv * bot.w;
        gix = wy1 * (c01 - c00) + wy0 * (c11 - c10);
        giy = wx1 * (c10 - c00) + wx0 * (c11 - c01);
        if (gu != 0.0f || gv != 0.0f) {
            const int64_t plane4 = (int64_t)A.H * A.W * 4;
            if (x0 >= 0 && x0 + 1 < A.W && y0 >= 0 && y0 + 1 < A.H) {
                float *blk = A.ws + ((int64_t)y0 * A.W + x0) * 4;
                red_add4(blk, make_float4(gu * nw, gu * ne, gu * sw, gu * se));
                red_add4(blk + plane4, make_float4(gv * nw, gv * ne, gv * sw, gv * se));
            } else {
                // border footprint: every tap inside the field is the TL tap of its own pixel's block
                const int xs_[4] = {x0, x0 + 1, x0, x0 + 1}, ys_[4] = {y0, y0, y0 + 1, y0 + 1};
                const float w_[4] = {nw, ne, sw, se};
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    if ((unsigned)xs_[k] >= (unsigned)A.W || (unsigned)ys_[k] >= (unsigned)A.H) continue;
                    float *blk = A.ws + ((int64_t)ys_[k] * A.W + xs_[k]) * 4;
                    red_add(blk, gu * w_[k]);
                    red_add(blk + plane4, gv * w_[k]);
                }
            }
        }
    }
    gx = gxo + gix;
    gy = gyo + giy;
    gt = gxo * u + gyo * v;
}

template <bool VEC4>
__global__ void __launch_bounds__(kGradThreads) warp_flow_grad_kernel(const FlowGradArgs A)
{
    const float wm1 = (float)(A.W - 1), hm1 = (float)(A.H - 1);
    const int64_t stride = (int64_t)gridDim.x * kGradThreads;
    const int64_t tid = (int64_t)blockIdx.x * kGradThreads + threadIdx.x;
    double s = 0.0;
    int64_t scalar_from = 0;
    if (VEC4) {
        const int64_t n4 = A.n >> 2;
        for (int64_t q = tid; q < n4; q += stride) {
            const float4 xe = ld_stream4(A.x + 4 * q), ye = ld_stream4(A.y + 4 * q), te = ld_stream4(A.t + 4 * q);
            const float4 ga = ld_stream4(A.gxw + 4 * q), gb = ld_stream4(A.gyw + 4 * q);
            float4 gx, gy, gt;
            flow_grad_one(A, xe.x, ye.x, te.x, ga.x, gb.x, wm1, hm1, gx.x, gy.x, gt.x);
            flow_grad_one(A, xe.y, ye.y, te.y, ga.y, gb.y, wm1, hm1, gx.y, gy.y, gt.y);
            flow_grad_one(A, xe.z, ye.z, te.z, ga.z, gb.z, wm1, hm1, gx.z, gy.z, gt.z);
            flow_grad_one(A, xe.w, ye.w, te.w, ga.w, gb.w, wm1, hm1, gx.w, gy.w, gt.w);
            s += (double)gt.x + (double)gt.y + (double)gt.z + (double)gt.w;
            if (A.gx) __stcs(reinterpret_cast<float4 *>(A.gx + 4 * q), gx);
            if (A.gy) __stcs(reinterpret_cast<float4 *>(A.gy + 4 * q), gy);
            if (A.gt) __stcs(reinterpret_cast<float4 *>(A.gt + 4 * q), gt);
        }
        scalar_from = n4 << 2;
    }
    for (int64_t i = scalar_from + tid; i < A.n; i += stride) {
        float gx, gy, gt;
        flow_grad_one(A, ld_stream(A.x + i), ld_stream(A.y + i), ld_stream(A.t + i), ld_stream(A.gxw + i), ld_stream(A.gyw + i),
                      wm1, hm1, gx, gy, gt);
        s += (double)gt;
        if (A.gx) A.gx[i] = gx;
        if (A.gy) A.gy[i] = gy;
        if (A.gt) A.gt[i] = gt;
    }
    block_red_add_f64(s, A.sum_gt);
}

// ---- voxel grid (evk_voxel_f32 / _aos_f32 / _negpos_f32 / _windows_f32) -------------------------
// The reference's bin weight is ps * max(0, 1 - |tn - b|) with tn = ((t - t0) / dt) * (B-1) per window
// (voxel_grid.py:133-139); autograd reaches ps and, through tn, ts.  The incoming gradient is re-laid out once per
// call as pixel-major rows of S = roundup(B, 4) floats ([w][grid][H*W][S]), so that an event's bins floor(tn)-1 ..
// floor(tn)+2 are one or two 16-byte loads from one 32-byte sector (B <= 8) instead of up to four sectors.
struct VoxGradArgs {
    const float *x, *y, *t, *p;  // SoA; AoS: x is the [n][4] record array and y / t / p point into it
    int64_t n;
    int ev_stride;               // floats between consecutive events: 1 (SoA) or 4 (AoS)
    const int64_t *pairs;        // [nw][2] (start, end), or null: one window [0, n)
    int nw, slices;              // CTA (w, s) takes slice s of window w
    int B, H, W, S;
    float bm1;
    int negpos, atomic_out;      // atomic_out: windows may overlap, per-event outputs are added (zeroed first)
    const float *gi;             // [nw][grids][H*W][S]
    float *gp, *gt;              // per event, each may be null
    double *sums;                // [nw][2]: sum G, sum G * tn
};

// One bin of the reference's autograd through w = p * max(0, v), v = 1 - |d|, d = tn - b, with torch's subgradients:
// maximum() gives half the gradient to each side on a tie (v == 0) and all of it to a NaN; abs'(d) = sign(d), and
// sign(0) = sign(NaN) = 0.  Same f32 operations as the forward (voxel_event / add_all_bins_slow).
__device__ __forceinline__ void voxel_bin_grad(float tn, int b, float p, float g, float &gp, float &gtn)
{
    const float d = __fsub_rn(tn, (float)b);
    const float v = __fsub_rn(1.0f, fabsf(d));
    const float bw = (v != v) ? v : (v > 0.0f ? v : 0.0f);
    gp = __fadd_rn(gp, __fmul_rn(g, bw));
    float gv = __fmul_rn(g, p);
    if (v == 0.0f) gv = __fmul_rn(gv, 0.5f);
    if (v < 0.0f) gv = 0.0f;
    const float sg = d > 0.0f ? 1.0f : (d < 0.0f ? -1.0f : 0.0f);
    gtn = __fadd_rn(gtn, __fmul_rn(-gv, sg));
}

// finite tn and p: every bin outside floor(tn)-1 .. floor(tn)+2 has v < 0 and adds 0.  Bin floor(tn)+2 has weight 0 but
// a tie when tn lies within half an ulp of 1 below an integer: d = frac - 2 rounds to -1 (tn = 1 - 2^-24, or tn = -2^-149)
__device__ __forceinline__ void voxel_bins_near(const float *row, int B, float tn, float p, float &gp, float &gtn)
{
    const int f = (int)floorf(tn);
    const int lo = f - 1 < 0 ? 0 : f - 1, hi = f + 2 > B - 1 ? B - 1 : f + 2;
    if (lo > hi) return;
    const float4 *r4 = reinterpret_cast<const float4 *>(row);
    const float4 q0 = __ldg(r4 + (lo >> 2));
    const float4 q1 = (hi >> 2) != (lo >> 2) ? __ldg(r4 + (hi >> 2)) : q0;
#pragma unroll
    for (int k = -1; k <= 2; ++k) {
        const int b = f + k;
        if (b < lo || b > hi) continue;
        const float4 q = (b >> 2) == (lo >> 2) ? q0 : q1;
        const int j = b & 3;
        voxel_bin_grad(tn, b, p, j == 0 ? q.x : j == 1 ? q.y : j == 2 ? q.z : q.w, gp, gtn);
    }
}

// rare path (non-finite tn or p): every bin, so that NaN reaches the gradients exactly where autograd puts it
__device__ __noinline__ float2 voxel_bins_all(const float *row, int B, float tn, float p)
{
    float gp = 0.0f, gtn = 0.0f;
    for (int b = 0; b < B; ++b) voxel_bin_grad(tn, b, p, row[b], gp, gtn);
    return make_float2(gp, gtn);
}

// grad_p and G = dL/dtn of one event; the pixel and tn exactly as voxel_event forms them
__device__ __forceinline__ void voxel_grad_event(const VoxGradArgs &A, const float *gw, float t0, float dt, float x, float y,
                                                 float t, float p, float &gp, float &gtn, float &tn)
{
    gp = 0.0f; gtn = 0.0f;
    tn = __fmul_rn(__fdiv_rn(__fsub_rn(t, t0), dt), A.bm1);
    int xi, yi;
    if (!wrap_trunc_index(x, A.W, xi) || !wrap_trunc_index(y, A.H, yi)) return;  // outside the grid: no taps
    const int64_t grid = (int64_t)A.H * A.W * A.S;
    const float *row = gw + ((int64_t)yi * A.W + xi) * A.S;
    const bool tfin = fabsf(tn) < 1.0e9f;
    if (A.negpos) {
        // weights [p>0] into grid 0 and [p<=0] into grid 1 (voxel_grid.py:172-175); ps gets no gradient
        const float wpos = p > 0.0f ? 1.0f : 0.0f, wneg = p <= 0.0f ? 1.0f : 0.0f;
        float unused = 0.0f;
        if (tfin) {
            if (wpos != 0.0f || wneg != 0.0f) voxel_bins_near(row + (wneg != 0.0f ? grid : 0), A.B, tn, 1.0f, unused, gtn);
        } else {
            const float2 a = voxel_bins_all(row, A.B, tn, wpos), b = voxel_bins_all(row + grid, A.B, tn, wneg);
            gtn = __fadd_rn(a.y, b.y);
        }
    } else if (tfin && fabsf(p) <= FLT_MAX) {
        voxel_bins_near(row, A.B, tn, p, gp, gtn);
    } else {
        const float2 a = voxel_bins_all(row, A.B, tn, p);
        gp = a.x; gtn = a.y;
    }
}

__device__ __forceinline__ void store_grad(float *dst, int atomic_out, float v)
{
    if (atomic_out) red_add(dst, v); else __stcs(dst, v);
}

template <bool VEC4>
__global__ void __launch_bounds__(kGradThreads) voxel_grad_kernel(const VoxGradArgs A)
{
    const int w = blockIdx.x / A.slices, s = blockIdx.x - w * A.slices;
    const int64_t first = A.pairs ? A.pairs[2 * w] : 0, last = A.pairs ? A.pairs[2 * w + 1] : A.n;
    double s_g = 0.0, s_gt = 0.0;
    if (last > first) {
        // t0 / dt of the window as voxel_windows_kernel and EVK_AUTO_SPAN take them
        const float t0 = A.t[first * A.ev_stride], dt = __fsub_rn(A.t[(last - 1) * A.ev_stride], t0);
        const float *gw = A.gi + (int64_t)w * (A.negpos ? 2 : 1) * A.H * A.W * A.S;
        const int64_t tid = (int64_t)s * kGradThreads + threadIdx.x, stride = (int64_t)A.slices * kGradThreads;
        // 16-byte body [a, b) four events at a time; the scalar head [first, a) and tail [b, last)
        int64_t a = first, b = first;
        if (VEC4) {
            a = (first + 3) & ~(int64_t)3;
            if (a > last) a = last;
            b = a + ((last - a) & ~(int64_t)3);
        }
        for (int64_t q = (a >> 2) + tid; q < (b >> 2); q += stride) {
            float4 X, Y, T, P;
            if (A.ev_stride == 4) {
                const float4 e0 = ld_stream4(A.x + 16 * q), e1 = ld_stream4(A.x + 16 * q + 4);
                const float4 e2 = ld_stream4(A.x + 16 * q + 8), e3 = ld_stream4(A.x + 16 * q + 12);
                X = make_float4(e0.x, e1.x, e2.x, e3.x); Y = make_float4(e0.y, e1.y, e2.y, e3.y);
                T = make_float4(e0.z, e1.z, e2.z, e3.z); P = make_float4(e0.w, e1.w, e2.w, e3.w);
            } else {
                X = ld_stream4(A.x + 4 * q); Y = ld_stream4(A.y + 4 * q); T = ld_stream4(A.t + 4 * q); P = ld_stream4(A.p + 4 * q);
            }
            float4 gp, G, tn;
            voxel_grad_event(A, gw, t0, dt, X.x, Y.x, T.x, P.x, gp.x, G.x, tn.x);
            voxel_grad_event(A, gw, t0, dt, X.y, Y.y, T.y, P.y, gp.y, G.y, tn.y);
            voxel_grad_event(A, gw, t0, dt, X.z, Y.z, T.z, P.z, gp.z, G.z, tn.z);
            voxel_grad_event(A, gw, t0, dt, X.w, Y.w, T.w, P.w, gp.w, G.w, tn.w);
            s_g += ((double)G.x + (double)G.y) + ((double)G.z + (double)G.w);
            s_gt += ((double)G.x * (double)tn.x + (double)G.y * (double)tn.y) + ((double)G.z * (double)tn.z + (double)G.w * (double)tn.w);
            if (A.gp) {
                if (A.atomic_out) red_add4(A.gp + 4 * q, gp); else __stcs(reinterpret_cast<float4 *>(A.gp + 4 * q), gp);
            }
            if (A.gt) {
                // dL/dt = G * (B-1) / dt, the reference's two f32 steps
                const float4 g4 = make_float4(__fdiv_rn(__fmul_rn(G.x, A.bm1), dt), __fdiv_rn(__fmul_rn(G.y, A.bm1), dt),
                                              __fdiv_rn(__fmul_rn(G.z, A.bm1), dt), __fdiv_rn(__fmul_rn(G.w, A.bm1), dt));
                if (A.atomic_out) red_add4(A.gt + 4 * q, g4); else __stcs(reinterpret_cast<float4 *>(A.gt + 4 * q), g4);
            }
        }
        const int64_t nhead = a - first, nrest = nhead + (last - b);
        for (int64_t j = tid; j < nrest; j += stride) {
            const int64_t i = j < nhead ? first + j : b + (j - nhead);
            float ex, ey, et, ep;
            if (A.ev_stride == 4) {
                const float4 e = ld_stream4(A.x + 4 * i);
                ex = e.x; ey = e.y; et = e.z; ep = e.w;
            } else {
                ex = ld_stream(A.x + i); ey = ld_stream(A.y + i); et = ld_stream(A.t + i); ep = ld_stream(A.p + i);
            }
            float gp, G, tn;
            voxel_grad_event(A, gw, t0, dt, ex, ey, et, ep, gp, G, tn);
            s_g += (double)G;
            s_gt += (double)G * (double)tn;
            if (A.gp) store_grad(A.gp + i, A.atomic_out, gp);
            if (A.gt) store_grad(A.gt + i, A.atomic_out, __fdiv_rn(__fmul_rn(G, A.bm1), dt));
        }
    }
    block_red_add_f64(s_g, A.sums + 2 * w);
    block_red_add_f64(s_gt, A.sums + 2 * w + 1);
}

// t0 = t[first] and dt = t[last-1] - t[first] depend on the window's end stamps:
//   t[first] += ((sum G * tn) - (B-1) * sum G) / dt,   t[last-1] += -(sum G * tn) / dt
// (atomic: with overlapping windows an end stamp may belong to two windows)
__global__ void __launch_bounds__(128) voxel_grad_ends_kernel(const VoxGradArgs A)
{
    const int w = blockIdx.x * 128 + threadIdx.x;
    if (w >= A.nw) return;
    const int64_t first = A.pairs ? A.pairs[2 * w] : 0, last = A.pairs ? A.pairs[2 * w + 1] : A.n;
    if (last <= first) return;
    const float t0 = A.t[first * A.ev_stride], dt = __fsub_rn(A.t[(last - 1) * A.ev_stride], t0);
    const double s0 = A.sums[2 * w], s1 = A.sums[2 * w + 1];
    atomicAdd(A.gt + first, (float)((s1 - (double)A.bm1 * s0) / (double)dt));
    atomicAdd(A.gt + last - 1, (float)(-s1 / (double)dt));
}

// planar [k][B][npix] -> pixel-major rows [k][npix][S], zero-padded past B
__global__ void __launch_bounds__(256) voxel_grad_interleave_kernel(const float *__restrict__ g, int64_t rows, int64_t npix, int B,
                                                                   int S, float *__restrict__ out)
{
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < rows; r += stride) {
        const int64_t k = r / npix, pix = r - k * npix;
        const float *src = g + k * B * npix + pix;
        float4 *dst = reinterpret_cast<float4 *>(out + r * S);
        for (int c = 0; c < S; c += 4) {
            float v[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) v[j] = c + j < B ? src[(int64_t)(c + j) * npix] : 0.0f;
            dst[c >> 2] = make_float4(v[0], v[1], v[2], v[3]);
        }
    }
}

static inline int voxel_grad_row(int B) { return (B + 3) & ~3; }

static inline bool aligned16(const void *p) { return ((uintptr_t)p & 15) == 0; }

}  // namespace evk

extern "C" {

int evk_image_grad_f32(const float *x, const float *y, const float *p, int64_t n, int Himg, int Wimg, float clipx,
                       float clipy, unsigned flags, const float *grad_img, float *grad_x, float *grad_y, float *grad_p,
                       void *stream)
{
    using namespace evk;
    const bool bil = (flags & EVK_BILINEAR) != 0;
    if (n < 0 || Himg < 1 || Wimg < 1 || !grad_img || (n > 0 && (!x || !y || !p))) {
        set_error("evk_image_grad_f32: bad arguments");
        return EVK_E_ARG;
    }
    if (bil && (Himg < 2 || Wimg < 2)) { set_error("evk_image_grad_f32: bilinear needs a canvas of at least 2x2"); return EVK_E_ARG; }
    if (n == 0 || (!grad_p && (!bil || (!grad_x && !grad_y)))) return EVK_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    ImageGradArgs A{};
    A.x = x; A.y = y; A.p = p; A.n = n; A.H = Himg; A.W = Wimg;
    A.clip = (flags & EVK_CLIP) ? 1 : 0; A.clipx = clipx; A.clipy = clipy;
    A.g = grad_img; A.gp = grad_p;
    if (bil) { A.gx = grad_x; A.gy = grad_y; }
    const bool vec = aligned16(x) && aligned16(y) && aligned16(p) && aligned16(A.gx) && aligned16(A.gy) && aligned16(A.gp);
    prof_count(1);
#define EVK_IG_LAUNCH(B, V) image_grad_kernel<B, V><<<grid_for(image_grad_kernel<B, V>, kGradThreads, n, kGradThreads * 8), kGradThreads, 0, st>>>(A)
    if (bil) { if (vec) EVK_IG_LAUNCH(true, true); else EVK_IG_LAUNCH(true, false); }
    else { if (vec) EVK_IG_LAUNCH(false, true); else EVK_IG_LAUNCH(false, false); }
#undef EVK_IG_LAUNCH
    EVK_CUDA(cudaGetLastError());
    return EVK_OK;
}

size_t evk_timestamp_image_grad_workspace_bytes(int Himg, int Wimg)
{
    if (Himg < 2 || Wimg < 2) return 0;
    return (size_t)2 * Himg * Wimg * sizeof(float2);
}

int evk_timestamp_image_grad_f32(const float *x, const float *y, const float *t, const float *p, int64_t n, float t_first,
                                 float t_last, int Himg, int Wimg, float clipx, float clipy, unsigned flags,
                                 const float *grad_pos, const float *grad_neg, const float *out_pos, const float *out_neg,
                                 const float *cnt_pos, const float *cnt_neg, float *grad_x, float *grad_y, float *grad_t,
                                 double *sums, void *workspace, size_t workspace_bytes, void *stream)
{
    using namespace evk;
    if (n < 0 || Himg < 2 || Wimg < 2 || !grad_pos || !grad_neg || !out_pos || !out_neg || !cnt_pos || !cnt_neg ||
        (n > 0 && (!x || !y || !t || !p)) || (flags & EVK_TS_RAW)) {
        set_error("evk_timestamp_image_grad_f32: bad arguments");
        return EVK_E_ARG;
    }
    const size_t need = evk_timestamp_image_grad_workspace_bytes(Himg, Wimg);
    if (!workspace || workspace_bytes < need || ((uintptr_t)workspace & 15)) {
        set_error("evk_timestamp_image_grad_f32: 16-byte aligned workspace of %zu bytes required", need);
        return EVK_E_WORKSPACE;
    }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (sums) EVK_CUDA(cudaMemsetAsync(sums, 0, 2 * sizeof(double), st));
    if (n == 0) return EVK_OK;
    const int64_t npix = (int64_t)Himg * Wimg;
    float2 *ab = static_cast<float2 *>(workspace);
    prof_count(1);
    tsimg_grad_prep_kernel<<<grid_simple(2 * npix, 256), 256, 0, st>>>(grad_pos, grad_neg, out_pos, out_neg, cnt_pos, cnt_neg, npix, ab);
    TsGradArgs A{};
    A.x = x; A.y = y; A.t = t; A.p = p; A.n = n;
    A.t_first = t_first; A.t_last = t_last;
    A.denom = (t_last - t_first) + 1e-6f;  // as evk_timestamp_image_f32
    A.reverse = (flags & EVK_TS_REVERSE) ? 1 : 0;
    A.tscale = (A.reverse ? -1.0f : 1.0f) / A.denom;  // d tn / d t
    A.H = Himg; A.W = Wimg; A.clip = (flags & EVK_CLIP) ? 1 : 0; A.clipx = clipx; A.clipy = clipy;
    A.ab = ab; A.gx = grad_x; A.gy = grad_y; A.gt = grad_t; A.sums = sums;
    prof_count(1);
    tsimg_grad_kernel<<<grid_for(tsimg_grad_kernel, kGradThreads, n, kGradThreads * 8), kGradThreads, 0, st>>>(A);
    EVK_CUDA(cudaGetLastError());
    return EVK_OK;
}

size_t evk_warp_flow_grad_workspace_bytes(int H, int W)
{
    if (H < 1 || W < 1) return 0;
    return (size_t)2 * H * W * 4 * sizeof(float);
}

int evk_warp_flow_grad_f32(const float *x, const float *y, const float *t, int64_t n, const float *flow, int H, int W,
                           float t0, const float *grad_xw, const float *grad_yw, float *grad_x, float *grad_y,
                           float *grad_t, float *grad_flow, double *sum_grad_t, void *workspace, size_t workspace_bytes,
                           void *stream)
{
    using namespace evk;
    if (n < 0 || H < 1 || W < 1 || !flow || !grad_flow || (n > 0 && (!x || !y || !t || !grad_xw || !grad_yw))) {
        set_error("evk_warp_flow_grad_f32: bad arguments");
        return EVK_E_ARG;
    }
    const size_t need = evk_warp_flow_grad_workspace_bytes(H, W);
    if (!workspace || workspace_bytes < need || ((uintptr_t)workspace & 15)) {
        set_error("evk_warp_flow_grad_f32: 16-byte aligned workspace of %zu bytes required", need);
        return EVK_E_WORKSPACE;
    }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int64_t npix = (int64_t)H * W;
    if (sum_grad_t) EVK_CUDA(cudaMemsetAsync(sum_grad_t, 0, sizeof(double), st));
    EVK_CUDA(cudaMemsetAsync(workspace, 0, need, st));
    if (n > 0) {
        FlowGradArgs A{};
        A.x = x; A.y = y; A.t = t; A.n = n; A.flow = flow; A.H = H; A.W = W; A.t0 = t0;
        A.gxw = grad_xw; A.gyw = grad_yw; A.gx = grad_x; A.gy = grad_y; A.gt = grad_t;
        A.ws = static_cast<float *>(workspace); A.sum_gt = sum_grad_t;
        const bool vec = aligned16(x) && aligned16(y) && aligned16(t) && aligned16(grad_xw) && aligned16(grad_yw) &&
                         aligned16(grad_x) && aligned16(grad_y) && aligned16(grad_t);
        prof_count(1);
        if (vec) warp_flow_grad_kernel<true><<<grid_for(warp_flow_grad_kernel<true>, kGradThreads, n, kGradThreads * 8), kGradThreads, 0, st>>>(A);
        else warp_flow_grad_kernel<false><<<grid_for(warp_flow_grad_kernel<false>, kGradThreads, n, kGradThreads * 4), kGradThreads, 0, st>>>(A);
    }
    const float *ws = static_cast<const float *>(workspace);
    launch_image_fold(ws, grad_flow, H, W, st);
    launch_image_fold(ws + npix * 4, grad_flow + npix, H, W, st);
    EVK_CUDA(cudaGetLastError());
    return EVK_OK;
}

size_t evk_voxel_grad_workspace_bytes(int n_windows, int B, int H, int W, unsigned flags)
{
    if (n_windows < 1 || B < 1 || H < 1 || W < 1) return 0;
    const size_t sums = ((size_t)n_windows * 2 * sizeof(double) + 255) & ~(size_t)255;
    const size_t grids = (flags & EVK_WINDOW_NEGPOS) ? 2 : 1;
    return sums + (size_t)n_windows * grids * H * W * evk::voxel_grad_row(B) * sizeof(float);
}

int evk_voxel_grad_f32(const float *x, const float *y, const float *t, const float *p, int64_t n, const int64_t *pairs,
                       int n_windows, int B, int H, int W, unsigned flags, const float *grad_out, float *grad_p,
                       float *grad_t, void *workspace, size_t workspace_bytes, void *stream)
{
    using namespace evk;
    const bool aos = (flags & EVK_EVENTS_AOS) != 0, negpos = (flags & EVK_WINDOW_NEGPOS) != 0;
    if (n < 0 || n_windows < 1 || B < 1 || H < 1 || W < 1 || !grad_out || (!pairs && n_windows != 1) ||
        (n > 0 && (!x || (!aos && (!y || !t || !p)))) || (aos && ((uintptr_t)x & 15)) || (flags & EVK_NEGPOS_TRUTHY) ||
        (flags & EVK_BILINEAR) || (int64_t)B * H * W >= ((int64_t)1 << 40)) {
        set_error("evk_voxel_grad_f32: bad arguments");
        return EVK_E_ARG;
    }
    const size_t need = evk_voxel_grad_workspace_bytes(n_windows, B, H, W, flags);
    if (!workspace || workspace_bytes < need || ((uintptr_t)workspace & 255)) {
        set_error("evk_voxel_grad_f32: 256-byte aligned workspace of %zu bytes required", need);
        return EVK_E_WORKSPACE;
    }
    if (negpos) grad_p = nullptr;
    if (n == 0 || (!grad_p && !grad_t)) return EVK_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    VoxGradArgs A{};
    A.x = x; A.n = n;
    if (aos) { A.y = x + 1; A.t = x + 2; A.p = x + 3; A.ev_stride = 4; }
    else { A.y = y; A.t = t; A.p = p; A.ev_stride = 1; }
    A.pairs = pairs; A.nw = n_windows;
    A.B = B; A.H = H; A.W = W; A.S = voxel_grad_row(B); A.bm1 = (float)(B - 1);
    A.negpos = negpos ? 1 : 0;
    A.atomic_out = (flags & EVK_WINDOW_OVERLAP) ? 1 : 0;
    A.gp = grad_p; A.gt = grad_t;
    A.sums = static_cast<double *>(workspace);
    const size_t sums_bytes = ((size_t)n_windows * 2 * sizeof(double) + 255) & ~(size_t)255;
    float *gi = reinterpret_cast<float *>(static_cast<char *>(workspace) + sums_bytes);
    A.gi = gi;
    EVK_CUDA(cudaMemsetAsync(A.sums, 0, (size_t)n_windows * 2 * sizeof(double), st));
    if (pairs) {
        // events outside every window get 0; overlapping windows add into the zeroed outputs
        if (A.gp) EVK_CUDA(cudaMemsetAsync(A.gp, 0, (size_t)n * sizeof(float), st));
        if (A.gt) EVK_CUDA(cudaMemsetAsync(A.gt, 0, (size_t)n * sizeof(float), st));
    } else {
        A.atomic_out = 0;
    }
    const int64_t npix = (int64_t)H * W, rows = (int64_t)n_windows * (negpos ? 2 : 1) * npix;
    prof_count(1);
    voxel_grad_interleave_kernel<<<grid_simple(rows, 256), 256, 0, st>>>(grad_out, rows, npix, B, A.S, gi);
    const bool vec = (aos || (aligned16(x) && aligned16(y) && aligned16(t) && aligned16(p))) && aligned16(A.gp) &&
                     aligned16(A.gt);
    // slices per window: a full wave for one window; for many, enough CTAs to fill the machine, at most one per 2K events
    const int cap = grid_for(voxel_grad_kernel<true>, kGradThreads, (int64_t)1 << 40, 1);
    const int64_t per = n / n_windows;
    int64_t slices = (per + kGradThreads * 8 - 1) / (kGradThreads * 8);
    const int64_t fill = (cap + n_windows - 1) / n_windows;
    if (slices > fill) slices = fill;
    if (slices < 1) slices = 1;
    if ((int64_t)n_windows * slices > 0x7fffffffLL) { set_error("evk_voxel_grad_f32: too many windows"); return EVK_E_ARG; }
    A.slices = (int)slices;
    prof_count(1);
    if (vec) voxel_grad_kernel<true><<<(unsigned)(n_windows * slices), kGradThreads, 0, st>>>(A);
    else voxel_grad_kernel<false><<<(unsigned)(n_windows * slices), kGradThreads, 0, st>>>(A);
    if (A.gt) {
        prof_count(1);
        voxel_grad_ends_kernel<<<(n_windows + 127) / 128, 128, 0, st>>>(A);
    }
    EVK_CUDA(cudaGetLastError());
    return EVK_OK;
}

}  // extern "C"
