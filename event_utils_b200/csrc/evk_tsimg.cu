// evk_tsimg.cu -- average-timestamp images (Zhu et al. 2019) of the positive / negative events.
//
// Semantics: events_to_timestamp_image_torch, reference lib/representations/image.py:286-353
// (and the numpy flavour :219-284, which is the same arithmetic after its casts):
//   tn = (t - t_first) / (t_last - t_first + 1e-6)         (reverse: (-t + t_last) / (...))
//   four bilinear accumulations -- tn*[p>0], [p>0], tn*[p<=0], [p<=0] -- then sum / count, where
//   the count images START AT ONE (image.py:333,335) and the clip mask zeroes only the INDEX of a
//   clipped event, not its weight (masked_ps is computed but unused, image.py:330).
//
// Design: an event touches only the two images of its own polarity.  They share one array
// of 32-byte blocks, block (s,y,x) = {T_TL,T_TR,T_BL,T_BR, C_TL,C_TR,C_BL,C_BR} for polarity s and
// the 2x2 footprint anchored at (y,x): the reference's 16 scalar scatters per event become TWO
// red.global.add.v4.f32 into one L2 sector.  A fold kernel sums the four blocks each pixel lives
// in, adds the count bias and divides.
#include "evk_common.cuh"

namespace evk {

struct TsArgs {
    const float *x, *y, *t, *p;
    int64_t n;
    float t_first, t_last, denom;
    int reverse;
    int H, W, clip;
    float clipx, clipy;
    float *ws;  // [2][H][W][8]
    unsigned long long *oob;
};

__global__ void __launch_bounds__(256) tsimg_scatter_kernel(const TsArgs A)
{
    unsigned oob = 0;
    const int64_t stride = (int64_t)gridDim.x * 256;
    const int64_t plane = (int64_t)A.H * A.W;
    for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < A.n; i += stride) {
        const float x = ld_stream(A.x + i), y = ld_stream(A.y + i), t = ld_stream(A.t + i), p = ld_stream(A.p + i);
        float m = 1.0f;
        if (A.clip) m = (x >= A.clipx ? 0.0f : 1.0f) * (y >= A.clipy ? 0.0f : 1.0f);
        const float pxf = floorf(x), pyf = floorf(y);
        const float dx = __fsub_rn(x, pxf), dy = __fsub_rn(y, pyf);
        int upx, upy, x0, x1, y0, y1;
        if (!trunc_checked(__fmul_rn(pxf, m), upx) || !trunc_checked(__fmul_rn(pyf, m), upy) ||
            !wrap_int_index(upx, A.W, x0) || !wrap_int_index(upx + 1, A.W, x1) ||
            !wrap_int_index(upy, A.H, y0) || !wrap_int_index(upy + 1, A.H, y1)) { ++oob; continue; }
        const bool pos = p > 0.0f, neg = p <= 0.0f;
        if (!pos && !neg) continue;  // NaN polarity: both masks are 0
        const float tn = A.reverse ? __fdiv_rn(__fadd_rn(-t, A.t_last), A.denom) : __fdiv_rn(__fsub_rn(t, A.t_first), A.denom);
        const float ox = __fsub_rn(1.0f, dx), oy = __fsub_rn(1.0f, dy);
        // weights: tn * 1 for the timestamp image, 1 for the count image (image.py:327-328)
        const float tl = __fmul_rn(tn, ox), tr = __fmul_rn(tn, dx);
        const float4 tt = make_float4(__fmul_rn(tl, oy), __fmul_rn(tr, oy), __fmul_rn(tl, dy), __fmul_rn(tr, dy));
        const float4 cc = make_float4(__fmul_rn(ox, oy), __fmul_rn(dx, oy), __fmul_rn(ox, dy), __fmul_rn(dx, dy));
        float *base = A.ws + (neg ? plane * 8 : 0);
        if (x1 == x0 + 1 && y1 == y0 + 1) {
            float *blk = base + ((int64_t)y0 * A.W + x0) * 8;
            red_add4(blk, tt);
            red_add4(blk + 4, cc);
        } else {
            const float tv[4] = {tt.x, tt.y, tt.z, tt.w}, cv[4] = {cc.x, cc.y, cc.z, cc.w};
            const int ys[4] = {y0, y0, y1, y1}, xs[4] = {x0, x1, x0, x1};
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                float *blk = base + ((int64_t)ys[k] * A.W + xs[k]) * 8;  // TL tap of that pixel's block
                red_add(blk, tv[k]);
                red_add(blk + 4, cv[k]);
            }
        }
    }
    flush_oob(A.oob, oob);
}

__global__ void __launch_bounds__(256) tsimg_fold_kernel(const float *__restrict__ ws, float *__restrict__ out_pos,
                                                         float *__restrict__ out_neg, int H, int W)
{
    const int64_t npix = (int64_t)H * W;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < 2 * npix; j += stride) {
        const int s = j >= npix;
        const int64_t i = j - s * npix;
        const int y = (int)(i / W), x = (int)(i - (int64_t)y * W);
        const float *b = ws + (s * npix + i) * 8;
        float tsum = b[0], csum = b[4];
        if (x > 0) { tsum += b[-8 + 1]; csum += b[-8 + 5]; }
        if (y > 0) { tsum += b[-8 * (int64_t)W + 2]; csum += b[-8 * (int64_t)W + 6]; }
        if (x > 0 && y > 0) { tsum += b[-8 * ((int64_t)W + 1) + 3]; csum += b[-8 * ((int64_t)W + 1) + 7]; }
        float c = __fadd_rn(1.0f, csum);  // count images are initialised to ones (image.py:333,335)
        if (c == 0.0f) c = 1.0f;
        (s ? out_neg : out_pos)[i] = __fdiv_rn(tsum, c);
    }
}

}  // namespace evk

extern "C" {

size_t evk_timestamp_image_workspace_bytes(int Himg, int Wimg)
{
    if (Himg < 2 || Wimg < 2) return 0;
    return (size_t)2 * Himg * Wimg * 8 * sizeof(float);
}

int evk_timestamp_image_f32(const float *x, const float *y, const float *t, const float *p, int64_t n, float t_first,
                            float t_last, int Himg, int Wimg, float clipx, float clipy, unsigned flags, float *out_pos,
                            float *out_neg, void *workspace, size_t workspace_bytes, unsigned long long *oob, void *stream)
{
    using namespace evk;
    if (n < 0 || Himg < 2 || Wimg < 2 || !out_pos || !out_neg || (n > 0 && (!x || !y || !t || !p))) {
        set_error("evk_timestamp_image_f32: bad arguments");
        return EVK_E_ARG;
    }
    const size_t need = evk_timestamp_image_workspace_bytes(Himg, Wimg);
    if (!workspace || workspace_bytes < need || ((uintptr_t)workspace & 15)) {
        set_error("evk_timestamp_image_f32: 16-byte aligned workspace of %zu bytes required", need);
        return EVK_E_WORKSPACE;
    }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    TsArgs A{};
    A.x = x; A.y = y; A.t = t; A.p = p; A.n = n;
    A.t_first = t_first; A.t_last = t_last;
    A.denom = (t_last - t_first) + 1e-6f;  // f32: ts[-1]-ts[0]+epsilon (image.py:317-321)
    if (flags & EVK_TS_RAW) { A.t_first = 0.0f; A.denom = 1.0f; }  // (t - 0) / 1 == t exactly: normalize_timestamps=False (image.py:261)
    A.reverse = (flags & EVK_TS_REVERSE) ? 1 : 0;
    A.H = Himg; A.W = Wimg; A.clip = (flags & EVK_CLIP) ? 1 : 0; A.clipx = clipx; A.clipy = clipy;
    A.ws = static_cast<float *>(workspace); A.oob = oob;
    EVK_CUDA(cudaMemsetAsync(A.ws, 0, need, st));
    if (n > 0) {
        ProfScope prof(st);
        prof_count(1);
        tsimg_scatter_kernel<<<grid_for(tsimg_scatter_kernel, 256, n, 256 * 8), 256, 0, st>>>(A);
    }
    prof_count(1);
    tsimg_fold_kernel<<<grid_simple((int64_t)2 * Himg * Wimg, 256), 256, 0, st>>>(A.ws, out_pos, out_neg, Himg, Wimg);
    EVK_CUDA(cudaGetLastError());
    return EVK_OK;
}

}  // extern "C"
