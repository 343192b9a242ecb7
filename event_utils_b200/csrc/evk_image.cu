// evk_image.cu -- events -> 2-D event image (nearest / bilinear), integer count image and the
// dense-flow warp on H100.
//
// Semantics:
//   events_to_image_torch   reference lib/representations/image.py:46-100
//   interpolate_to_image    reference lib/representations/image.py:102-115
//   warp_events_flow_torch  reference lib/transforms/optic_flow.py:5-46
//
// Variants (DESIGN.md section 3):
//   GLOBAL_RED : one red.global.add.f32 per tap straight into out.
//   VECTOR_RED : (bilinear) a "block" workspace ws[H][W][4]: block (y,x) collects the four taps
//                TL,TR,BL,BR of every event whose 2x2 footprint is anchored at (y,x), so an event is
//                ONE red.global.add.v4.f32 instead of 4 scalar reds; a fold kernel sums the four
//                blocks each pixel lives in.
//   WARP_AGG   : lanes of a warp that hit the same cell are combined with match.any before the
//                red (hot-spot / Zipf streams, where same-address serialisation in L2 dominates).
#include "evk_common.cuh"

namespace evk {

struct ImageArgs {
    const float *x, *y, *p;
    int64_t n;
    int H, W;  // canvas
    int clip;
    float clipx, clipy;
    float *out;
    float *ws;
    unsigned *out_u32;
    unsigned long long *oob;
};

enum { ISINK_SCALAR = 0, ISINK_QUAD = 1, ISINK_WARPAGG = 2 };

// Combine lanes that target the same cell: every lane learns its peers, the lowest peer lane
// adds the group's sum.  Returns true in the lane that must issue the red, with `v` = group sum.
__device__ __forceinline__ bool warp_combine(int64_t cell, bool active, float &v)
{
    // inactive lanes use a cell id no active lane can have
    const unsigned long long key = active ? (unsigned long long)cell : ~0ull - (threadIdx.x & 31);
    unsigned peers = __match_any_sync(0xffffffffu, key);
    const int lane = threadIdx.x & 31;
    const int leader = __ffs(peers) - 1;
    // segmented sum: walk the peer mask (groups are small except on the hottest cells)
    float sum = 0.0f;
    unsigned any_multi = __ballot_sync(0xffffffffu, peers != (1u << lane));
    if (any_multi == 0) return active;  // all cells distinct: nothing to combine
    // every lane publishes its value; leaders accumulate their peers in lane order
    for (int src = 0; src < 32; ++src) {
        float o = __shfl_sync(0xffffffffu, v, src);
        if ((peers >> src) & 1u) sum += o;
    }
    v = sum;
    return active && lane == leader;
}

template <int SINK, bool BIL>
__device__ __forceinline__ void image_event(const ImageArgs &A, float x, float y, float p, bool valid,
                                            unsigned &oob)
{
    if (!BIL) {
        // image.py:88-95: index = trunc(coord) * mask, weight NOT masked
        int xi = 0, yi = 0;
        bool ok = valid;
        if (ok) {
            const bool keep = !A.clip || (!(x >= A.clipx) && !(y >= A.clipy));
            int ux, uy;
            if (!trunc_checked(x, ux) || !trunc_checked(y, uy)) { ok = false; ++oob; }
            else {
                if (!keep) { ux = 0; uy = 0; }
                if (!wrap_int_index(ux, A.W, xi) || !wrap_int_index(uy, A.H, yi)) { ok = false; ++oob; }
            }
        }
        const int64_t cell = (int64_t)yi * A.W + xi;
        if (SINK == ISINK_WARPAGG) {
            float v = ok ? p : 0.0f;
            if (warp_combine(cell, ok, v) && v != 0.0f) red_add(A.out + cell, v);
        } else {
            if (ok && p != 0.0f) red_add(A.out + cell, p);
        }
    } else {
        // image.py:79-86 + 111-114
        if (!valid) return;
        float m = 1.0f;
        if (A.clip) m = (x >= A.clipx ? 0.0f : 1.0f) * (y >= A.clipy ? 0.0f : 1.0f);
        const float pxf = floorf(x), pyf = floorf(y);
        const float dx = __fsub_rn(x, pxf), dy = __fsub_rn(y, pyf);
        int upx, upy, x0, x1, y0, y1;
        if (!trunc_checked(__fmul_rn(pxf, m), upx) || !trunc_checked(__fmul_rn(pyf, m), upy) ||
            !wrap_int_index(upx, A.W, x0) || !wrap_int_index(upx + 1, A.W, x1) ||
            !wrap_int_index(upy, A.H, y0) || !wrap_int_index(upy + 1, A.H, y1)) { ++oob; return; }
        const float w = __fmul_rn(p, m);
        const float ox = __fsub_rn(1.0f, dx), oy = __fsub_rn(1.0f, dy);
        const float wl = __fmul_rn(w, ox), wr = __fmul_rn(w, dx);
        const float v00 = __fmul_rn(wl, oy), v01 = __fmul_rn(wr, oy);
        const float v10 = __fmul_rn(wl, dy), v11 = __fmul_rn(wr, dy);
        if (SINK == ISINK_QUAD) {
            // block workspace ws[H][W][4]: the whole 2x2 footprint anchored at (y0,x0) is ONE
            // red.global.add.v4.f32 {TL,TR,BL,BR}; image_fold_kernel sums the four blocks a pixel is in
            if (v00 == 0.0f && v01 == 0.0f && v10 == 0.0f && v11 == 0.0f) return;
            if (x1 == x0 + 1 && y1 == y0 + 1) {
                red_add4(A.ws + ((int64_t)y0 * A.W + x0) * 4, make_float4(v00, v01, v10, v11));
            } else {
                // wrapped footprint (negative px / py): each tap is the TL tap of its own pixel's block
                if (v00 != 0.0f) red_add(A.ws + ((int64_t)y0 * A.W + x0) * 4, v00);
                if (v01 != 0.0f) red_add(A.ws + ((int64_t)y0 * A.W + x1) * 4, v01);
                if (v10 != 0.0f) red_add(A.ws + ((int64_t)y1 * A.W + x0) * 4, v10);
                if (v11 != 0.0f) red_add(A.ws + ((int64_t)y1 * A.W + x1) * 4, v11);
            }
        } else {
            if (v00 != 0.0f) red_add(A.out + (int64_t)y0 * A.W + x0, v00);
            if (v01 != 0.0f) red_add(A.out + (int64_t)y0 * A.W + x1, v01);
            if (v10 != 0.0f) red_add(A.out + (int64_t)y1 * A.W + x0, v10);
            if (v11 != 0.0f) red_add(A.out + (int64_t)y1 * A.W + x1, v11);
        }
    }
}

constexpr int kThreads = 256;

template <int SINK, bool BIL, bool VEC4>
__global__ void __launch_bounds__(kThreads) image_scatter_kernel(const ImageArgs A)
{
    unsigned oob = 0;
    const int64_t tid = (int64_t)blockIdx.x * kThreads + threadIdx.x;
    const int64_t stride = (int64_t)gridDim.x * kThreads;
    if (VEC4) {
        const int64_t n4 = A.n >> 2;
        // warp-uniform trip count so that the warp-aggregated variant can use full-mask collectives
        const int64_t iters = (n4 + stride - 1) / stride;
        for (int64_t it = 0; it < iters; ++it) {
            const int64_t g = tid + it * stride;
            const bool v = g < n4;
            float4 X = make_float4(0, 0, 0, 0), Y = X, P = X;
            if (v) { X = ld_stream4(A.x + 4 * g); Y = ld_stream4(A.y + 4 * g); P = ld_stream4(A.p + 4 * g); }
            image_event<SINK, BIL>(A, X.x, Y.x, P.x, v, oob);
            image_event<SINK, BIL>(A, X.y, Y.y, P.y, v, oob);
            image_event<SINK, BIL>(A, X.z, Y.z, P.z, v, oob);
            image_event<SINK, BIL>(A, X.w, Y.w, P.w, v, oob);
        }
        const int64_t tail0 = n4 << 2;
        const int64_t j = tail0 + tid;
        if (tail0 < A.n && tid < 32 * ((A.n - tail0 + 31) / 32)) {
            const bool v = j < A.n;
            image_event<SINK, BIL>(A, v ? A.x[j] : 0.f, v ? A.y[j] : 0.f, v ? A.p[j] : 0.f, v, oob);
        }
    } else {
        const int64_t iters = (A.n + stride - 1) / stride;
        for (int64_t it = 0; it < iters; ++it) {
            const int64_t i = tid + it * stride;
            const bool v = i < A.n;
            image_event<SINK, BIL>(A, v ? ld_stream(A.x + i) : 0.f, v ? ld_stream(A.y + i) : 0.f,
                                   v ? ld_stream(A.p + i) : 0.f, v, oob);
        }
    }
    flush_oob(A.oob, oob);
}

__global__ void __launch_bounds__(256) fill_kernel(float *out, int64_t n, float v)
{
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) out[i] = v;
}

// block workspace -> out[H][W] (+ fill): pixel (y,x) = TL of block (y,x) + TR of (y,x-1) + BL of
// (y-1,x) + BR of (y-1,x-1)
template <bool ACCUM>
__global__ void __launch_bounds__(256) image_fold_kernel(const float *__restrict__ ws, float *__restrict__ out,
                                                         int H, int W, float fill)
{
    const int64_t npix = (int64_t)H * W;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < npix; i += stride) {
        const int y = (int)(i / W), x = (int)(i - (int64_t)y * W);
        float v = ws[i * 4];
        if (x > 0) v += ws[(i - 1) * 4 + 1];
        if (y > 0) v += ws[(i - W) * 4 + 2];
        if (x > 0 && y > 0) v += ws[(i - W - 1) * 4 + 3];
        out[i] = ACCUM ? (out[i] + v) : (fill + v);
    }
}

// ---- integer-exact count image ------------------------------------------------------------
template <bool AGG>
__global__ void __launch_bounds__(kThreads) count_kernel(const ImageArgs A)
{
    unsigned oob = 0;
    const int64_t tid = (int64_t)blockIdx.x * kThreads + threadIdx.x;
    const int64_t stride = (int64_t)gridDim.x * kThreads;
    const int64_t iters = (A.n + stride - 1) / stride;
    for (int64_t it = 0; it < iters; ++it) {
        const int64_t i = tid + it * stride;
        bool ok = i < A.n;
        int xi = 0, yi = 0;
        if (ok) {
            const float x = ld_stream(A.x + i), y = ld_stream(A.y + i);
            const bool keep = !A.clip || (!(x >= A.clipx) && !(y >= A.clipy));
            int ux, uy;
            if (!trunc_checked(x, ux) || !trunc_checked(y, uy)) { ok = false; ++oob; }
            else {
                if (!keep) { ux = 0; uy = 0; }
                if (!wrap_int_index(ux, A.W, xi) || !wrap_int_index(uy, A.H, yi)) { ok = false; ++oob; }
            }
        }
        const int64_t cell = (int64_t)yi * A.W + xi;
        if (AGG) {
            const unsigned long long key = ok ? (unsigned long long)cell : ~0ull - (threadIdx.x & 31);
            const unsigned peers = __match_any_sync(0xffffffffu, key);
            if (ok && (__ffs(peers) - 1) == (int)(threadIdx.x & 31)) red_add_u32(A.out_u32 + cell, (unsigned)__popc(peers));
        } else {
            if (ok) red_add_u32(A.out_u32 + cell, 1u);
        }
    }
    flush_oob(A.oob, oob);
}

// ---- dense-flow warp (optic_flow.py:37-44 + ATen grid_sampler bilinear/zeros/align_corners) ---
// flow [2][H][W] -> interleaved [H][W][2] = {u, v} per pixel, so that the taps of one image row are contiguous
__global__ void __launch_bounds__(256) flow_interleave_kernel(const float *__restrict__ flow, int64_t npix, float2 *__restrict__ uv)
{
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < npix; i += stride) uv[i] = make_float2(flow[i], flow[npix + i]);
}

template <bool INTERLEAVED>
__device__ __forceinline__ void flow_one(float xe, float ye, float te, const float *flow, const float2 *uv, int H, int W, float wm1,
                                         float hm1, float t0, float &xo, float &yo)
{
    // the reference normalises to [-1,1] (optic_flow.py:37-38) and grid_sample maps back
    const float gx = __fsub_rn(__fmul_rn(__fdiv_rn(xe, wm1), 2.0f), 1.0f);
    const float gy = __fsub_rn(__fmul_rn(__fdiv_rn(ye, hm1), 2.0f), 1.0f);
    const float ix = __fmul_rn(__fdiv_rn(__fadd_rn(gx, 1.0f), 2.0f), wm1);
    const float iy = __fmul_rn(__fdiv_rn(__fadd_rn(gy, 1.0f), 2.0f), hm1);
    float u = 0.0f, v = 0.0f;
    if (fabsf(ix) < 1.0e9f && fabsf(iy) < 1.0e9f) {
        const float fx = floorf(ix), fy = floorf(iy);
        const int x0 = (int)fx, y0 = (int)fy;
        const float xs = fx + 1.0f, ys = fy + 1.0f;
        const float nw = __fmul_rn(__fsub_rn(xs, ix), __fsub_rn(ys, iy));
        const float ne = __fmul_rn(__fsub_rn(ix, fx), __fsub_rn(ys, iy));
        const float sw = __fmul_rn(__fsub_rn(xs, ix), __fsub_rn(iy, fy));
        const float se = __fmul_rn(__fsub_rn(ix, fx), __fsub_rn(iy, fy));
        const float4 top = flow_row<INTERLEAVED>(flow, uv, H, W, y0, x0), bot = flow_row<INTERLEAVED>(flow, uv, H, W, y0 + 1, x0);
        // accumulation order of ATen's grid_sampler: nw, ne, sw, se
        u = __fadd_rn(u, __fmul_rn(top.x, nw)); v = __fadd_rn(v, __fmul_rn(top.y, nw));
        u = __fadd_rn(u, __fmul_rn(top.z, ne)); v = __fadd_rn(v, __fmul_rn(top.w, ne));
        u = __fadd_rn(u, __fmul_rn(bot.x, sw)); v = __fadd_rn(v, __fmul_rn(bot.y, sw));
        u = __fadd_rn(u, __fmul_rn(bot.z, se)); v = __fadd_rn(v, __fmul_rn(bot.w, se));
    }
    const float d = __fsub_rn(te, t0);
    xo = __fadd_rn(xe, __fmul_rn(u, d));
    yo = __fadd_rn(ye, __fmul_rn(v, d));
}

// VEC4: every thread takes four consecutive events with 16-byte loads / stores (the host checks the
// alignment), which also puts eight independent flow gathers in flight per thread.
template <bool INTERLEAVED, bool VEC4>
__global__ void __launch_bounds__(256) warp_flow_kernel(const float *__restrict__ x, const float *__restrict__ y,
                                                        const float *__restrict__ t, int64_t n,
                                                        const float *__restrict__ flow, const float2 *__restrict__ uv, int H, int W,
                                                        float t0, float *__restrict__ xw, float *__restrict__ yw)
{
    const float wm1 = (float)(W - 1), hm1 = (float)(H - 1);
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t scalar_from = 0;
    if (VEC4) {
        const int64_t n4 = n >> 2;
        for (int64_t q = tid; q < n4; q += stride) {
            const float4 xe = ld_stream4(x + 4 * q), ye = ld_stream4(y + 4 * q), te = ld_stream4(t + 4 * q);
            float4 xo, yo;
            flow_one<INTERLEAVED>(xe.x, ye.x, te.x, flow, uv, H, W, wm1, hm1, t0, xo.x, yo.x);
            flow_one<INTERLEAVED>(xe.y, ye.y, te.y, flow, uv, H, W, wm1, hm1, t0, xo.y, yo.y);
            flow_one<INTERLEAVED>(xe.z, ye.z, te.z, flow, uv, H, W, wm1, hm1, t0, xo.z, yo.z);
            flow_one<INTERLEAVED>(xe.w, ye.w, te.w, flow, uv, H, W, wm1, hm1, t0, xo.w, yo.w);
            __stcs(reinterpret_cast<float4 *>(xw + 4 * q), xo);
            __stcs(reinterpret_cast<float4 *>(yw + 4 * q), yo);
        }
        scalar_from = n4 << 2;
    }
    for (int64_t i = scalar_from + tid; i < n; i += stride) {
        float xo, yo;
        flow_one<INTERLEAVED>(ld_stream(x + i), ld_stream(y + i), ld_stream(t + i), flow, uv, H, W, wm1, hm1, t0, xo, yo);
        xw[i] = xo;
        yw[i] = yo;
    }
}

void launch_flow_interleave(const float *flow, int64_t npix, float2 *uv, cudaStream_t st)
{
    flow_interleave_kernel<<<grid_simple(npix, 256), 256, 0, st>>>(flow, npix, uv);
}

}  // namespace evk

extern "C" {

size_t evk_image_workspace_bytes(int Himg, int Wimg, unsigned flags)
{
    if (Himg < 1 || Wimg < 1 || !(flags & EVK_BILINEAR)) return 0;
    return (size_t)Himg * Wimg * 4 * sizeof(float);
}

int evk_image_f32(const float *x, const float *y, const float *p, int64_t n, int Himg, int Wimg, float clipx,
                  float clipy, unsigned flags, float fill, float *out, void *workspace, size_t workspace_bytes,
                  unsigned long long *oob, void *stream)
{
    using namespace evk;
    if (n < 0 || Himg < 1 || Wimg < 1 || !out || (n > 0 && (!x || !y || !p))) {
        set_error("evk_image_f32: bad arguments");
        return EVK_E_ARG;
    }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const bool bil = (flags & EVK_BILINEAR) != 0, accum = (flags & EVK_ACCUMULATE) != 0;
    if (bil && (Himg < 2 || Wimg < 2)) { set_error("evk_image_f32: bilinear needs a canvas of at least 2x2"); return EVK_E_ARG; }
    ImageArgs A{};
    A.x = x; A.y = y; A.p = p; A.n = n; A.H = Himg; A.W = Wimg;
    A.clip = (flags & EVK_CLIP) ? 1 : 0; A.clipx = clipx; A.clipy = clipy;
    A.out = out; A.oob = oob;
    unsigned variant = variant_of(flags);
    // AUTO: large nearest streams take the adaptive hot-spot kernel (it falls back to plain global
    // reductions by itself when the stream is not contended); bilinear keeps the vector-red form.
    const bool have_ws = workspace && workspace_bytes >= (size_t)Himg * Wimg * 4 * sizeof(float) && !((uintptr_t)workspace & 15);
    if (variant == EVK_VARIANT_AUTO)
        variant = (n >= ((int64_t)1 << 18)) ? EVK_VARIANT_SMEM_TILE : (bil && have_ws) ? EVK_VARIANT_VECTOR_RED : EVK_VARIANT_GLOBAL_RED;
    if (variant == EVK_VARIANT_VECTOR_RED && !bil) variant = EVK_VARIANT_GLOBAL_RED;
    if (variant == EVK_VARIANT_WARP_AGG && bil) variant = EVK_VARIANT_GLOBAL_RED;
    const int64_t npix = (int64_t)Himg * Wimg;
    const bool vec4 = ((((uintptr_t)x | (uintptr_t)y | (uintptr_t)p) & 15) == 0);
    if (variant == EVK_VARIANT_VECTOR_RED) {
        const size_t need = (size_t)Himg * Wimg * 4 * sizeof(float);
        if (!workspace || workspace_bytes < need || ((uintptr_t)workspace & 15)) {
            set_error("evk_image_f32: 16-byte aligned workspace of %zu bytes required", need);
            return EVK_E_WORKSPACE;
        }
        A.ws = static_cast<float *>(workspace);
        EVK_CUDA(cudaMemsetAsync(A.ws, 0, need, st));
        if (n > 0) {
            ProfScope prof(st);
            prof_count(1);
            if (vec4) image_scatter_kernel<ISINK_QUAD, true, true><<<grid_for(image_scatter_kernel<ISINK_QUAD, true, true>, kThreads, n, kThreads * 16), kThreads, 0, st>>>(A);
            else image_scatter_kernel<ISINK_QUAD, true, false><<<grid_for(image_scatter_kernel<ISINK_QUAD, true, false>, kThreads, n, kThreads * 16), kThreads, 0, st>>>(A);
        }
        const int g2 = grid_simple(npix, 256);
        prof_count(1);
        if (accum) image_fold_kernel<true><<<g2, 256, 0, st>>>(A.ws, out, Himg, Wimg, fill);
        else image_fold_kernel<false><<<g2, 256, 0, st>>>(A.ws, out, Himg, Wimg, fill);
    } else if (variant == EVK_VARIANT_GLOBAL_RED || variant == EVK_VARIANT_WARP_AGG) {
        if (!accum) {
            if (fill == 0.0f) EVK_CUDA(cudaMemsetAsync(out, 0, (size_t)npix * sizeof(float), st));
            else { prof_count(1); fill_kernel<<<grid_simple(npix, 256), 256, 0, st>>>(out, npix, fill); }
        }
        if (n > 0) {
            ProfScope prof(st);
            prof_count(1);
            if (bil) {
                if (vec4) image_scatter_kernel<ISINK_SCALAR, true, true><<<grid_for(image_scatter_kernel<ISINK_SCALAR, true, true>, kThreads, n, kThreads * 16), kThreads, 0, st>>>(A);
                else image_scatter_kernel<ISINK_SCALAR, true, false><<<grid_for(image_scatter_kernel<ISINK_SCALAR, true, false>, kThreads, n, kThreads * 16), kThreads, 0, st>>>(A);
            } else if (variant == EVK_VARIANT_WARP_AGG) {
                if (vec4) image_scatter_kernel<ISINK_WARPAGG, false, true><<<grid_for(image_scatter_kernel<ISINK_WARPAGG, false, true>, kThreads, n, kThreads * 16), kThreads, 0, st>>>(A);
                else image_scatter_kernel<ISINK_WARPAGG, false, false><<<grid_for(image_scatter_kernel<ISINK_WARPAGG, false, false>, kThreads, n, kThreads * 16), kThreads, 0, st>>>(A);
            } else {
                if (vec4) image_scatter_kernel<ISINK_SCALAR, false, true><<<grid_for(image_scatter_kernel<ISINK_SCALAR, false, true>, kThreads, n, kThreads * 16), kThreads, 0, st>>>(A);
                else image_scatter_kernel<ISINK_SCALAR, false, false><<<grid_for(image_scatter_kernel<ISINK_SCALAR, false, false>, kThreads, n, kThreads * 16), kThreads, 0, st>>>(A);
            }
        }
    } else if (variant == EVK_VARIANT_SMEM_TILE) {
        // explicit request = cache always on; reached through AUTO = adaptive (per-CTA contention probe)
        const int force = variant_of(flags) == EVK_VARIANT_SMEM_TILE ? 1 : 0;
        float *blocks = (bil && have_ws) ? static_cast<float *>(workspace) : nullptr;
        if (blocks) {
            EVK_CUDA(cudaMemsetAsync(blocks, 0, (size_t)npix * 4 * sizeof(float), st));
        } else if (!accum) {
            if (fill == 0.0f) EVK_CUDA(cudaMemsetAsync(out, 0, (size_t)npix * sizeof(float), st));
            else { prof_count(1); fill_kernel<<<grid_simple(npix, 256), 256, 0, st>>>(out, npix, fill); }
        }
        int rc = launch_image_hot(x, y, p, n, Himg, Wimg, A.clip, clipx, clipy, bil ? 1 : 0, force, out, blocks, nullptr, oob, st);
        if (rc) return rc;
        if (blocks) {
            const int g2 = grid_simple(npix, 256);
            prof_count(1);
            if (accum) image_fold_kernel<true><<<g2, 256, 0, st>>>(blocks, out, Himg, Wimg, fill);
            else image_fold_kernel<false><<<g2, 256, 0, st>>>(blocks, out, Himg, Wimg, fill);
        }
    } else {
        set_error("evk_image_f32: variant 0x%x not available", variant);
        return EVK_E_UNSUPPORTED;
    }
    EVK_CUDA(cudaGetLastError());
    return EVK_OK;
}

int evk_count_u32(const float *x, const float *y, int64_t n, int Himg, int Wimg, float clipx, float clipy,
                  unsigned flags, unsigned int *out, unsigned long long *oob, void *stream)
{
    using namespace evk;
    if (n < 0 || Himg < 1 || Wimg < 1 || !out || (n > 0 && (!x || !y))) { set_error("evk_count_u32: bad arguments"); return EVK_E_ARG; }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    ImageArgs A{};
    A.x = x; A.y = y; A.n = n; A.H = Himg; A.W = Wimg;
    A.clip = (flags & EVK_CLIP) ? 1 : 0; A.clipx = clipx; A.clipy = clipy;
    A.out_u32 = out; A.oob = oob;
    if (!(flags & EVK_ACCUMULATE)) EVK_CUDA(cudaMemsetAsync(out, 0, (size_t)Himg * Wimg * sizeof(unsigned), st));
    const unsigned cvariant = variant_of(flags);
    if (n > 0 && (cvariant == EVK_VARIANT_SMEM_TILE || cvariant == EVK_VARIANT_AUTO)) {
        int rc = launch_image_hot(x, y, nullptr, n, Himg, Wimg, A.clip, clipx, clipy, 2, cvariant == EVK_VARIANT_SMEM_TILE ? 1 : 0,
                                  nullptr, nullptr, out, oob, st);
        if (rc) return rc;
    } else if (n > 0) {
        ProfScope prof(st);
        prof_count(1);
        if (variant_of(flags) == EVK_VARIANT_GLOBAL_RED) count_kernel<false><<<grid_for(count_kernel<false>, kThreads, n, kThreads * 8), kThreads, 0, st>>>(A);
        else count_kernel<true><<<grid_for(count_kernel<true>, kThreads, n, kThreads * 8), kThreads, 0, st>>>(A);
    }
    EVK_CUDA(cudaGetLastError());
    return EVK_OK;
}

size_t evk_warp_flow_workspace_bytes(int H, int W)
{
    if (H < 1 || W < 1) return 0;
    return (size_t)H * W * sizeof(float2);
}

int evk_warp_flow_f32(const float *x, const float *y, const float *t, int64_t n, const float *flow, int H, int W,
                      float t0, float *xw, float *yw, void *workspace, size_t workspace_bytes, void *stream)
{
    using namespace evk;
    if (n < 0 || H < 1 || W < 1 || !flow || (n > 0 && (!x || !y || !t || !xw || !yw))) { set_error("evk_warp_flow_f32: bad arguments"); return EVK_E_ARG; }
    if (n == 0) return EVK_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int64_t npix = (int64_t)H * W;
    // with a workspace (and enough events to pay for the 8 B/pixel re-layout) the flow is interleaved first
    const bool inter = workspace && workspace_bytes >= (size_t)npix * sizeof(float2) && !((uintptr_t)workspace & 15) && n >= npix / 4;
    const bool vec = !(((uintptr_t)x | (uintptr_t)y | (uintptr_t)t | (uintptr_t)xw | (uintptr_t)yw) & 15);
    const float2 *uv = nullptr;
    if (inter) {
        prof_count(1);
        launch_flow_interleave(flow, npix, static_cast<float2 *>(workspace), st);
        uv = static_cast<const float2 *>(workspace);
    }
    prof_count(1);
#define EVK_FLOW_LAUNCH(I, V)                                                                                                  \
    warp_flow_kernel<I, V><<<grid_for(warp_flow_kernel<I, V>, 256, n, 256 * (V ? 8 : 4)), 256, 0, st>>>(x, y, t, n, flow, uv, H, W, t0, xw, yw)
    if (inter && vec) EVK_FLOW_LAUNCH(true, true);
    else if (inter) EVK_FLOW_LAUNCH(true, false);
    else if (vec) EVK_FLOW_LAUNCH(false, true);
    else EVK_FLOW_LAUNCH(false, false);
#undef EVK_FLOW_LAUNCH
    EVK_CUDA(cudaGetLastError());
    return EVK_OK;
}

}  // extern "C"
