// evk_voxel.cu -- events -> (B,H,W) voxel grid on H100.
//
// Semantics: events_to_voxel_torch, reference lib/representations/voxel_grid.py:129-153
// (per-bin weights :136-139, scatter through events_to_image_torch image.py:88-95).
//
// Design (DESIGN.md section 3):
//   * the reference makes B passes over all N events and scatters B*N values (mostly zeros);
//     an event has at most TWO non-zero temporal taps (bins floor(tau), floor(tau)+1), so one
//     pass over the events with <= 2 taps is the same sum.
//   * events are streamed once with 16-byte evict-first loads (16 B/event of HBM traffic);
//     the accumulation grid (B*H*W*4 B = 6.1 MB at 5x480x640) stays L2 resident.
//   * GLOBAL_RED variant : one red.global.add.f32 per tap straight into out[B][H][W].
//   * VECTOR_RED variant : the two temporal taps of an event are adjacent in a pixel-major
//     "quad" workspace ws[H*W][nq][4]; quad q holds bins 3q..3q+3 (neighbouring quads overlap by
//     one bin so that EVERY (b, b+1) pair lives inside one 16-byte aligned quad) and the event is
//     ONE red.global.add.v4.f32 (sm_90+ vector reduction, SASS REDG.E.ADD.F32x4).  A gather
//     epilogue folds the quads back into out[B][H][W].  Halves the number of L2 reduction
//     operations, which (not HBM) is what bounds this kernel.
#include "evk_common.cuh"

namespace evk {

struct VoxelArgs {
    const float *x, *y, *t, *p;  // SoA arrays (AoS: x is the interleaved base)
    // storage layout (LAYOUT_PACKED): int16 x, int16 y, float64 t, uint8 p (0/1), 13 B/event
    const short *px16, *py16;
    const double *pt64;
    const unsigned char *pp8;
    double t_first;  // PACKED: timestamps are made relative to this in float64, then cast to float32
    int64_t n;
    int64_t head;  // SoA vec4 layout: scalar events before the 16-byte aligned body
    float t0, dt, bm1;
    int B, H, W, nq;
    int hot_force;  // SINK_QUAD_HOT: 1 = cache always on, 0 = adaptive
    int auto_span;  // 1: t0 = t[0], dt = t[n-1] - t[0] read on the device (voxel_grid.py:133) -- no host sync
    int negpos;  // 0: weights = p.  1: two grids, [p>0] -> grid 0, [p<=0] -> grid 1 (voxel_grid.py:172-175).
                 // 2: numpy truthiness, [p!=0] -> grid 0, [p==0] -> grid 1 (voxel_grid.py:234-235)
    int clip;  // trilinear only
    float clipx, clipy;
    float *out;  // [B][H][W]
    float *ws;   // [H*W][nq][4]
    unsigned long long *oob;
    const unsigned *skip_unless;  // launch-level choice between the plain and the hot-pixel instantiation: return unless *skip_unless != 0
    const unsigned *skip_if;  // AUTO with the routed kernel in play: this kernel returns at once when *skip_if != 0 (the
                              // probe chose the routed kernel, which has already built the grid)
};

enum { SINK_SCALAR = 0, SINK_QUAD = 1, SINK_QUAD_HOT = 2 };

// evk_voxel_routed.cu: output tiles in shared memory, events routed to the owning SM through L2-resident rings
size_t voxel_routed_workspace_bytes(int B, int H, int W);
bool voxel_routed_supported(int B, int H, int W);
int launch_voxel_routed(const float *x, const float *y, const float *t, const float *p, int64_t n, int64_t head, float t0, float dt,
                        int B, int H, int W, int auto_span, float *out, void *workspace, size_t workspace_bytes,
                        unsigned long long *oob, cudaStream_t st, int probe);
const unsigned *voxel_routed_mode_flag(void *workspace, int B, int H, int W);   // device word the probe writes: 1 = routed ran
int64_t voxel_routed_min_events();

// Per-CTA write-combining cache in front of the vector reductions (SINK_QUAD_HOT): a direct-mapped
// {quad index -> float4 partial sum} table in shared memory, same idea as evk_hot.cu.  Real sensors
// have hot pixels (the reference ships remove_hot_pixels for them, event_util.py:166-187); every
// event of such a pixel hits the same two grid cells and global reductions to one address serialise
// in its L2 slice (~1.5 ns each).  Adaptive: switched on per CTA by a match.any contention probe.
constexpr int kVoxHotLog2 = 11;
constexpr int kVoxHotSlots = 1 << kVoxHotLog2;  // 8 KB keys + 32 KB values
constexpr unsigned kVoxEmpty = 0xffffffffu;

struct HotCtx {
    unsigned *keys;
    uint4 *vals;        // biased 2^22 fixed point (round 2: native ATOMS.ADD; f32 shared-memory adds are CAS loops on sm_90a)
    bool on;
};

constexpr int kVoxFixBits = 22;
constexpr unsigned kVoxBias = 0x80000000u;

__device__ __forceinline__ unsigned vox_atoms_ret(unsigned *cell, unsigned v)
{
    unsigned old;
    asm volatile("atom.relaxed.cta.shared::cta.add.u32 %0, [%1], %2;" : "=r"(old) : "r"((unsigned)__cvta_generic_to_shared(cell)), "r"(v));
    return old;
}

// two-way set-associative {quad index -> four fixed-point partial sums}; values the scale cannot carry (|v| > 1, NaN, inf)
// and quads whose set is taken go straight to L2.  A wrapped cell is carried out by the thread that wrapped it (the scheme
// of evk_cmax.cu / evk_hot.cu), so the table cannot overflow whatever the hot-pixel load.
__device__ __forceinline__ void hot_add4(const HotCtx &hc, float *ws_base, float *addr16, float4 v)
{
    if (hc.on && fabsf(v.x) <= 1.0f && fabsf(v.y) <= 1.0f && fabsf(v.z) <= 1.0f && fabsf(v.w) <= 1.0f) {
        const unsigned cell = (unsigned)((addr16 - ws_base) >> 2);
        const unsigned s0 = ((cell * 2654435761u) >> (32 - (kVoxHotLog2 - 1))) * 2u;
        int slot = -1;
        const uint2 k = *reinterpret_cast<const uint2 *>(hc.keys + s0);
        if (k.x == cell) slot = (int)s0;
        else if (k.y == cell) slot = (int)s0 + 1;
        else {
            if (k.x == kVoxEmpty) {
                const unsigned old = atomicCAS(hc.keys + s0, kVoxEmpty, cell);
                if (old == kVoxEmpty || old == cell) slot = (int)s0;
            }
            if (slot < 0) {
                const unsigned k1 = *(volatile unsigned *)(hc.keys + s0 + 1);
                if (k1 == cell) slot = (int)s0 + 1;
                else if (k1 == kVoxEmpty) {
                    const unsigned old = atomicCAS(hc.keys + s0 + 1, kVoxEmpty, cell);
                    if (old == kVoxEmpty || old == cell) slot = (int)s0 + 1;
                }
            }
        }
        if (slot >= 0) {
            unsigned *acc = reinterpret_cast<unsigned *>(&hc.vals[slot]);
            const float S = (float)(1 << kVoxFixBits);
            const float vv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const unsigned q = (unsigned)__float2int_rn(__fmul_rn(vv[j], S));
                if (q == 0u) continue;
                const unsigned old = vox_atoms_ret(acc + j, q), nw = old + q;
                if (((old ^ nw) & ~(nw ^ q)) >> 31)
                    red_add(addr16 + j, (int)q >= 0 ? (float)(1u << (32 - kVoxFixBits)) : -(float)(1u << (32 - kVoxFixBits)));
            }
            return;
        }
    }
    red_add4(addr16, v);
}
enum { LAYOUT_SOA4 = 0, LAYOUT_SOA1 = 1, LAYOUT_AOS = 2, LAYOUT_PACKED = 3 };

static inline int quads_for_bins(int B) { return B <= 1 ? 1 : (B - 1 + 2) / 3; }

// Add the temporal tap pair (value v0 at bin b0, v1 at bin b0+1) of one pixel.
template <int SINK>
__device__ __forceinline__ void add_bin_pair(const VoxelArgs &A, const HotCtx &hc, float *out, float *ws, int64_t pix, int b0,
                                             float v0, float v1)
{
    if (SINK == SINK_SCALAR) {
        const int64_t plane = (int64_t)A.H * A.W;
        if ((unsigned)b0 < (unsigned)A.B && v0 != 0.0f) red_add(out + (int64_t)b0 * plane + pix, v0);
        if ((unsigned)(b0 + 1) < (unsigned)A.B && v1 != 0.0f) red_add(out + (int64_t)(b0 + 1) * plane + pix, v1);
    } else {
        int lo = b0 < 0 ? 0 : b0;
        int hi = (b0 + 1 > A.B - 1) ? A.B - 1 : b0 + 1;
        if (lo > hi) return;
        float a = (lo == b0) ? v0 : v1;                       // value of bin lo
        float b = (lo + 1 == b0 + 1 && lo + 1 <= hi) ? v1 : 0.0f;  // value of bin lo+1
        if (a == 0.0f && b == 0.0f) return;
        int q = lo / 3;
        if (q > A.nq - 1) q = A.nq - 1;
        int s = lo - 3 * q;  // 0..3 (3 only in the clamped last quad, where b is 0)
        float4 v;
        v.x = (s == 0) ? a : 0.0f;
        v.y = (s == 1) ? a : ((s == 0) ? b : 0.0f);
        v.z = (s == 2) ? a : ((s == 1) ? b : 0.0f);
        v.w = (s == 3) ? a : ((s == 2) ? b : 0.0f);
        if (SINK == SINK_QUAD_HOT) hot_add4(hc, A.ws, ws + (pix * A.nq + q) * 4, v);
        else red_add4(ws + (pix * A.nq + q) * 4, v);
    }
}

// Rare path: non-finite tau or polarity.  Literal restatement of voxel_grid.py:138-139 for
// every bin so that NaN propagation matches (dt == 0 -> NaN in V[:, y, x]).
template <int SINK>
__device__ __noinline__ void add_all_bins_slow(const VoxelArgs &A, float *out, float *ws, int64_t pix, float tn, float p)
{
    for (int b = 0; b < A.B; ++b) {
        float w = __fsub_rn(1.0f, fabsf(__fsub_rn(tn, (float)b)));
        float wb = (w != w) ? w : (w > 0.0f ? w : 0.0f);  // torch.max(zeros, w) propagates NaN
        float v = __fmul_rn(p, wb);
        if (v == 0.0f) continue;
        if (SINK == SINK_SCALAR) {
            red_add(out + ((int64_t)b * A.H * A.W) + pix, v);
        } else {
            int q = b / 3;
            if (q > A.nq - 1) q = A.nq - 1;
            red_add(ws + (pix * A.nq + q) * 4 + (b - 3 * q), v);
        }
    }
}

// Trilinear extension, one temporal bin: the 2x2 spatial footprint of weight pw in bin b.
// Vector sink: the workspace is an array of 16-byte BLOCKS ws[B][H][W][4]; block (b,y,x) collects
// the taps TL,TR,BL,BR of every event whose footprint is anchored at (y,x), so the whole footprint
// is ONE red.global.add.v4.f32 (each pixel lives in four blocks; voxel_fold_blocks_kernel sums them).
template <int SINK>
__device__ __forceinline__ void tri_bin(const VoxelArgs &A, int b, float pw, int x0, int x1, int y0, int y1, float ox,
                                        float dx, float oy, float dy)
{
    const float wl = __fmul_rn(pw, ox), wr = __fmul_rn(pw, dx);
    const float v00 = __fmul_rn(wl, oy), v01 = __fmul_rn(wr, oy), v10 = __fmul_rn(wl, dy), v11 = __fmul_rn(wr, dy);
    if (v00 == 0.0f && v01 == 0.0f && v10 == 0.0f && v11 == 0.0f) return;
    const int64_t plane = (int64_t)b * A.H * A.W;
    if (SINK == SINK_SCALAR) {
        float *o = A.out + plane;
        if (v00 != 0.0f) red_add(o + (int64_t)y0 * A.W + x0, v00);
        if (v01 != 0.0f) red_add(o + (int64_t)y0 * A.W + x1, v01);
        if (v10 != 0.0f) red_add(o + (int64_t)y1 * A.W + x0, v10);
        if (v11 != 0.0f) red_add(o + (int64_t)y1 * A.W + x1, v11);
    } else if (x1 == x0 + 1 && y1 == y0 + 1) {
        red_add4(A.ws + (plane + (int64_t)y0 * A.W + x0) * 4, make_float4(v00, v01, v10, v11));
    } else {
        // wrapped footprint: each tap is the TL tap of its own pixel's block
        if (v00 != 0.0f) red_add(A.ws + (plane + (int64_t)y0 * A.W + x0) * 4, v00);
        if (v01 != 0.0f) red_add(A.ws + (plane + (int64_t)y0 * A.W + x1) * 4, v01);
        if (v10 != 0.0f) red_add(A.ws + (plane + (int64_t)y1 * A.W + x0) * 4, v10);
        if (v11 != 0.0f) red_add(A.ws + (plane + (int64_t)y1 * A.W + x1) * 4, v11);
    }
}

template <int SINK, bool SPATIAL_BILINEAR>
__device__ __forceinline__ void voxel_event(const VoxelArgs &A, const HotCtx &hc, float x, float y, float t, float p,
                                            unsigned &oob)
{
    // tau = (t - t0) / dt * (B-1), evaluated in exactly this order, no FMA (voxel_grid.py:134)
    const float tn = __fmul_rn(__fdiv_rn(__fsub_rn(t, A.t0), A.dt), A.bm1);
    const bool finite = (fabsf(tn) < 1.0e9f) && (fabsf(p) <= FLT_MAX);

    if (!SPATIAL_BILINEAR) {
        int xi, yi;
        if (!wrap_trunc_index(x, A.W, xi) || !wrap_trunc_index(y, A.H, yi)) { ++oob; return; }
        const int64_t pix = (int64_t)yi * A.W + xi;
        float *out = A.out, *ws = A.ws;
        if (A.negpos) {
            if (tn != tn) {
                // dt == 0 (one event, or all stamps equal): the temporal weight is NaN and the reference's
                // {0,1} polarity weight times NaN poisons the pixel in BOTH grids, every bin
                const int64_t cells = (int64_t)A.H * A.W;
                add_all_bins_slow<SINK>(A, out, ws, pix, tn, 1.0f);
                add_all_bins_slow<SINK>(A, SINK == SINK_SCALAR ? out + cells * A.B : out, SINK == SINK_SCALAR ? ws : ws + cells * A.nq * 4,
                                        pix, tn, 1.0f);
                return;
            }
            // fused neg/pos split: the event goes to exactly one of two grids with weight 1
            const bool pos = (A.negpos == 1) ? (p > 0.0f) : (p != 0.0f);
            const bool neg = (A.negpos == 1) ? (p <= 0.0f) : (p == 0.0f);
            if (!pos && !neg) return;  // NaN polarity: weight 0 in both (torch.where on NaN)
            if (neg) {
                const int64_t cells = (int64_t)A.H * A.W;
                if (SINK == SINK_SCALAR) out += cells * A.B; else ws += cells * A.nq * 4;
            }
            p = 1.0f;
        }
        if (!((fabsf(tn) < 1.0e9f) && (fabsf(p) <= FLT_MAX))) { add_all_bins_slow<SINK>(A, out, ws, pix, tn, p); return; }
        const float fl = floorf(tn);
        const float w0 = __fsub_rn(1.0f, fabsf(__fsub_rn(tn, fl)));         // bin floor(tau)
        const float w1 = __fsub_rn(1.0f, fabsf(__fsub_rn(tn, fl + 1.0f)));  // bin floor(tau)+1
        add_bin_pair<SINK>(A, hc, out, ws, pix, (int)fl, __fmul_rn(p, w0), __fmul_rn(p, w1));
    } else {
        // trilinear extension: per-bin events_to_image_torch(..., interpolation='bilinear')
        // (image.py:78-86,102-115) with the bin weight folded into the polarity.
        float m = 1.0f;
        if (A.clip) m = (x >= A.clipx ? 0.0f : 1.0f) * (y >= A.clipy ? 0.0f : 1.0f);
        const float pxf = floorf(x), pyf = floorf(y);
        const float dx = __fsub_rn(x, pxf), dy = __fsub_rn(y, pyf);
        int upx, upy, x0, x1, y0, y1;
        if (!trunc_checked(__fmul_rn(pxf, m), upx) || !trunc_checked(__fmul_rn(pyf, m), upy) ||
            !wrap_int_index(upx, A.W, x0) || !wrap_int_index(upx + 1, A.W, x1) ||
            !wrap_int_index(upy, A.H, y0) || !wrap_int_index(upy + 1, A.H, y1)) { ++oob; return; }
        if (m == 0.0f && finite) return;  // masked events only add zeros at pixel (0,0)..(1,1)
        const float ox = __fsub_rn(1.0f, dx), oy = __fsub_rn(1.0f, dy);
        if (!finite) {
            // keep NaN semantics: every bin, every tap
            for (int b = 0; b < A.B; ++b) {
                float w = __fsub_rn(1.0f, fabsf(__fsub_rn(tn, (float)b)));
                float wb = (w != w) ? w : (w > 0.0f ? w : 0.0f);
                tri_bin<SINK>(A, b, __fmul_rn(__fmul_rn(p, wb), m), x0, x1, y0, y1, ox, dx, oy, dy);
            }
            return;
        }
        const float fl = floorf(tn);
        const int b0 = (int)fl;
        const float wb0 = __fsub_rn(1.0f, fabsf(__fsub_rn(tn, fl)));
        const float wb1 = __fsub_rn(1.0f, fabsf(__fsub_rn(tn, fl + 1.0f)));
        if ((unsigned)b0 < (unsigned)A.B) tri_bin<SINK>(A, b0, __fmul_rn(__fmul_rn(p, wb0), m), x0, x1, y0, y1, ox, dx, oy, dy);
        if ((unsigned)(b0 + 1) < (unsigned)A.B) tri_bin<SINK>(A, b0 + 1, __fmul_rn(__fmul_rn(p, wb1), m), x0, x1, y0, y1, ox, dx, oy, dy);
    }
}

constexpr int kThreads = 256;
// 4 co-resident CTAs per SM (at most 64 registers): the QUAD instantiation the bench times has no spills on sm_90a and ran
// 2 % faster on H100 than with 5 (48 registers, 12-24 bytes of spills); three rarely used instantiations still spill
// 4-36 bytes, against 8-268 bytes each at 5 CTAs per SM.  DESIGN.md section 6
#ifndef EVK_VOXEL_MIN_CTAS
#define EVK_VOXEL_MIN_CTAS 4
#endif

// The event loop of the scatter kernel for one (sink, layout) combination.
template <int SINK, bool BIL, int LAYOUT>
__device__ __forceinline__ void scatter_events(const VoxelArgs &A, const HotCtx &hc, int64_t tid, int64_t stride, unsigned &oob)
{
    if (LAYOUT == LAYOUT_SOA4) {
        // 16-byte aligned body: 4 events per thread per iteration, four LDG.128 in flight
        const int64_t head = A.head;
        const int64_t n4 = (A.n - head) >> 2;
        const float *bx = A.x + head, *by = A.y + head, *bt = A.t + head, *bp = A.p + head;
        for (int64_t g = tid; g < n4; g += stride) {
            const float4 X = ld_stream4(bx + 4 * g), Y = ld_stream4(by + 4 * g);
            const float4 T = ld_stream4(bt + 4 * g), P = ld_stream4(bp + 4 * g);
            voxel_event<SINK, BIL>(A, hc, X.x, Y.x, T.x, P.x, oob);
            voxel_event<SINK, BIL>(A, hc, X.y, Y.y, T.y, P.y, oob);
            voxel_event<SINK, BIL>(A, hc, X.z, Y.z, T.z, P.z, oob);
            voxel_event<SINK, BIL>(A, hc, X.w, Y.w, T.w, P.w, oob);
        }
        // scalar head [0, head) and tail [head + 4*n4, n)
        const int64_t tail0 = head + 4 * n4;
        const int64_t nrest = head + (A.n - tail0);
        for (int64_t i = tid; i < nrest; i += stride) {
            const int64_t j = (i < head) ? i : tail0 + (i - head);
            voxel_event<SINK, BIL>(A, hc, ld_stream(A.x + j), ld_stream(A.y + j), ld_stream(A.t + j), ld_stream(A.p + j), oob);
        }
    } else if (LAYOUT == LAYOUT_SOA1) {
        // arbitrary 4-byte alignment: coalesced scalar loads, 4 independent events in flight
        int64_t i = tid;
        for (; i + 3 * stride < A.n; i += 4 * stride) {
            float xs[4], ys[4], ts[4], ps[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                xs[k] = ld_stream(A.x + i + k * stride); ys[k] = ld_stream(A.y + i + k * stride);
                ts[k] = ld_stream(A.t + i + k * stride); ps[k] = ld_stream(A.p + i + k * stride);
            }
#pragma unroll
            for (int k = 0; k < 4; ++k) voxel_event<SINK, BIL>(A, hc, xs[k], ys[k], ts[k], ps[k], oob);
        }
        for (; i < A.n; i += stride)
            voxel_event<SINK, BIL>(A, hc, ld_stream(A.x + i), ld_stream(A.y + i), ld_stream(A.t + i), ld_stream(A.p + i), oob);
    } else if (LAYOUT == LAYOUT_PACKED) {
        // the on-disk layout of the reference's HDF5 / memmap formats (event_packagers.py:90-93,
        // h5_to_memmap.py:115-117): int16 x, int16 y, float64 t, bool / uint8 p, with the loader's
        // polarity map p*2-1 (hdf5_dataset.py:22) and the stamps made relative in float64 before the
        // float32 cast.  13 B/event instead of 16, and no host-side casts.
        for (int64_t i = tid; i < A.n; i += stride) {
            const float ex = (float)__ldcs(A.px16 + i), ey = (float)__ldcs(A.py16 + i);
            const float et = (float)(__ldcs(A.pt64 + i) - A.t_first);
            const float ep = __ldcs(A.pp8 + i) ? 1.0f : -1.0f;
            voxel_event<SINK, BIL>(A, hc, ex, ey, et, ep, oob);
        }
    } else {
        // AoS: one 16-byte [x,y,t,p] record per event
        int64_t i = tid;
        for (; i + 3 * stride < A.n; i += 4 * stride) {
            float4 e[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) e[k] = ld_stream4(A.x + 4 * (i + k * stride));
#pragma unroll
            for (int k = 0; k < 4; ++k) voxel_event<SINK, BIL>(A, hc, e[k].x, e[k].y, e[k].z, e[k].w, oob);
        }
        for (; i < A.n; i += stride) {
            const float4 e = ld_stream4(A.x + 4 * i);
            voxel_event<SINK, BIL>(A, hc, e.x, e.y, e.z, e.w, oob);
        }
    }
}

template <int SINK, bool BIL, int LAYOUT>
__global__ void __launch_bounds__(kThreads, EVK_VOXEL_MIN_CTAS) voxel_scatter_kernel(const VoxelArgs A_in)
{
    if (A_in.skip_if && *A_in.skip_if) return;
    if (A_in.skip_unless && !*A_in.skip_unless) return;
    VoxelArgs A = A_in;
    if (A.auto_span && A.n > 0) {
        // first / last timestamp straight from the (time-sorted) stream; AoS keeps t at offset 2
        const float first = (LAYOUT == LAYOUT_PACKED) ? 0.0f : (LAYOUT == LAYOUT_AOS) ? A.x[2] : A.t[0];
        const float last = (LAYOUT == LAYOUT_PACKED) ? (float)(A.pt64[A.n - 1] - A.pt64[0])
                           : (LAYOUT == LAYOUT_AOS)  ? A.x[4 * (A.n - 1) + 2] : A.t[A.n - 1];
        if (LAYOUT == LAYOUT_PACKED) A.t_first = A.pt64[0];
        A.t0 = first;
        A.dt = __fsub_rn(last, first);
    }
    unsigned oob = 0;
    const int64_t tid = (int64_t)blockIdx.x * kThreads + threadIdx.x;
    const int64_t stride = (int64_t)gridDim.x * kThreads;

    // write-combining cache (SINK_QUAD_HOT only; the arrays vanish from the other instantiations)
    __shared__ unsigned hot_keys[SINK == SINK_QUAD_HOT ? kVoxHotSlots : 1];
    __shared__ uint4 hot_vals[SINK == SINK_QUAD_HOT ? kVoxHotSlots : 1];
    HotCtx hc{hot_keys, hot_vals, false};
    if (SINK == SINK_QUAD_HOT) {
        hc.on = A.hot_force != 0;
        if (!hc.on) {
            // contention probe: lanes whose first event shares its pixel with another lane of the warp,
            // counted over the CTA by the barrier itself (one __syncthreads_count, no shared-memory traffic)
            unsigned long long key = ~0ull - (threadIdx.x & 31);
            if (tid < A.n) {
                const float ex = (LAYOUT == LAYOUT_PACKED) ? (float)A.px16[tid] : (LAYOUT == LAYOUT_AOS) ? A.x[4 * tid] : A.x[tid];
                const float ey = (LAYOUT == LAYOUT_PACKED) ? (float)A.py16[tid] : (LAYOUT == LAYOUT_AOS) ? A.x[4 * tid + 1] : A.y[tid];
                int ux, uy;
                if (trunc_checked(ex, ux) && trunc_checked(ey, uy)) key = ((unsigned long long)(unsigned)uy << 32) | (unsigned)ux;
            }
            const int hot_dups = __syncthreads_count(__popc(__match_any_sync(0xffffffffu, key)) > 1);
            hc.on = hot_dups * 64 > kThreads;  // > 4 of 256 lanes collide inside their warp (uniform streams: ~0.03)
        }
        if (hc.on) {   // the table is only initialised (40 KB of stores) by CTAs that will use it
            for (int s = threadIdx.x; s < kVoxHotSlots; s += kThreads) { hot_keys[s] = kVoxEmpty; hot_vals[s] = make_uint4(kVoxBias, kVoxBias, kVoxBias, kVoxBias); }
            __syncthreads();
        }
    }

    // the adaptive kernel runs the PLAIN vector-red loop when its cache is off, so an uncontended stream
    // executes exactly the instructions of the non-adaptive kernel
    if (SINK == SINK_QUAD_HOT && !hc.on) scatter_events<SINK_QUAD, BIL, LAYOUT>(A, hc, tid, stride, oob);
    else scatter_events<SINK, BIL, LAYOUT>(A, hc, tid, stride, oob);
    if (SINK == SINK_QUAD_HOT) {
        __syncthreads();
        if (hc.on)
            for (int s = threadIdx.x; s < kVoxHotSlots; s += kThreads) {
                const unsigned k = hot_keys[s];
                if (k == kVoxEmpty) continue;
                const uint4 u = hot_vals[s];
                const float inv = 1.0f / (float)(1 << kVoxFixBits);
                const float4 v = make_float4(__fmul_rn((float)(int)(u.x - kVoxBias), inv), __fmul_rn((float)(int)(u.y - kVoxBias), inv),
                                             __fmul_rn((float)(int)(u.z - kVoxBias), inv), __fmul_rn((float)(int)(u.w - kVoxBias), inv));
                if (v.x != 0.0f || v.y != 0.0f || v.z != 0.0f || v.w != 0.0f) red_add4(A.ws + (size_t)k * 4, v);
            }
    }
    flush_oob(A.oob, oob);
}

// quad workspace -> out[B][H][W]; bin b lives in quad b/3 (slot b%3) and, when b%3==0 and b>0,
// also in quad b/3-1 (slot 3).
template <bool ACCUM>
__global__ void __launch_bounds__(256) voxel_fold_kernel(const float *__restrict__ ws, float *__restrict__ out,
                                                         int64_t npix, int B, int nq, const unsigned *skip_if = nullptr)
{
    if (skip_if && *skip_if) return;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t pix = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; pix < npix; pix += stride) {
        const float4 *src = reinterpret_cast<const float4 *>(ws) + pix * nq;
        float4 prev = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int q = 0; q < nq; ++q) {
            const float4 cur = src[q];
            const float vals[4] = {cur.x, cur.y, cur.z, cur.w};
#pragma unroll
            for (int s = 0; s < 4; ++s) {
                const int b = 3 * q + s;
                if (b >= B) break;
                const bool shared_with_next = (s == 3) && (q + 1 < nq);
                if (shared_with_next) continue;  // emitted by the next quad (slot 0) together with this slot 3
                float v = vals[s];
                if (s == 0 && q > 0) v += prev.w;
                float *o = out + (int64_t)b * npix + pix;
                *o = ACCUM ? (*o + v) : v;
            }
            prev = cur;
        }
    }
}

// Fused fold + all-reduce over NVLink peer memory (one process per GPU, every rank launches this
// kernel on its own slice): rank r owns the pixels [pix_lo, pix_hi); for each of them it reads the
// temporal quads of EVERY rank's workspace (16-byte peer loads, coalesced), sums them in rank order,
// folds the overlapping quads into the B bins and stores the result into EVERY rank's output grid
// (coalesced peer stores).  No intermediate partial grid, no NCCL; every cell is computed once, so all
// ranks end up with bit-identical grids.  The caller separates it from the scatters before and the
// readers after by a cross-GPU barrier (symmetric-memory signal pads).
constexpr int kMaxPeers = 16;
struct VoxelPeers {
    const float4 *ws[kMaxPeers];
    float *out[kMaxPeers];
};

// WORLD > 0: compile-time peer count (the peer loads of a pixel are all issued before the first add);
// WORLD == 0: run-time count.  NQ likewise (2 quads = the 5-bin grid of the data loaders).
template <int WORLD, int NQ>
__global__ void __launch_bounds__(256) voxel_fold_allreduce_kernel(const VoxelPeers P, int world_rt, int64_t pix_lo, int64_t pix_hi,
                                                                   int64_t npix, int B, int nq_rt)
{
    const int world = WORLD ? WORLD : world_rt;
    const int nq = NQ ? NQ : nq_rt;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t pix = pix_lo + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; pix < pix_hi; pix += stride) {
        float4 prev = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int q = 0; q < nq; ++q) {
            float4 part[WORLD ? WORLD : 1];
            float4 cur;
            if (WORLD) {
#pragma unroll
                for (int r = 0; r < WORLD; ++r) part[r] = __ldcg(P.ws[r] + pix * nq + q);
                cur = part[0];
#pragma unroll
                for (int r = 1; r < WORLD; ++r) { cur.x += part[r].x; cur.y += part[r].y; cur.z += part[r].z; cur.w += part[r].w; }
            } else {
                cur = __ldcg(P.ws[0] + pix * nq + q);
                for (int r = 1; r < world; ++r) {
                    const float4 o = __ldcg(P.ws[r] + pix * nq + q);
                    cur.x += o.x; cur.y += o.y; cur.z += o.z; cur.w += o.w;
                }
            }
            const float vals[4] = {cur.x, cur.y, cur.z, cur.w};
#pragma unroll
            for (int s = 0; s < 4; ++s) {
                const int b = 3 * q + s;
                if (b >= B) break;
                if (s == 3 && q + 1 < nq) continue;  // emitted with slot 0 of the next quad
                float v = vals[s];
                if (s == 0 && q > 0) v += prev.w;
#pragma unroll
                for (int r = 0; r < world; ++r) __stcg(P.out[r] + (int64_t)b * npix + pix, v);
            }
            prev = cur;
        }
    }
}

// The same step through the NVSwitch (NVLS): `ws_mc` / `out_mc` are MULTICAST addresses bound to every
// rank's workspace / grid.  One multimem.ld_reduce returns the sum of a quad over all ranks (the switch
// reduces, one 16-byte response crosses this GPU's link instead of N-1), one multimem.st writes a bin value
// into every rank's grid.  Per GPU: 9.8 MB / N in, 6.1 MB / N out at 5x480x640, whatever N is.
__device__ __forceinline__ float4 multimem_ld_reduce_add4(const float4 *mc)
{
    float4 v;
    asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0, %1, %2, %3}, [%4];"
                 : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(mc) : "memory");
    return v;
}

__device__ __forceinline__ void multimem_st(float *mc, float v)
{
    asm volatile("multimem.st.relaxed.sys.global.f32 [%0], %1;" ::"l"(mc), "f"(v) : "memory");
}

__global__ void __launch_bounds__(128) voxel_fold_allreduce_nvls_kernel(const float4 *__restrict__ ws_mc, float *__restrict__ out_mc,
                                                                        int64_t pix_lo, int64_t pix_hi, int64_t npix, int B, int nq)
{
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t pix = pix_lo + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; pix < pix_hi; pix += stride) {
        float4 prev = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int q = 0; q < nq; ++q) {
            const float4 cur = multimem_ld_reduce_add4(ws_mc + pix * nq + q);
            const float vals[4] = {cur.x, cur.y, cur.z, cur.w};
#pragma unroll
            for (int s = 0; s < 4; ++s) {
                const int b = 3 * q + s;
                if (b >= B) break;
                if (s == 3 && q + 1 < nq) continue;  // emitted with slot 0 of the next quad
                float v = vals[s];
                if (s == 0 && q > 0) v += prev.w;
                multimem_st(out_mc + (int64_t)b * npix + pix, v);
            }
            prev = cur;
        }
    }
}

// Batched windows: CTA (w, s) scatters slice s of window w into out[w] with that window's own
// t0 / dt (voxel_grid.py:133-134 applied per window, as voxel_grids_fixed_n_torch :53-56 does).
__global__ void __launch_bounds__(kThreads) voxel_windows_kernel(const VoxelArgs A, const int64_t *__restrict__ offsets,
                                                                 int n_windows, int slices, int pairs)
{
    unsigned oob = 0;
    const int w = blockIdx.x / slices, s = blockIdx.x - w * slices;
    if (w < n_windows) {
        const int64_t first = pairs ? offsets[2 * w] : offsets[w], last = pairs ? offsets[2 * w + 1] : offsets[w + 1];
        if (last > first) {
            VoxelArgs Aw = A;
            Aw.t0 = A.t[first];
            Aw.dt = __fsub_rn(A.t[last - 1], Aw.t0);
            Aw.out = A.out + (int64_t)w * A.B * A.H * A.W * (A.negpos ? 2 : 1);
            for (int64_t i = first + (int64_t)s * kThreads + threadIdx.x; i < last; i += (int64_t)slices * kThreads)
                voxel_event<SINK_SCALAR, false>(Aw, HotCtx{nullptr, nullptr, false}, A.x[i], A.y[i], A.t[i], A.p[i], oob);
        }
    }
    flush_oob(A.oob, oob);
}

// block workspace ws[B][H][W][4] -> out[B][H][W]: pixel (y,x) = TL of block (y,x) + TR of (y,x-1)
// + BL of (y-1,x) + BR of (y-1,x-1)
template <bool ACCUM>
__global__ void __launch_bounds__(256) voxel_fold_blocks_kernel(const float *__restrict__ ws, float *__restrict__ out,
                                                                int B, int H, int W)
{
    const int64_t total = (int64_t)B * H * W;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) {
        const int x = (int)(i % W), y = (int)((i / W) % H);
        float v = ws[i * 4];
        if (x > 0) v += ws[(i - 1) * 4 + 1];
        if (y > 0) v += ws[(i - W) * 4 + 2];
        if (x > 0 && y > 0) v += ws[(i - W - 1) * 4 + 3];
        out[i] = ACCUM ? (out[i] + v) : v;
    }
}

// Launch-level contention probe (one CTA): 1024 events at a stride through the whole stream; a lane is "contended" when
// another lane of its warp samples the same pixel.  Uniform streams over >= 1e4 pixels: ~0.1 % of the lanes; one hot pixel
// with 1 % of the events: ~25 %.  The verdict picks between the plain vector-reduction kernel and the one with the
// shared-memory hot-pixel table -- as two launches of which one returns at once -- because the table's 40 KB of static
// shared memory and its registers slow the plain event loop down when both live in one kernel.
template <int LAYOUT>
__global__ void __launch_bounds__(1024) voxel_hot_probe_kernel(const VoxelArgs A, unsigned *verdict)
{
    int dup = 0;
    {   // one sample per thread (one round of dependent HBM latency: the probe sits in front of the scatter kernel)
        const int64_t k = threadIdx.x;
        unsigned long long key = ~0ull - (unsigned long long)(threadIdx.x & 31);
        const int64_t j = (A.n >= 1024) ? k * (A.n / 1024) : k;
        if (j < A.n) {
            const float ex = (LAYOUT == LAYOUT_PACKED) ? (float)A.px16[j] : (LAYOUT == LAYOUT_AOS) ? A.x[4 * j] : A.x[j];
            const float ey = (LAYOUT == LAYOUT_PACKED) ? (float)A.py16[j] : (LAYOUT == LAYOUT_AOS) ? A.x[4 * j + 1] : A.y[j];
            int ux, uy;
            if (trunc_checked(ex, ux) && trunc_checked(ey, uy)) key = ((unsigned long long)(unsigned)uy << 32) | (unsigned)ux;
        }
        if (__popc(__match_any_sync(0xffffffffu, key)) > 1) ++dup;
    }
    const int dup_all = __syncthreads_count(dup > 0);
    if (threadIdx.x == 0) *verdict = (dup_all * 64 > 1024) ? 1u : 0u;
}

static int launch_voxel(const VoxelArgs &A0, unsigned flags, int layout, cudaStream_t st,
                        void *workspace, size_t workspace_bytes)
{
    VoxelArgs A = A0;
    const int grids = A.negpos ? 2 : 1;  // neg/pos mode writes out[2][B][H][W]
    const bool bil = (flags & EVK_BILINEAR) != 0;
    const bool accum = (flags & EVK_ACCUMULATE) != 0;
    const int64_t npix = (int64_t)A.H * A.W;
    unsigned variant = variant_of(flags);
    // AUTO: big streams take the vector-red path with the adaptive hot-pixel cache; small ones the
    // scalar path (no workspace, no fold).  SMEM_TILE forces the cache on, VECTOR_RED leaves it out.
    bool hot = false;
    bool routed_probe = false;
    if (variant == EVK_VARIANT_AUTO) {
        variant = (A.n >= (int64_t)1 << 20 && workspace != nullptr) ? EVK_VARIANT_VECTOR_RED : EVK_VARIANT_GLOBAL_RED;
        hot = variant == EVK_VARIANT_VECTOR_RED && !bil;
        // large plain streams: a probe looks at a sample of the events on the device and picks the routed kernel (unit
        // polarities, no hot pixels) or the vector-reduction kernel below; the one not chosen returns at once
        routed_probe = A.n >= voxel_routed_min_events() && !bil && !A.negpos && !(flags & EVK_NO_FOLD) && !accum && layout == LAYOUT_SOA4 &&
                       voxel_routed_supported(A.B, A.H, A.W) && workspace != nullptr &&
                       workspace_bytes >= voxel_routed_workspace_bytes(A.B, A.H, A.W) + (size_t)npix * quads_for_bins(A.B) * 16;
    } else if (variant == EVK_VARIANT_SMEM_TILE && !bil) {
        variant = EVK_VARIANT_VECTOR_RED;
        hot = true;
        A.hot_force = 1;
    }
    const bool no_fold = (flags & EVK_NO_FOLD) != 0;
    if (variant == EVK_VARIANT_ROUTED &&
        (bil || A.negpos || no_fold || layout != LAYOUT_SOA4 || !voxel_routed_supported(A.B, A.H, A.W) ||
         workspace == nullptr || workspace_bytes < voxel_routed_workspace_bytes(A.B, A.H, A.W))) {
        // the routed kernel covers the plain (nearest, combined) grid on f32 SoA arrays with a common alignment whose
        // B*H*W/SMs cells fit in shared memory; everything else takes the automatic choice
        variant = (A.n >= (int64_t)1 << 20 && workspace != nullptr) ? EVK_VARIANT_VECTOR_RED : EVK_VARIANT_GLOBAL_RED;
        hot = variant == EVK_VARIANT_VECTOR_RED && !bil;
    }
    if (variant == EVK_VARIANT_ROUTED) {
        if (!accum) EVK_CUDA(cudaMemsetAsync(A.out, 0, (size_t)npix * A.B * sizeof(float), st));
        if (A.n == 0) return EVK_OK;
        return launch_voxel_routed(A.x, A.y, A.t, A.p, A.n, A.head, A.t0, A.dt, A.B, A.H, A.W, A.auto_span, A.out, workspace,
                                   workspace_bytes, A.oob, st, 0);
    }
    if (no_fold) {
        // the caller folds (and reduces across GPUs) itself: the sums stay in the quad workspace
        if (bil || A.negpos || workspace == nullptr) { set_error("evk_voxel: EVK_NO_FOLD needs a workspace and the plain (nearest, combined) grid"); return EVK_E_UNSUPPORTED; }
        if (variant == EVK_VARIANT_GLOBAL_RED) variant = EVK_VARIANT_VECTOR_RED;
    }
    if ((uint64_t)npix * quads_for_bins(A.B) * (A.negpos ? 2 : 1) >= 0xffffffffull) hot = false;  // 32-bit quad ids
    if (variant != EVK_VARIANT_VECTOR_RED && variant != EVK_VARIANT_GLOBAL_RED) {
        set_error("evk_voxel: variant 0x%x not available for this entry point", variant);
        return EVK_E_UNSUPPORTED;
    }
    // probe mode: ONE timed scope for "probe + the kernel it selects" (the inner scopes of the two alternatives nest in it)
    struct OptScope { ProfScope *p = nullptr; ~OptScope() { delete p; } } outer;
    if (routed_probe) {
        outer.p = new ProfScope(st);
        // the routed kernel's rings come first in the workspace, the quad workspace of the fallback after them
        EVK_CUDA(cudaMemsetAsync(A.out, 0, (size_t)npix * A.B * sizeof(float), st));
        int rc = launch_voxel_routed(A.x, A.y, A.t, A.p, A.n, A.head, A.t0, A.dt, A.B, A.H, A.W, A.auto_span, A.out, workspace,
                                     workspace_bytes, A.oob, st, 1);
        if (rc) return rc;
        A.skip_if = voxel_routed_mode_flag(workspace, A.B, A.H, A.W);
        const size_t roff = (voxel_routed_workspace_bytes(A.B, A.H, A.W) + 255) & ~(size_t)255;
        workspace = static_cast<char *>(workspace) + roff;
        workspace_bytes -= roff;
    }
    const int sink = (variant == EVK_VARIANT_VECTOR_RED) ? SINK_QUAD : SINK_SCALAR;
    A.nq = quads_for_bins(A.B);
    unsigned *hot_flag = nullptr;      // device word for the launch-level contention verdict (room behind the quad workspace)
    if (sink == SINK_QUAD) {
        const size_t need = (bil ? (size_t)npix * A.B * 4 * sizeof(float) : (size_t)npix * A.nq * 4 * sizeof(float)) * grids;
        if (workspace == nullptr || workspace_bytes < need) {
            set_error("evk_voxel: workspace of %zu bytes required, %zu given", need, workspace_bytes);
            return EVK_E_WORKSPACE;
        }
        if (((uintptr_t)workspace & 15) != 0) { set_error("evk_voxel: workspace must be 16-byte aligned"); return EVK_E_ARG; }
        A.ws = static_cast<float *>(workspace);
        EVK_CUDA(cudaMemsetAsync(A.ws, 0, need, st));
        const size_t flag_off = (need + 255) & ~(size_t)255;
        if (workspace_bytes >= flag_off + 256 && !A.skip_if) hot_flag = reinterpret_cast<unsigned *>(static_cast<char *>(workspace) + flag_off);
    } else if (!accum) {
        EVK_CUDA(cudaMemsetAsync(A.out, 0, (size_t)npix * A.B * sizeof(float) * grids, st));
    }
    if (A.n > 0) {
        const int per_thread = (layout == LAYOUT_SOA4) ? 4 : 1;
#define EVK_LAUNCH(S, BL, L)                                                                                   \
    voxel_scatter_kernel<S, BL, L><<<grid_for(voxel_scatter_kernel<S, BL, L>, kThreads, A.n, kThreads * per_thread * 4), \
                                     kThreads, 0, st>>>(A)
#define EVK_DISPATCH_L(S, BL)                                  \
    do {                                                       \
        if (layout == LAYOUT_SOA4) EVK_LAUNCH(S, BL, LAYOUT_SOA4); \
        else if (layout == LAYOUT_SOA1) EVK_LAUNCH(S, BL, LAYOUT_SOA1); \
        else if (layout == LAYOUT_PACKED) EVK_LAUNCH(S, BL, LAYOUT_PACKED); \
        else EVK_LAUNCH(S, BL, LAYOUT_AOS);                    \
    } while (0)
        {
            ProfScope prof(st);
            prof_count(1);
            if (sink == SINK_QUAD && hot && !A.hot_force && hot_flag != nullptr) {
                // adaptive, decided once per launch on the device: probe, then both instantiations -- one returns at once
                prof_count(2);
                if (layout == LAYOUT_SOA4 || layout == LAYOUT_SOA1) voxel_hot_probe_kernel<LAYOUT_SOA1><<<1, 1024, 0, st>>>(A, hot_flag);
                else if (layout == LAYOUT_PACKED) voxel_hot_probe_kernel<LAYOUT_PACKED><<<1, 1024, 0, st>>>(A, hot_flag);
                else voxel_hot_probe_kernel<LAYOUT_AOS><<<1, 1024, 0, st>>>(A, hot_flag);
                const unsigned *outer_skip = A.skip_if;
                A.skip_if = hot_flag;                          // plain kernel: unless the probe found contention
                EVK_DISPATCH_L(SINK_QUAD, false);
                A.skip_if = outer_skip;
                A.skip_unless = hot_flag;                      // table kernel: only if it did
                A.hot_force = 1;
                EVK_DISPATCH_L(SINK_QUAD_HOT, false);
                A.skip_unless = nullptr;
                A.hot_force = 0;
            } else if (sink == SINK_QUAD && hot) EVK_DISPATCH_L(SINK_QUAD_HOT, false);
            else if (sink == SINK_QUAD) { if (bil) EVK_DISPATCH_L(SINK_QUAD, true); else EVK_DISPATCH_L(SINK_QUAD, false); }
            else { if (bil) EVK_DISPATCH_L(SINK_SCALAR, true); else EVK_DISPATCH_L(SINK_SCALAR, false); }
        }
#undef EVK_DISPATCH_L
#undef EVK_LAUNCH
        EVK_CUDA(cudaGetLastError());
    }
    delete outer.p;
    outer.p = nullptr;
    if (sink == SINK_QUAD && !no_fold) {
        const int grid = grid_simple(npix, 256);
        prof_count(1);
        if (bil) {
            if (accum) voxel_fold_blocks_kernel<true><<<grid, 256, 0, st>>>(A.ws, A.out, A.B, A.H, A.W);
            else voxel_fold_blocks_kernel<false><<<grid, 256, 0, st>>>(A.ws, A.out, A.B, A.H, A.W);
        } else {
            for (int g = 0; g < grids; ++g) {
                const float *wsg = A.ws + (size_t)g * npix * A.nq * 4;
                float *og = A.out + (size_t)g * npix * A.B;
                if (g) prof_count(1);
                if (accum) voxel_fold_kernel<true><<<grid, 256, 0, st>>>(wsg, og, npix, A.B, A.nq, A.skip_if);
                else voxel_fold_kernel<false><<<grid, 256, 0, st>>>(wsg, og, npix, A.B, A.nq, A.skip_if);
            }
        }
        EVK_CUDA(cudaGetLastError());
    }
    return EVK_OK;
}

static int check_common(int64_t n, int B, int H, int W, const void *out)
{
    if (n < 0 || B < 1 || H < 1 || W < 1 || out == nullptr) {
        set_error("evk_voxel: bad arguments (n=%lld B=%d H=%d W=%d out=%p)", (long long)n, B, H, W, out);
        return EVK_E_ARG;
    }
    if ((int64_t)B * H * W >= ((int64_t)1 << 40)) { set_error("evk_voxel: grid too large"); return EVK_E_ARG; }
    return EVK_OK;
}

}  // namespace evk

extern "C" {

size_t evk_voxel_workspace_bytes(int B, int H, int W, unsigned flags)
{
    if (B < 1 || H < 1 || W < 1) return 0;
    if (flags & EVK_BILINEAR) return (size_t)B * H * W * 4 * sizeof(float);   // 2x2 blocks per bin
    size_t need = (size_t)H * W * evk::quads_for_bins(B) * 4 * sizeof(float);      // temporal quads per pixel
    need = ((need + 255) & ~(size_t)255) + 256;                                    // + the launch-level contention verdict
    const unsigned v = evk::variant_of(flags);
    if ((v == EVK_VARIANT_AUTO || v == EVK_VARIANT_ROUTED) && evk::voxel_routed_supported(B, H, W)) {
        // the routed kernel's rings, followed (AUTO) by the quad workspace of the kernel the probe may choose instead
        const size_t r = (evk::voxel_routed_workspace_bytes(B, H, W) + 255) & ~(size_t)255;
        need = (v == EVK_VARIANT_AUTO) ? r + need : (r > need ? r : need);
    }
    return need;
}

int evk_voxel_f32(const float *x, const float *y, const float *t, const float *p, int64_t n, float t0,
                  float dt, int B, int H, int W, unsigned flags, float *out, void *workspace,
                  size_t workspace_bytes, unsigned long long *oob, void *stream)
{
    using namespace evk;
    int rc = check_common(n, B, H, W, (flags & EVK_NO_FOLD) ? static_cast<const void *>(&rc) : out);
    if (rc) return rc;
    if (n > 0 && (!x || !y || !t || !p)) { set_error("evk_voxel_f32: null event array"); return EVK_E_ARG; }
    VoxelArgs A{};
    A.x = x; A.y = y; A.t = t; A.p = p; A.n = n;
    A.t0 = t0; A.dt = dt; A.bm1 = (float)(B - 1);
    A.B = B; A.H = H; A.W = W;
    A.clip = (flags & EVK_CLIP) ? 1 : 0;
    A.clipx = (float)(W - 1); A.clipy = (float)(H - 1);
    A.auto_span = (flags & EVK_AUTO_SPAN) ? 1 : 0;
    A.out = out; A.oob = oob;
    // choose the load layout: 16-byte body if all four arrays share their misalignment
    const uintptr_t ax = (uintptr_t)x & 15, ay = (uintptr_t)y & 15, at = (uintptr_t)t & 15, ap = (uintptr_t)p & 15;
    int layout = LAYOUT_SOA1;
    if (ax == ay && ay == at && at == ap && (ax & 3) == 0) {
        layout = LAYOUT_SOA4;
        A.head = ((16 - ax) & 15) >> 2;
        if (A.head > n) A.head = n;
    }
    return launch_voxel(A, flags, layout, static_cast<cudaStream_t>(stream), workspace, workspace_bytes);
}

int evk_voxel_aos_f32(const float *ev, int64_t n, float t0, float dt, int B, int H, int W, unsigned flags,
                      float *out, void *workspace, size_t workspace_bytes, unsigned long long *oob,
                      void *stream)
{
    using namespace evk;
    int rc = check_common(n, B, H, W, out);
    if (rc) return rc;
    if (n > 0 && (!ev || ((uintptr_t)ev & 15))) { set_error("evk_voxel_aos_f32: ev must be a 16-byte aligned device pointer"); return EVK_E_ARG; }
    VoxelArgs A{};
    A.x = ev; A.n = n;
    A.t0 = t0; A.dt = dt; A.bm1 = (float)(B - 1);
    A.B = B; A.H = H; A.W = W;
    A.clip = (flags & EVK_CLIP) ? 1 : 0;
    A.clipx = (float)(W - 1); A.clipy = (float)(H - 1);
    A.auto_span = (flags & EVK_AUTO_SPAN) ? 1 : 0;
    A.out = out; A.oob = oob;
    return launch_voxel(A, flags, LAYOUT_AOS, static_cast<cudaStream_t>(stream), workspace, workspace_bytes);
}

int evk_voxel_windows_f32(const float *x, const float *y, const float *t, const float *p, const int64_t *offsets,
                          int n_windows, int64_t n_events_hint, int B, int H, int W, unsigned flags, float *out,
                          unsigned long long *oob, void *stream)
{
    using namespace evk;
    if (n_windows < 0 || B < 1 || H < 1 || W < 1 || !out || (n_windows > 0 && (!x || !y || !t || !p || !offsets))) {
        set_error("evk_voxel_windows_f32: bad arguments");
        return EVK_E_ARG;
    }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int grids = (flags & EVK_WINDOW_NEGPOS) ? 2 : 1;
    if (!(flags & EVK_ACCUMULATE))
        EVK_CUDA(cudaMemsetAsync(out, 0, (size_t)n_windows * grids * B * H * W * sizeof(float), st));
    if (n_windows == 0) return EVK_OK;
    VoxelArgs A{};
    A.x = x; A.y = y; A.t = t; A.p = p;
    A.negpos = grids == 2 ? ((flags & EVK_NEGPOS_TRUTHY) ? 2 : 1) : 0;
    A.bm1 = (float)(B - 1);
    A.B = B; A.H = H; A.W = W; A.nq = quads_for_bins(B);
    A.out = out; A.oob = oob;
    // slices per window: enough CTAs to fill the machine, at most one slice per 2K events
    int64_t per = n_events_hint > 0 ? n_events_hint / n_windows : 8192;
    int64_t slices = (per + 2047) / 2048;
    const int64_t fill = ((int64_t)num_sms() * 8 + n_windows - 1) / n_windows;
    if (slices > fill) slices = fill;
    if (slices < 1) slices = 1;
    if ((int64_t)n_windows * slices > 0x7fffffffLL) { set_error("evk_voxel_windows_f32: too many windows"); return EVK_E_ARG; }
    {
        ProfScope prof(st);
        prof_count(1);
        voxel_windows_kernel<<<(unsigned)(n_windows * slices), kThreads, 0, st>>>(A, offsets, n_windows, (int)slices,
                                                                                  (flags & EVK_WINDOW_PAIRS) ? 1 : 0);
    }
    EVK_CUDA(cudaGetLastError());
    return EVK_OK;
}

int evk_voxel_fold_allreduce_f32(const void *const *peer_workspaces, float *const *peer_outs, int world, int rank, int B, int H,
                                 int W, unsigned flags, void *stream)
{
    using namespace evk;
    if (world < 1 || world > kMaxPeers || rank < 0 || rank >= world || B < 1 || H < 1 || W < 1 || !peer_workspaces || !peer_outs) {
        set_error("evk_voxel_fold_allreduce_f32: bad arguments (world=%d rank=%d, at most %d peers)", world, rank, kMaxPeers);
        return EVK_E_ARG;
    }
    if (flags & EVK_PEER_MULTICAST) {
        // entry 0 of both arrays is the multicast address of the buffer
        if (!peer_workspaces[0] || !peer_outs[0] || ((uintptr_t)peer_workspaces[0] & 15)) {
            set_error("evk_voxel_fold_allreduce_f32: null or misaligned multicast pointer");
            return EVK_E_ARG;
        }
        const int64_t npix_mc = (int64_t)H * W;
        const int64_t lo_mc = npix_mc * rank / world, hi_mc = npix_mc * (rank + 1) / world;
        if (hi_mc > lo_mc) {
            prof_count(1);
            voxel_fold_allreduce_nvls_kernel<<<grid_simple(hi_mc - lo_mc, 128), 128, 0, static_cast<cudaStream_t>(stream)>>>(
                static_cast<const float4 *>(peer_workspaces[0]), peer_outs[0], lo_mc, hi_mc, npix_mc, B, quads_for_bins(B));
            EVK_CUDA(cudaGetLastError());
        }
        return EVK_OK;
    }
    VoxelPeers P{};
    for (int r = 0; r < world; ++r) {
        if (!peer_workspaces[r] || !peer_outs[r] || ((uintptr_t)peer_workspaces[r] & 15)) {
            set_error("evk_voxel_fold_allreduce_f32: peer %d: null or misaligned pointer", r);
            return EVK_E_ARG;
        }
        P.ws[r] = static_cast<const float4 *>(peer_workspaces[r]);
        P.out[r] = peer_outs[r];
    }
    const int64_t npix = (int64_t)H * W;
    const int64_t lo = npix * rank / world, hi = npix * (rank + 1) / world;
    if (hi > lo) {
        prof_count(1);
        const int nq = quads_for_bins(B);
        cudaStream_t st = static_cast<cudaStream_t>(stream);
        // 128-thread CTAs: the slice is small (npix / world pixels), spread it over the SMs
        const int grid = grid_simple(hi - lo, 128);
#define EVK_FAR(WN, QN) voxel_fold_allreduce_kernel<WN, QN><<<grid, 128, 0, st>>>(P, world, lo, hi, npix, B, nq)
        if (nq == 2 && world == 2) EVK_FAR(2, 2);
        else if (nq == 2 && world == 4) EVK_FAR(4, 2);
        else if (nq == 2 && world == 8) EVK_FAR(8, 2);
        else EVK_FAR(0, 0);
#undef EVK_FAR
        EVK_CUDA(cudaGetLastError());
    }
    return EVK_OK;
}

int evk_voxel_negpos_f32(const float *x, const float *y, const float *t, const float *p, int64_t n, float t0, float dt,
                         int B, int H, int W, unsigned flags, float *out_pos_neg, void *workspace, size_t workspace_bytes,
                         unsigned long long *oob, void *stream)
{
    using namespace evk;
    int rc = check_common(n, B, H, W, out_pos_neg);
    if (rc) return rc;
    if (n > 0 && (!x || !y || !t || !p)) { set_error("evk_voxel_negpos_f32: null event array"); return EVK_E_ARG; }
    if (flags & EVK_BILINEAR) { set_error("evk_voxel_negpos_f32: spatial bilinear is not available in neg/pos mode"); return EVK_E_UNSUPPORTED; }
    VoxelArgs A{};
    A.x = x; A.y = y; A.t = t; A.p = p; A.n = n;
    A.t0 = t0; A.dt = dt; A.bm1 = (float)(B - 1);
    A.B = B; A.H = H; A.W = W;
    A.negpos = (flags & EVK_NEGPOS_TRUTHY) ? 2 : 1;
    A.auto_span = (flags & EVK_AUTO_SPAN) ? 1 : 0;
    A.out = out_pos_neg; A.oob = oob;
    const uintptr_t ax = (uintptr_t)x & 15, ay = (uintptr_t)y & 15, at = (uintptr_t)t & 15, ap = (uintptr_t)p & 15;
    int layout = LAYOUT_SOA1;
    if (ax == ay && ay == at && at == ap && (ax & 3) == 0) {
        layout = LAYOUT_SOA4;
        A.head = ((16 - ax) & 15) >> 2;
        if (A.head > n) A.head = n;
    }
    return launch_voxel(A, flags, layout, static_cast<cudaStream_t>(stream), workspace, workspace_bytes);
}

int evk_voxel_packed_f32(const int16_t *x, const int16_t *y, const double *t, const uint8_t *p, int64_t n, double t_first,
                         double t_last, int B, int H, int W, unsigned flags, float *out, void *workspace,
                         size_t workspace_bytes, unsigned long long *oob, void *stream)
{
    using namespace evk;
    int rc = check_common(n, B, H, W, out);
    if (rc) return rc;
    if (n > 0 && (!x || !y || !t || !p)) { set_error("evk_voxel_packed_f32: null event array"); return EVK_E_ARG; }
    if (flags & EVK_BILINEAR) { set_error("evk_voxel_packed_f32: spatial bilinear is not available for the packed layout"); return EVK_E_UNSUPPORTED; }
    VoxelArgs A{};
    A.px16 = x; A.py16 = y; A.pt64 = t; A.pp8 = p; A.n = n;
    A.t_first = t_first;
    A.t0 = 0.0f; A.dt = (float)(t_last - t_first); A.bm1 = (float)(B - 1);
    A.B = B; A.H = H; A.W = W;
    A.auto_span = (flags & EVK_AUTO_SPAN) ? 1 : 0;
    A.out = out; A.oob = oob;
    return launch_voxel(A, flags, LAYOUT_PACKED, static_cast<cudaStream_t>(stream), workspace, workspace_bytes);
}

}  // extern "C"
