// evk_hot.cu -- hot-spot (contention-aware) event-image scatter: a per-CTA write-combining cache
// in shared memory in front of the global reductions.
//
// Same semantics as evk_image.cu (events_to_image_torch, reference
// lib/representations/image.py:46-115); only the accumulation strategy differs.
//
// Why: on a Zipf-distributed stream (BASELINE config 4) a few pixels receive millions of events.
// Global reductions to ONE address serialise in its L2 slice, so such a stream takes many times
// longer than a uniform one.  Each CTA therefore keeps a
// small direct-mapped table {cell -> partial sum} in shared memory: an event whose cell owns its
// slot is accumulated with a shared-memory atomic, everything else (slot taken by another cell)
// goes straight to L2, and the table is flushed with one reduction per occupied slot at the end.
// Round 2: 8192-slot two-way set-associative table per 512-thread CTA, INTEGER (fixed-point) values so that the hot
// cells use native shared-memory atomics, 16-byte event loads in the cached path as well.
// Hot cells are thereby reduced to one L2 reduction per CTA.  The kernel is ADAPTIVE: a prologue
// counts intra-warp duplicates (match.any) among the CTA's first events and turns the cache off
// for streams without contention, where it would only add shared-memory traffic.
#include "evk_common.cuh"

namespace evk {

struct HotArgs {
    const float *x, *y, *p;
    int64_t n;
    int H, W;
    int clip;
    float clipx, clipy;
    float *out;
    float *ws;         // bilinear only: block workspace ws[H][W][4] (TL,TR,BL,BR); NULL -> taps go to `out`
    unsigned *out_u32;
    unsigned long long *oob;
    int force_cache;  // 0 adaptive, 1 always on
    int vec4;         // x, y (and p) are 16-byte aligned
};

constexpr int kHotThreads = 512;
constexpr int kHotLog2 = 13;
constexpr int kHotSlots = 1 << kHotLog2;  // 8192 slots (4096 two-way sets): 32 KB keys + 32 KB values of dynamic shared memory
constexpr unsigned kEmpty = 0xffffffffu;
constexpr unsigned kHotBias = 0x80000000u;
// Table values are INTEGERS (native ATOMS.ADD; f32 shared-memory adds are CAS loops on sm_90a):
//   nearest  value * 2^10 -- exact for the integer polarities event cameras produce (+-1, 0/1), so hot cells keep
//            bit-exact sums; a weight that is not a multiple of 2^-10 below 2^20 bypasses the table (global f32 reduction)
//   bilinear tap * 2^22 (|tap| <= 1; quantisation 2^-23 per tap, below f32 rounding of the accumulation itself)
//   count    plain u32
// A float-mode cell is biased by 2^31; the returning atomic tells the thread whether ITS add wrapped the 32 bits and that
// thread carries +-2^(32-F) to the global image, so the table can never overflow silently.
constexpr int kHotFixNearest = 10, kHotFixBilinear = 22;
// bilinear: ONE table entry per 2x2 footprint -- key = the anchor cell, value = the four taps {TL, TR, BL, BR} -- so an event
// is one lookup and four adjacent native atomics instead of four lookups; flushed as one vector reduction into the block
// workspace (the layout of the uncontended path).  4096 slots (2048 two-way sets): 16 KB keys + 64 KB values.
constexpr int kHotLog2B = 12;
constexpr int kHotSlotsB = 1 << kHotLog2B;

// `gs` = element stride of a cell in the global target (4 when the target is the TL slot of a block)
__device__ __forceinline__ void global_add(float *out, unsigned cell, float v, int gs) { red_add(out + (size_t)cell * gs, v); }
__device__ __forceinline__ void global_add(unsigned *out, unsigned cell, unsigned v, int gs) { red_add_u32(out + (size_t)cell * gs, v); }

// find (or claim) the cell's slot in its two-way set; -1 = both ways belong to other cells
template <int LOG2 = kHotLog2>
__device__ __forceinline__ int hot_slot(unsigned *keys, unsigned cell)
{
    const unsigned s0 = ((cell * 2654435761u) >> (32 - (LOG2 - 1))) * 2u;
    const uint2 k = *reinterpret_cast<const uint2 *>(keys + s0);
    if (k.x == cell) return (int)s0;
    if (k.y == cell) return (int)s0 + 1;
    if (k.x == kEmpty) {
        const unsigned old = atomicCAS(keys + s0, kEmpty, cell);
        if (old == kEmpty || old == cell) return (int)s0;
    }
    const unsigned k1 = *(volatile unsigned *)(keys + s0 + 1);
    if (k1 == cell) return (int)s0 + 1;
    if (k1 == kEmpty) {
        const unsigned old = atomicCAS(keys + s0 + 1, kEmpty, cell);
        if (old == kEmpty || old == cell) return (int)s0 + 1;
    }
    return -1;
}

__device__ __forceinline__ unsigned hot_atoms_ret(unsigned *cell, unsigned v)
{
    unsigned old;
    asm volatile("atom.relaxed.cta.shared::cta.add.u32 %0, [%1], %2;" : "=r"(old) : "r"((unsigned)__cvta_generic_to_shared(cell)), "r"(v));
    return old;
}

// float modes: add value v (already known to be representable: q == v * 2^FIX) to the cell through the table
template <int FIX>
__device__ __forceinline__ void hot_add_fixed(unsigned *keys, unsigned *vals, float *gout, unsigned cell, float v, unsigned q, int gs)
{
    const int slot = hot_slot(keys, cell);
    if (slot < 0) { global_add(gout, cell, v, gs); return; }
    const unsigned old = hot_atoms_ret(vals + slot, q);
    const unsigned nw = old + q;
    if (((old ^ nw) & ~(nw ^ q)) >> 31)      // this add wrapped the cell (see evk_cmax.cu wrap_bit): carry it out
        global_add(gout, cell, (int)q >= 0 ? (float)(1u << (32 - FIX)) : -(float)(1u << (32 - FIX)), gs);
}

enum { HOT_NEAREST = 0, HOT_BILINEAR = 1, HOT_COUNT = 2 };

// one event; CACHE is a compile-time switch so that the cache-off instantiation is the plain scatter code
template <int MODE, bool CACHE>
__device__ __forceinline__ void hot_event(const HotArgs &A, unsigned *keys, unsigned *vals, float x, float y, float pin, unsigned &oob)
{
    float *gf = (MODE == HOT_BILINEAR && A.ws) ? A.ws : A.out;
    const int gs = (MODE == HOT_BILINEAR && A.ws) ? 4 : 1;
    if (MODE == HOT_NEAREST || MODE == HOT_COUNT) {
        // image.py:88-95
        const bool keep = !A.clip || (!(x >= A.clipx) && !(y >= A.clipy));
        int ux, uy, xi, yi;
        if (!trunc_checked(x, ux) || !trunc_checked(y, uy)) { ++oob; return; }
        if (!keep) { ux = 0; uy = 0; }
        if (!wrap_int_index(ux, A.W, xi) || !wrap_int_index(uy, A.H, yi)) { ++oob; return; }
        const unsigned cell = (unsigned)yi * (unsigned)A.W + (unsigned)xi;
        if (MODE == HOT_COUNT) {
            int slot = -1;
            if (CACHE) slot = hot_slot(keys, cell);
            if (slot >= 0) atomicAdd(vals + slot, 1u);
            else red_add_u32(A.out_u32 + cell, 1u);
        } else {
            const float p = pin;
            if (p == 0.0f) return;
            if (CACHE) {
                const float ps = __fmul_rn(p, (float)(1 << kHotFixNearest));
                const int q = __float2int_rn(ps);
                if (fabsf(p) < 1048576.0f && (float)q == ps) { hot_add_fixed<kHotFixNearest>(keys, vals, gf, cell, p, (unsigned)q, 1); return; }
            }
            red_add(gf + cell, p);
        }
    } else {
        // image.py:79-86 + 111-114
        const float p = pin;
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
        const float v00 = __fmul_rn(wl, oy), v01 = __fmul_rn(wr, oy), v10 = __fmul_rn(wl, dy), v11 = __fmul_rn(wr, dy);
        const unsigned r0 = (unsigned)y0 * (unsigned)A.W, r1 = (unsigned)y1 * (unsigned)A.W;
        if (!CACHE && A.ws && x1 == x0 + 1 && y1 == y0 + 1) {
            // uncontended stream: the whole footprint as ONE vector reduction into its block
            if (v00 != 0.0f || v01 != 0.0f || v10 != 0.0f || v11 != 0.0f)
                red_add4(A.ws + ((size_t)r0 + x0) * 4, make_float4(v00, v01, v10, v11));
        } else if (CACHE && fabsf(w) <= 1.0f && x1 == x0 + 1 && y1 == y0 + 1) {
            if (w == 0.0f) return;
            const float S = (float)(1 << kHotFixBilinear);
            const unsigned q[4] = {(unsigned)__float2int_rn(__fmul_rn(v00, S)), (unsigned)__float2int_rn(__fmul_rn(v01, S)),
                                   (unsigned)__float2int_rn(__fmul_rn(v10, S)), (unsigned)__float2int_rn(__fmul_rn(v11, S))};
            const unsigned cell = r0 + x0;                      // the footprint's anchor
            const int slot = hot_slot<kHotLog2B>(keys, cell);
            if (slot < 0) {
                if (A.ws) red_add4(A.ws + (size_t)cell * 4, make_float4(v00, v01, v10, v11));
                else { red_add(A.out + cell, v00); red_add(A.out + cell + 1, v01); red_add(A.out + r1 + x0, v10); red_add(A.out + r1 + x1, v11); }
                return;
            }
            unsigned *vp = vals + 4 * slot;
            const unsigned o0 = hot_atoms_ret(vp + 0, q[0]), o1 = hot_atoms_ret(vp + 1, q[1]);
            const unsigned o2 = hot_atoms_ret(vp + 2, q[2]), o3 = hot_atoms_ret(vp + 3, q[3]);
            const unsigned o[4] = {o0, o1, o2, o3};
            unsigned any = 0;
#pragma unroll
            for (int k = 0; k < 4; ++k) { const unsigned nw = o[k] + q[k]; any |= (o[k] ^ nw) & ~(nw ^ q[k]); }
            if (any >> 31) {
                const unsigned cells[4] = {cell, cell + 1, r1 + x0, r1 + x1};
                const float carry = (float)(1u << (32 - kHotFixBilinear));
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    const unsigned nw = o[k] + q[k];
                    if (((o[k] ^ nw) & ~(nw ^ q[k])) >> 31) {
                        // the wrapped tap's 2^32 goes to the global image: tap k of block `cell` (or its own pixel without blocks)
                        if (A.ws) red_add(A.ws + (size_t)cell * 4 + k, (int)q[k] >= 0 ? carry : -carry);
                        else red_add(A.out + cells[k], (int)q[k] >= 0 ? carry : -carry);
                    }
                }
            }
        } else {
            if (v00 != 0.0f) global_add(gf, r0 + x0, v00, gs);
            if (v01 != 0.0f) global_add(gf, r0 + x1, v01, gs);
            if (v10 != 0.0f) global_add(gf, r1 + x0, v10, gs);
            if (v11 != 0.0f) global_add(gf, r1 + x1, v11, gs);
        }
    }
}

// the event loop; VEC4: 16-byte loads (x, y, p all 16-byte aligned)
template <int MODE, bool CACHE, bool VEC4>
__device__ __forceinline__ void hot_loop(const HotArgs &A, unsigned *keys, unsigned *vals, int64_t tid, int64_t stride, unsigned &oob)
{
    if (VEC4) {
        const int64_t n4 = A.n >> 2;
        for (int64_t g = tid; g < n4; g += stride) {
            const float4 X = ld_stream4(A.x + 4 * g), Y = ld_stream4(A.y + 4 * g);
            const float4 P = (MODE == HOT_COUNT) ? make_float4(1.f, 1.f, 1.f, 1.f) : ld_stream4(A.p + 4 * g);
            hot_event<MODE, CACHE>(A, keys, vals, X.x, Y.x, P.x, oob);
            hot_event<MODE, CACHE>(A, keys, vals, X.y, Y.y, P.y, oob);
            hot_event<MODE, CACHE>(A, keys, vals, X.z, Y.z, P.z, oob);
            hot_event<MODE, CACHE>(A, keys, vals, X.w, Y.w, P.w, oob);
        }
        for (int64_t i = (n4 << 2) + tid; i < A.n; i += stride)
            hot_event<MODE, CACHE>(A, keys, vals, A.x[i], A.y[i], (MODE == HOT_COUNT) ? 1.0f : A.p[i], oob);
    } else {
        for (int64_t i = tid; i < A.n; i += stride)
            hot_event<MODE, CACHE>(A, keys, vals, ld_stream(A.x + i), ld_stream(A.y + i), (MODE == HOT_COUNT) ? 1.0f : ld_stream(A.p + i), oob);
    }
}

template <int MODE>
__global__ void __launch_bounds__(kHotThreads) image_hot_kernel(const HotArgs A)
{
    extern __shared__ __align__(16) unsigned hot_smem[];      // [slots] keys, [slots] (bilinear: [slots][4]) values
    constexpr int kSlots = (MODE == HOT_BILINEAR) ? kHotSlotsB : kHotSlots;
    constexpr int kValsPer = (MODE == HOT_BILINEAR) ? 4 : 1;
    unsigned *keys = hot_smem, *vals = hot_smem + kSlots;
    const int64_t tid = (int64_t)blockIdx.x * kHotThreads + threadIdx.x;
    const int64_t stride = (int64_t)gridDim.x * kHotThreads;

    // ---- prologue: is this stream contended?  (lanes whose first event shares its pixel with
    // another lane of the same warp)
    bool use_cache = A.force_cache != 0;
    if (!use_cache) {
        unsigned long long key = ~0ull - (threadIdx.x & 31);
        if (tid < A.n) {
            int ux, uy;
            if (trunc_checked(A.x[tid], ux) && trunc_checked(A.y[tid], uy)) key = ((unsigned long long)(unsigned)uy << 32) | (unsigned)ux;
        }
        // counted over the CTA by the barrier itself: one __syncthreads_count, no shared-memory traffic
        const int dup_lanes = __syncthreads_count(__popc(__match_any_sync(0xffffffffu, key)) > 1);
        use_cache = dup_lanes * 64 > kHotThreads;  // > 1/64 of the lanes collide inside their warp (uniform streams: ~0.01 %)
    }
    const unsigned init = (MODE == HOT_COUNT) ? 0u : kHotBias;
    if (use_cache) {   // only CTAs that will use the table pay for initialising it
        for (int s = threadIdx.x; s < kSlots; s += kHotThreads) keys[s] = kEmpty;
        for (int s = threadIdx.x; s < kSlots * kValsPer; s += kHotThreads) vals[s] = init;
        __syncthreads();
    }

    unsigned oob = 0;
    // cache off -> the plain scatter code, cache on -> the table; 16-byte loads when the arrays allow
    if (use_cache) { if (A.vec4) hot_loop<MODE, true, true>(A, keys, vals, tid, stride, oob); else hot_loop<MODE, true, false>(A, keys, vals, tid, stride, oob); }
    else if (A.vec4) hot_loop<MODE, false, true>(A, keys, vals, tid, stride, oob);
    else hot_loop<MODE, false, false>(A, keys, vals, tid, stride, oob);
    __syncthreads();
    if (use_cache) {
        float *gf = (MODE == HOT_BILINEAR && A.ws) ? A.ws : A.out;
        const int gs = (MODE == HOT_BILINEAR && A.ws) ? 4 : 1;
        const float inv = 1.0f / (float)(1 << (MODE == HOT_BILINEAR ? kHotFixBilinear : kHotFixNearest));
        for (int s = threadIdx.x; s < kSlots; s += kHotThreads) {
            const unsigned k = keys[s];
            if (k == kEmpty) continue;
            if (MODE == HOT_BILINEAR) {
                const uint4 v = *reinterpret_cast<const uint4 *>(vals + 4 * s);
                const float4 f = make_float4(__fmul_rn((float)(int)(v.x - kHotBias), inv), __fmul_rn((float)(int)(v.y - kHotBias), inv),
                                             __fmul_rn((float)(int)(v.z - kHotBias), inv), __fmul_rn((float)(int)(v.w - kHotBias), inv));
                if (f.x == 0.0f && f.y == 0.0f && f.z == 0.0f && f.w == 0.0f) continue;
                if (A.ws) red_add4(A.ws + (size_t)k * 4, f);
                else { red_add(A.out + k, f.x); red_add(A.out + k + 1, f.y); red_add(A.out + k + A.W, f.z); red_add(A.out + k + A.W + 1, f.w); }
            } else {
                const unsigned v = vals[s];
                if (v == init) continue;
                if (MODE == HOT_COUNT) red_add_u32(A.out_u32 + k, v);
                else global_add(gf, k, __fmul_rn((float)(int)(v - kHotBias), inv), gs);
            }
        }
    }
    flush_oob(A.oob, oob);
}

template <int MODE>
static int launch_hot_mode(const HotArgs &A, cudaStream_t st)
{
    const size_t smem = (MODE == HOT_BILINEAR) ? (size_t)kHotSlotsB * 5 * sizeof(unsigned) : (size_t)kHotSlots * 2 * sizeof(unsigned);
    EVK_CUDA(cudaFuncSetAttribute(image_hot_kernel<MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    // ONE wave of resident CTAs: every CTA that uses its table flushes it at the end (up to 8192 reductions, most of them
    // the single count of a tail cell), so the number of CTAs is what the flush traffic scales with (4 waves: 14.5 M
    // flush reductions per 50 M-event launch, as many as the misses themselves)
    int64_t need = (A.n + (int64_t)kHotThreads * 16 - 1) / ((int64_t)kHotThreads * 16);
    const int64_t cap = (int64_t)num_sms() * resident_ctas_per_sm((const void *)image_hot_kernel<MODE>, kHotThreads, smem);
    if (need < 1) need = 1;
    image_hot_kernel<MODE><<<(int)(need < cap ? need : cap), kHotThreads, smem, st>>>(A);
    return EVK_OK;
}

int launch_image_hot(const float *x, const float *y, const float *p, int64_t n, int H, int W, int clip, float clipx,
                     float clipy, int mode, int force_cache, float *out, float *ws, unsigned *out_u32,
                     unsigned long long *oob, cudaStream_t st)
{
    if ((int64_t)H * W >= 0xffffffffLL) { set_error("hot-spot variant: image too large for 32-bit cell ids"); return EVK_E_UNSUPPORTED; }
    HotArgs A{};
    A.x = x; A.y = y; A.p = p; A.n = n; A.H = H; A.W = W;
    A.clip = clip; A.clipx = clipx; A.clipy = clipy;
    A.out = out; A.ws = ws; A.out_u32 = out_u32; A.oob = oob; A.force_cache = force_cache;
    A.vec4 = ((((uintptr_t)x | (uintptr_t)y | (uintptr_t)(p ? p : x)) & 15) == 0) ? 1 : 0;
    if (n <= 0) return EVK_OK;
    ProfScope prof(st);
    prof_count(1);
    int rc;
    if (mode == HOT_NEAREST) rc = launch_hot_mode<HOT_NEAREST>(A, st);
    else if (mode == HOT_BILINEAR) rc = launch_hot_mode<HOT_BILINEAR>(A, st);
    else rc = launch_hot_mode<HOT_COUNT>(A, st);
    if (rc) return rc;
    EVK_CUDA(cudaGetLastError());
    return EVK_OK;
}

}  // namespace evk
