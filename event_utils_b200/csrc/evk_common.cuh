// evk_common.cuh -- shared host/device helpers for libevk.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <float.h>
#include <stdint.h>

#include <type_traits>

#include "evk.h"

#if defined(__CUDA_ARCH__) && (__CUDA_ARCH__ != 900)
#error "libevk is written for sm_90a (H100) only"
#endif

namespace evk {

// ---- host side ---------------------------------------------------------------------------
void set_error(const char *fmt, ...);
int cuda_fail(cudaError_t e, const char *what);
int num_sms();  // SM count of the current device (cached)

#define EVK_CUDA(call)                                              \
    do {                                                            \
        cudaError_t e__ = (call);                                   \
        if (e__ != cudaSuccess) return ::evk::cuda_fail(e__, #call); \
    } while (0)

#define EVK_REQUIRE(cond, msg)                      \
    do {                                            \
        if (!(cond)) {                              \
            ::evk::set_error("%s: %s", __func__, msg); \
            return EVK_E_ARG;                       \
        }                                           \
    } while (0)

// measurement hooks (evk_core.cu): count a kernel launch / bracket a dominant kernel with events
void prof_count(int launches);
struct ProfScope {
    cudaStream_t st;
    int slot;
    ProfScope(cudaStream_t s);
    ~ProfScope();
};

// evk_hot.cu: adaptive shared-memory write-combining scatter (mode 0 nearest f32, 1 bilinear f32, 2 count u32)
int launch_image_hot(const float *x, const float *y, const float *p, int64_t n, int H, int W, int clip, float clipx,
                     float clipy, int mode, int force_cache, float *out, float *ws, unsigned *out_u32,
                     unsigned long long *oob, cudaStream_t st);

// evk_image.cu: dense flow [2][H][W] -> interleaved [H][W] {u, v} pairs (see flow_row below)
void launch_flow_interleave(const float *flow, int64_t npix, float2 *uv, cudaStream_t st);
// evk_image.cu: 2x2-block workspace [H][W][4] {TL,TR,BL,BR} -> out[H][W] (overwritten)
void launch_image_fold(const float *ws, float *out, int H, int W, cudaStream_t st);

static inline unsigned variant_of(unsigned flags) { return flags & EVK_VARIANT_MASK; }

// Persistent-style launch geometry: exactly ONE wave -- SM count x the number of CTAs of this
// kernel that are co-resident on an SM (occupancy query, cached per kernel) -- capped by the work
// available.  A grid-stride kernel launched with more CTAs than are resident pays a partial
// second wave.
int resident_ctas_per_sm(const void *kernel, int threads, size_t dyn_smem);
double grid_waves();  // waves of CTAs per launch (EVK_GRID_WAVES, default in evk_core.cu)

template <typename K>
static inline int grid_for(K kernel, int threads, int64_t work_items, int items_per_cta, size_t dyn_smem = 0)
{
    int64_t need = (work_items + items_per_cta - 1) / items_per_cta;
    int64_t cap = (int64_t)(num_sms() * resident_ctas_per_sm((const void *)kernel, threads, dyn_smem) * grid_waves());
    if (need < 1) need = 1;
    return (int)(need < cap ? need : cap);
}

// plain elementwise kernels: enough CTAs to cover the items, at most 8 per SM
static inline int grid_simple(int64_t work_items, int items_per_cta)
{
    int64_t need = (work_items + items_per_cta - 1) / items_per_cta;
    int64_t cap = (int64_t)num_sms() * 8;
    if (need < 1) need = 1;
    return (int)(need < cap ? need : cap);
}

// ---- device side -------------------------------------------------------------------------
#ifdef __CUDACC__

// torch `Tensor.long()` (truncate toward zero) followed by python index wrapping:
// [-size,-1] wraps once, everything else outside [0,size) is the reference's IndexError.
// NaN / inf / |v| >= 2^31 can never be a valid index.
__device__ __forceinline__ bool wrap_trunc_index(float v, int size, int &out)
{
    if (!(fabsf(v) < 2.0e9f)) return false;
    int i = __float2int_rz(v);
    if (i < 0) i += size;
    out = i;
    return (unsigned)i < (unsigned)size;
}

// float -> int truncation that refuses NaN / inf / values no index can take
__device__ __forceinline__ bool trunc_checked(float v, int &i)
{
    if (!(fabsf(v) < 2.0e9f)) return false;
    i = __float2int_rz(v);
    return true;
}

__device__ __forceinline__ bool wrap_int_index(int i, int size, int &out)
{
    if (i < 0) i += size;
    out = i;
    return (unsigned)i < (unsigned)size;
}

// streaming (evict-first) loads: the event arrays are read exactly once and must not push the
// L2-resident accumulation grid out.
__device__ __forceinline__ float4 ld_stream4(const float *p) { return __ldcs(reinterpret_cast<const float4 *>(p)); }
__device__ __forceinline__ float ld_stream(const float *p) { return __ldcs(p); }
__device__ __forceinline__ double ld_stream(const double *p) { return __ldcs(p); }
__device__ __forceinline__ double2 ld_stream2(const double *p) { return __ldcs(reinterpret_cast<const double2 *>(p)); }

// no-return global reductions, spelled in PTX so that (a) the address space is explicit -- a
// pointer read from a by-value argument struct is a GENERIC pointer and atomicAdd() on it compiles
// to ATOM.E + shared-memory CAS fall-backs instead of REDG -- and (b) no return value is requested.
// SASS: REDG.E.ADD.F32 / REDG.E.ADD.F32x2 / REDG.E.ADD.F32x4 (vector forms are sm_90+).
// No "memory" clobber on purpose: the reductions are relaxed, nothing in the same kernel reads the
// accumulators back, and the compiler must stay free to hoist the next events' loads above them.
__device__ __forceinline__ void red_add(float *addr, float v)
{
    asm volatile("red.relaxed.gpu.global.add.f32 [%0], %1;" ::"l"(__cvta_generic_to_global(addr)), "f"(v));
}
__device__ __forceinline__ void red_add4(float *addr16, float4 v)
{
    asm volatile("red.relaxed.gpu.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(__cvta_generic_to_global(addr16)),
                 "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w));
}
__device__ __forceinline__ void red_add2(float *addr8, float2 v)
{
    asm volatile("red.relaxed.gpu.global.add.v2.f32 [%0], {%1, %2};" ::"l"(__cvta_generic_to_global(addr8)), "f"(v.x), "f"(v.y));
}
__device__ __forceinline__ void red_add_u32(unsigned *addr, unsigned v)
{
    asm volatile("red.relaxed.gpu.global.add.u32 [%0], %1;" ::"l"(__cvta_generic_to_global(addr)), "r"(v));
}

__device__ __forceinline__ void flush_oob(unsigned long long *oob, unsigned local)
{
    // one atomic per warp, only when something was out of range
    unsigned tot = __reduce_add_sync(0xffffffffu, local);
    if (tot != 0 && (threadIdx.x & 31) == 0 && oob != nullptr)
        asm volatile("red.relaxed.gpu.global.add.u64 [%0], %1;" ::"l"(__cvta_generic_to_global(oob)), "l"((unsigned long long)tot) : "memory");
}

// ---- dense-flow gather (optic_flow.py:37-44 + ATen grid_sampler bilinear/zeros/align_corners) ----
// the two taps (x0, x0+1) of row yy as {u0, v0, u1, v1}; out-of-image taps are zero (grid_sample zero padding).
// INTERLEAVED: 16 contiguous bytes -> one LDG.128 when x0 is even, two LDG.64 otherwise; planar: four LDG.32.
template <bool INTERLEAVED>
__device__ __forceinline__ float4 flow_row(const float *flow, const float2 *uv, int H, int W, int yy, int x0)
{
    float4 r = make_float4(0.f, 0.f, 0.f, 0.f);
    if ((unsigned)yy >= (unsigned)H) return r;
    const bool in0 = (unsigned)x0 < (unsigned)W, in1 = (unsigned)(x0 + 1) < (unsigned)W;
    if (INTERLEAVED) {
        const float2 *row = uv + (int64_t)yy * W;
        if (in0 && in1 && ((x0 & 1) == 0) && ((W & 1) == 0)) {
            r = __ldg(reinterpret_cast<const float4 *>(row + x0));
        } else {
            if (in0) { const float2 a = __ldg(row + x0); r.x = a.x; r.y = a.y; }
            if (in1) { const float2 c = __ldg(row + x0 + 1); r.z = c.x; r.w = c.y; }
        }
    } else {
        const float *fu = flow + (int64_t)yy * W, *fv = fu + (int64_t)H * W;
        if (in0) { r.x = __ldg(fu + x0); r.y = __ldg(fv + x0); }
        if (in1) { r.z = __ldg(fu + x0 + 1); r.w = __ldg(fv + x0 + 1); }
    }
    return r;
}

#endif  // __CUDACC__

}  // namespace evk
