// evk_norm.cu -- RobustNorm: clamp a tensor between two of its percentiles and rescale it.
//
// Semantics: RobustNorm.__call__ / .percentile, reference lib/data_loaders/data_augmentation.py:82-130
//   t = kthvalue(x, k), k = 1 + round(.01 q (numel-1))           (exact order statistic, no interpolation)
//   if t_max == 0 and t_min == 0: return x
//   y = clamp(x, t_min, t_max);  y = (y - min(y)) / (max(y) + 1e-6)        (min(y) = min(t_min, t_max), max(y) = t_max)
// NaN: kthvalue ranks every NaN above +inf whatever its sign bit, and torch.min / torch.max of a tensor holding a NaN
// are NaN, so any NaN in x makes every output NaN unless the identity short-cut is taken.  ordered_key maps every NaN
// to the top key and the first histogram pass (which sees every key) counts them.
// It is the step right AFTER the voxel grid in the data loaders (base_dataset.py:471).
//
// Design: the reference sorts the whole tensor twice (kthvalue).  Here BOTH order statistics are found
// by one 3-pass radix select over the order-preserving 32-bit image of the floats (11 + 11 + 10 bits): each
// pass is one histogram kernel (shared-memory histograms, native u32 atomics) and one single-CTA scan that
// narrows the two prefixes; then one elementwise kernel.  The tensor (<= a few MB) stays in L2 throughout.
#include "evk_common.cuh"

namespace evk {

struct SelectState {
    unsigned prefix[2];          // key bits decided so far, per target
    unsigned long long rank[2];  // remaining 1-based rank inside the prefix class
    float value[2];              // the selected values (after the last pass)
    unsigned long long nans;     // NaNs in x (counted by the first pass)
};

constexpr unsigned kNanKey = 0xffffffffu;   // above +inf (0xff800000); the last bin of every pass

__device__ __forceinline__ unsigned ordered_key(float f)
{
    const unsigned b = __float_as_uint(f);
    if ((b & 0x7fffffffu) > 0x7f800000u) return kNanKey;   // NaN of either sign ranks last, as in kthvalue
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float key_to_float(unsigned u)
{
    return __uint_as_float((u & 0x80000000u) ? (u & 0x7fffffffu) : ~u);
}

constexpr int kBins = 2048;

// pass geometry: bits [shift, shift+nbits) are examined; keys must match `prefix` on the bits above
__global__ void __launch_bounds__(256) select_hist_kernel(const float *__restrict__ x, int64_t n, int shift, int nbits,
                                                          const SelectState *st, unsigned *hist /* [2][kBins] */)
{
    __shared__ unsigned h[2][kBins];
    for (int i = threadIdx.x; i < 2 * kBins; i += 256) (&h[0][0])[i] = 0;
    __syncthreads();
    const unsigned hi_mask = (shift + nbits >= 32) ? 0u : (0xffffffffu << (shift + nbits));
    const unsigned p0 = st->prefix[0] & hi_mask, p1 = st->prefix[1] & hi_mask;
    const unsigned bmask = (1u << nbits) - 1u;
    const int64_t stride = (int64_t)gridDim.x * 256;
    for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < n; i += stride) {
        const unsigned k = ordered_key(x[i]);
        const unsigned b = (k >> shift) & bmask;
        if ((k & hi_mask) == p0) atomicAdd(&h[0][b], 1u);
        if ((k & hi_mask) == p1) atomicAdd(&h[1][b], 1u);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < 2 * kBins; i += 256) {
        const unsigned c = (&h[0][0])[i];
        if (c) atomicAdd(hist + i, c);
    }
}

// one CTA: for each target find the bin holding its rank, narrow the prefix, clear the histogram
__global__ void __launch_bounds__(64) select_scan_kernel(unsigned *hist, int shift, int nbits, int last, SelectState *st)
{
    const int t = threadIdx.x >> 5;  // warp 0 -> target 0, warp 1 -> target 1
    if ((threadIdx.x & 31) == 0) {
        unsigned long long rank = st->rank[t], cum = 0;
        const int nb = 1 << nbits;
        int b = 0;
        for (; b < nb; ++b) {
            const unsigned c = hist[t * kBins + b];
            if (cum + c >= rank) break;
            cum += c;
        }
        if (b == nb) b = nb - 1;
        if (t == 0 && shift + nbits >= 32) st->nans = hist[nb - 1];   // first pass: every key was counted, kNanKey in the last bin
        st->prefix[t] |= (unsigned)b << shift;
        st->rank[t] = rank - cum;
        if (last) st->value[t] = key_to_float(st->prefix[t]);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < 2 * kBins; i += 64) hist[i] = 0;
}

__global__ void __launch_bounds__(256) robust_norm_kernel(const float *__restrict__ x, int64_t n, const SelectState *st,
                                                          float *__restrict__ out)
{
    const float t_min = st->value[0], t_max = st->value[1];
    const bool identity = (t_max == 0.0f && t_min == 0.0f);     // data_augmentation.py:124-125
    const bool all_nan = !identity && st->nans != 0;           // min(y) / max(y) are NaN (data_augmentation.py:129)
    // min(clamp(x, t_min, t_max)): t_min, or t_max when t_min > t_max (torch.clamp then yields t_max everywhere)
    const float lo = fminf(t_min, t_max);
    const float denom = __fadd_rn(t_max, 1e-6f);
    const int64_t stride = (int64_t)gridDim.x * 256;
    for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < n; i += stride) {
        const float v = x[i];
        if (identity) { out[i] = v; continue; }
        if (all_nan) { out[i] = __int_as_float(0x7fffffff); continue; }
        // torch.clamp(x, min, max) = min(max(x, t_min), t_max)
        float c = fminf(fmaxf(v, t_min), t_max);
        out[i] = __fdiv_rn(__fsub_rn(c, lo), denom);
    }
}

}  // namespace evk

extern "C" {

size_t evk_robust_norm_workspace_bytes(void) { return 2 * evk::kBins * sizeof(unsigned) + 256; }

int evk_robust_norm_f32(const float *x, int64_t n, int64_t k_low, int64_t k_top, float *out, float *t_min_max, void *workspace,
                        size_t workspace_bytes, void *stream)
{
    using namespace evk;
    if (!x || !out || n < 1 || k_low < 1 || k_top < 1 || k_low > n || k_top > n || !workspace ||
        workspace_bytes < evk_robust_norm_workspace_bytes() || ((uintptr_t)workspace & 15)) {
        set_error("evk_robust_norm_f32: bad arguments (1 <= k <= n, 16-byte aligned workspace of %zu bytes)", evk_robust_norm_workspace_bytes());
        return EVK_E_ARG;
    }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    unsigned *hist = static_cast<unsigned *>(workspace);
    SelectState *state = reinterpret_cast<SelectState *>(hist + 2 * kBins);
    SelectState init{};
    init.rank[0] = (unsigned long long)k_low; init.rank[1] = (unsigned long long)k_top;
    EVK_CUDA(cudaMemsetAsync(hist, 0, 2 * kBins * sizeof(unsigned), st));
    EVK_CUDA(cudaMemcpyAsync(state, &init, sizeof(init), cudaMemcpyHostToDevice, st));
    const int shifts[3] = {21, 10, 0}, bits[3] = {11, 11, 10};
    const int grid = grid_for(select_hist_kernel, 256, n, 256 * 8);
    for (int p = 0; p < 3; ++p) {
        prof_count(2);
        select_hist_kernel<<<grid, 256, 0, st>>>(x, n, shifts[p], bits[p], state, hist);
        select_scan_kernel<<<1, 64, 0, st>>>(hist, shifts[p], bits[p], p == 2, state);
    }
    prof_count(1);
    robust_norm_kernel<<<grid_simple(n, 256 * 4), 256, 0, st>>>(x, n, state, out);
    if (t_min_max) EVK_CUDA(cudaMemcpyAsync(t_min_max, state->value, 2 * sizeof(float), cudaMemcpyDeviceToDevice, st));
    EVK_CUDA(cudaGetLastError());
    return EVK_OK;
}

}  // extern "C"
