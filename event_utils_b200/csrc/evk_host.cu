// evk_host.cu -- host-buffer pipeline: voxel build for events that live in HOST memory.
//
// The reference's consumers hand over host arrays (numpy / CPU tensors: data loaders
// lib/data_loaders/base_dataset.py:446-453).  Moving 16 B/event over PCIe costs far more than the
// scatter itself, so the copy is chunked and double-buffered: while chunk k is scattered on the
// compute stream, chunk k+1 is in flight on the copy stream.  The accumulation grid stays on the
// device (L2 resident) for the whole call and is read back once.
#include <pthread.h>
#include <sched.h>
#include <stdlib.h>
#include <string.h>
#if defined(__x86_64__)
#include <emmintrin.h>
#endif

#include <atomic>
#include <condition_variable>
#include <functional>
#include <mutex>
#include <thread>
#include <vector>

#include "evk_common.cuh"

// ---- persistent host worker pool -------------------------------------------------------------------
// The staging copy of a chunk (64 MB) and the content hash of an event set are too short to pay for two dozen serial
// thread creations each time: the workers are created once, sleep on a condition variable and
// take jobs from one atomic counter (the caller works too).  Never destroyed: the workers are detached and end with
// the process.  Runs are serialised, so any number of caller threads may use it.
namespace {
class HostPool {
public:
    static HostPool &get()
    {
        static HostPool *pool = new HostPool();      // leaked on purpose (no destruction order problems at exit)
        return *pool;
    }
    // fn(j) for every j in [0, njobs) on at most `width` threads (the caller included); returns when all are done
    void run(size_t njobs, int width, const std::function<void(size_t)> &fn)
    {
        if (njobs == 0) return;
        int helpers = width - 1;
        if (helpers > nworkers_) helpers = nworkers_;
        if ((size_t)helpers > njobs - 1) helpers = (int)(njobs - 1);
        if (helpers <= 0) { for (size_t j = 0; j < njobs; ++j) fn(j); return; }
        std::lock_guard<std::mutex> serial(run_mutex_);
        {
            std::lock_guard<std::mutex> lk(m_);
            fn_ = &fn; njobs_ = njobs; next_.store(0, std::memory_order_relaxed);
            helpers_ = helpers; running_ = helpers;
            ++generation_;
        }
        cv_work_.notify_all();
        drain(fn, njobs);
        std::unique_lock<std::mutex> lk(m_);
        cv_done_.wait(lk, [&] { return running_ == 0; });
        fn_ = nullptr;
    }

private:
    HostPool()
    {
        // half of the CPUs this process may run on (it may be bound to the GPU's NUMA node), 3..31 workers;
        // EVK_HOST_THREADS overrides the total (workers + caller)
        int avail = 0;
        cpu_set_t set;
        if (sched_getaffinity(0, sizeof(set), &set) == 0) avail = CPU_COUNT(&set);
        if (avail <= 0) avail = (int)std::thread::hardware_concurrency();
        int total = avail / 2;
        const char *e = getenv("EVK_HOST_THREADS");
        if (e && *e) total = atoi(e);
        if (total < 4 && !(e && *e)) total = 4;
        if (total < 1) total = 1;
        if (total > 32) total = 32;
        nworkers_ = total - 1;
        for (int i = 0; i < nworkers_; ++i) std::thread(&HostPool::worker, this, i).detach();
        // a forked child (e.g. a DataLoader worker) inherits this object but none of its threads: it works serially
        self_ = this;
        pthread_atfork(nullptr, nullptr, [] { if (self_) self_->nworkers_ = 0; });
    }
    static HostPool *self_;
    void drain(const std::function<void(size_t)> &fn, size_t njobs)
    {
        for (size_t j = next_.fetch_add(1, std::memory_order_relaxed); j < njobs; j = next_.fetch_add(1, std::memory_order_relaxed)) fn(j);
    }
    void worker(int index)
    {
        uint64_t seen = 0;
        for (;;) {
            const std::function<void(size_t)> *fn;
            size_t njobs;
            {
                std::unique_lock<std::mutex> lk(m_);
                cv_work_.wait(lk, [&] { return generation_ != seen; });
                seen = generation_;
                if (index >= helpers_) continue;       // this run is narrower than the pool
                fn = fn_; njobs = njobs_;
            }
            drain(*fn, njobs);
            std::lock_guard<std::mutex> lk(m_);
            if (--running_ == 0) cv_done_.notify_one();
        }
    }
    std::mutex run_mutex_, m_;
    std::condition_variable cv_work_, cv_done_;
    const std::function<void(size_t)> *fn_ = nullptr;
    size_t njobs_ = 0;
    std::atomic<size_t> next_{0};
    uint64_t generation_ = 0;
    int helpers_ = 0, running_ = 0, nworkers_ = 0;
};
HostPool *HostPool::self_ = nullptr;
}  // namespace

// ---- content hash of a host buffer (identity of a cached event set) ---------------------------------
// Four independent multiply-rotate lanes over 32-byte stripes (the structure of XXH64), merged and
// avalanched; the tail is zero-padded into one more stripe and the length is mixed in.  Every byte of
// the buffer enters the result.  Large buffers are cut into equal pieces hashed on separate threads and
// the piece hashes are chained in order, so the value does not depend on the thread count.
namespace {
constexpr uint64_t kP1 = 0x9E3779B185EBCA87ull, kP2 = 0xC2B2AE3D27D4EB4Full, kP3 = 0x165667B19E3779F9ull,
                   kP4 = 0x85EBCA77C2B2AE63ull, kP5 = 0x27D4EB2F165667C5ull;
inline uint64_t rotl64(uint64_t v, int r) { return (v << r) | (v >> (64 - r)); }
inline uint64_t lane_round(uint64_t acc, uint64_t in) { return rotl64(acc + in * kP2, 31) * kP1; }
inline uint64_t lane_merge(uint64_t h, uint64_t v) { return (h ^ lane_round(0, v)) * kP1 + kP4; }

uint64_t hash_piece(const unsigned char *p, size_t n, uint64_t seed)
{
    uint64_t v0 = seed + kP1 + kP2, v1 = seed + kP2, v2 = seed, v3 = seed - kP1;
    size_t i = 0;
    for (; i + 32 <= n; i += 32) {
        uint64_t w[4];
        memcpy(w, p + i, 32);
        v0 = lane_round(v0, w[0]); v1 = lane_round(v1, w[1]); v2 = lane_round(v2, w[2]); v3 = lane_round(v3, w[3]);
    }
    if (i < n) {
        uint64_t w[4] = {0, 0, 0, 0};
        memcpy(w, p + i, n - i);
        v0 = lane_round(v0, w[0]); v1 = lane_round(v1, w[1]); v2 = lane_round(v2, w[2]); v3 = lane_round(v3, w[3]);
    }
    uint64_t h = rotl64(v0, 1) + rotl64(v1, 7) + rotl64(v2, 12) + rotl64(v3, 18);
    h = lane_merge(h, v0); h = lane_merge(h, v1); h = lane_merge(h, v2); h = lane_merge(h, v3);
    h += (uint64_t)n * kP5;
    h ^= h >> 33; h *= kP2; h ^= h >> 29; h *= kP3; h ^= h >> 32;
    return h;
}
}  // namespace

// hash k buffers at once: all 1 MiB pieces of all buffers are spread over one set of threads
static void hash_many(const void *const *ptrs, const size_t *nbytes, int k, const uint64_t *seeds, uint64_t *out)
{
    constexpr size_t kPiece = (size_t)1 << 20;               // fixed piece size: the result is thread-count independent
    struct Job { const unsigned char *p; size_t len; uint64_t seed; uint64_t *dst; };
    std::vector<Job> jobs;
    std::vector<std::vector<uint64_t>> piece_hash(k);
    for (int a = 0; a < k; ++a) {
        const unsigned char *p = (const unsigned char *)ptrs[a];
        const size_t n = p ? nbytes[a] : 0;
        const size_t pieces = n ? (n + kPiece - 1) / kPiece : 1;
        piece_hash[a].resize(pieces);
        for (size_t j = 0; j < pieces; ++j) {
            const size_t off = j * kPiece, len = n ? ((n - off < kPiece) ? n - off : kPiece) : 0;
            jobs.push_back({n ? p + off : (const unsigned char *)"", len, seeds[a] + j, &piece_hash[a][j]});
        }
    }
    // at most 8 threads (the hash runs at memory speed well before that), one job per 1 MiB piece
    int width = (int)(jobs.size() / 2);
    if (width > 8) width = 8;
    HostPool::get().run(jobs.size(), width, [&](size_t j) { *jobs[j].dst = hash_piece(jobs[j].p, jobs[j].len, jobs[j].seed); });
    for (int a = 0; a < k; ++a) {
        const std::vector<uint64_t> &h = piece_hash[a];
        out[a] = (h.size() == 1) ? h[0] : hash_piece((const unsigned char *)h.data(), h.size() * sizeof(uint64_t), seeds[a] ^ (uint64_t)nbytes[a]);
    }
}

extern "C" uint64_t evk_host_hash64(const void *data, size_t nbytes, uint64_t seed)
{
    uint64_t out = 0;
    hash_many(&data, &nbytes, 1, &seed, &out);
    return out;
}

extern "C" void evk_host_hash64_multi(const void *const *ptrs, const size_t *nbytes, int k, uint64_t seed, uint64_t *out)
{
    if (k <= 0 || !ptrs || !nbytes || !out) return;
    std::vector<uint64_t> seeds(k);
    for (int a = 0; a < k; ++a) seeds[a] = seed + 0x9E3779B97F4A7C15ull * (uint64_t)a;
    hash_many(ptrs, nbytes, k, seeds.data(), out);
}

struct evk_pipeline {
    int64_t chunk;            // events per chunk
    float *stage[2][4];       // device staging: x,y,t,p per slot
    cudaStream_t copy, compute;
    cudaEvent_t copied[2], consumed[2];
    float *grid;              // device output grid
    size_t grid_bytes;
    void *ws;                 // voxel workspace
    size_t ws_bytes;
    unsigned long long *oob_dev;
    unsigned long long *oob_pinned;
    // pageable sources: pinned bounce buffers filled by host threads (cudaMemcpyAsync from pageable memory is a
    // single-threaded staged copy inside the driver, far below PCIe speed)
    void *bounce[2][4];
    int64_t bounce_events;    // capacity of one bounce slot
};

namespace {
// is `ptr` ordinary pageable host memory (not pinned / registered / managed / device)?
bool is_pageable(const void *ptr)
{
    cudaPointerAttributes at{};
    if (cudaPointerGetAttributes(&at, ptr) != cudaSuccess) { cudaGetLastError(); return true; }
    return at.type == cudaMemoryTypeUnregistered;
}

// One block of the staging copy.  The destination is a pinned bounce buffer that the DMA engine reads next and the CPU
// never again: non-temporal stores skip the read-for-ownership of the destination lines (2 instead of 3 memory
// transfers per byte) and leave the caches to the source.  EVK_HOST_COPY_STREAM=0 -> plain memcpy.
void copy_block(char *dst, const char *src, size_t n, bool stream)
{
#if defined(__x86_64__)
    if (stream && n >= 256) {
        size_t head = (16 - ((uintptr_t)dst & 15)) & 15;
        memcpy(dst, src, head);
        dst += head; src += head; n -= head;
        size_t i = 0;
        for (; i + 64 <= n; i += 64) {
            const __m128i a = _mm_loadu_si128((const __m128i *)(src + i)), b = _mm_loadu_si128((const __m128i *)(src + i + 16));
            const __m128i c = _mm_loadu_si128((const __m128i *)(src + i + 32)), d = _mm_loadu_si128((const __m128i *)(src + i + 48));
            _mm_stream_si128((__m128i *)(dst + i), a); _mm_stream_si128((__m128i *)(dst + i + 16), b);
            _mm_stream_si128((__m128i *)(dst + i + 32), c); _mm_stream_si128((__m128i *)(dst + i + 48), d);
        }
        memcpy(dst + i, src + i, n - i);
        _mm_sfence();                      // the stores are globally visible before the block counts as done
        return;
    }
#endif
    (void)stream;
    memcpy(dst, src, n);
}

// copy k arrays (bytes[a] each) on the worker pool, 1 MiB blocks (a single memcpy stream tops out well below PCIe 5 x16)
void parallel_copy(void *const *dst, const void *const *src, int k, const size_t *bytes)
{
    static const bool stream = [] { const char *e = getenv("EVK_HOST_COPY_STREAM"); return !(e && *e && atoi(e) == 0); }();
    // 8 threads by default: enough to keep the staging copy ahead of a PCIe 5 x16 link.  More threads copy faster but can
    // make the whole call SLOWER: the copy bursts take DRAM bandwidth from the DMA reads of the previous chunk.
    // EVK_HOST_COPY_THREADS overrides.
    static const int width = [] { const char *e = getenv("EVK_HOST_COPY_THREADS"); return (e && *e && atoi(e) > 0) ? atoi(e) : 8; }();
    if (k <= 0) return;
    constexpr size_t kBlock = (size_t)1 << 20;
    std::vector<size_t> first((size_t)k + 1, 0);        // first[a] = index of array a's first block
    size_t total = 0;
    for (int a = 0; a < k; ++a) { first[a + 1] = first[a] + (bytes[a] + kBlock - 1) / kBlock; total += bytes[a]; }
    HostPool::get().run(first[k], total < ((size_t)4 << 20) ? 1 : width, [&](size_t b) {
        int a = 0;
        while (first[a + 1] <= b) ++a;
        const size_t off = (b - first[a]) * kBlock, len = (bytes[a] - off < kBlock) ? bytes[a] - off : kBlock;
        copy_block((char *)dst[a] + off, (const char *)src[a] + off, len, stream);
    });
}

// bytes per event a bounce / staging slot holds: x, y, polarity up to 4, timestamps up to 8 (float64 in the storage layout)
constexpr size_t kSlotWidth[4] = {4, 4, 8, 4};
}  // namespace

// the pinned bounce slots of a pipeline (allocated at the first pageable call)
static int ensure_bounce(evk_pipeline *p)
{
    if (p->bounce_events >= p->chunk) return EVK_OK;
    for (int s = 0; s < 2; ++s)
        for (int a = 0; a < 4; ++a) {
            cudaFreeHost(p->bounce[s][a]);
            p->bounce[s][a] = nullptr;
            EVK_CUDA(cudaMallocHost(&p->bounce[s][a], (size_t)p->chunk * kSlotWidth[a]));
        }
    p->bounce_events = p->chunk;
    return EVK_OK;
}

extern "C" {

void evk_host_copy(void *const *dst, const void *const *src, int k, size_t nbytes)
{
    if (!dst || !src || k <= 0) return;
    std::vector<size_t> bytes((size_t)k, nbytes);
    parallel_copy(dst, src, k, bytes.data());
}

int evk_pipeline_create(evk_pipeline_t **out, int64_t chunk_events)
{
    using namespace evk;
    if (!out) { set_error("evk_pipeline_create: null out"); return EVK_E_ARG; }
    if (chunk_events <= 0) chunk_events = (int64_t)4 << 20;
    chunk_events = (chunk_events + 3) & ~(int64_t)3;
    evk_pipeline *p = (evk_pipeline *)calloc(1, sizeof(evk_pipeline));
    if (!p) { set_error("evk_pipeline_create: out of host memory"); return EVK_E_ARG; }
    p->chunk = chunk_events;
    for (int s = 0; s < 2; ++s)
        for (int a = 0; a < 4; ++a)   // slot 2 (timestamps) is 8 bytes wide so that it can also stage float64 stamps
            EVK_CUDA(cudaMalloc(&p->stage[s][a], (size_t)chunk_events * (a == 2 ? sizeof(double) : sizeof(float))));
    EVK_CUDA(cudaStreamCreateWithFlags(&p->copy, cudaStreamNonBlocking));
    EVK_CUDA(cudaStreamCreateWithFlags(&p->compute, cudaStreamNonBlocking));
    for (int s = 0; s < 2; ++s) {
        EVK_CUDA(cudaEventCreateWithFlags(&p->copied[s], cudaEventDisableTiming));
        EVK_CUDA(cudaEventCreateWithFlags(&p->consumed[s], cudaEventDisableTiming));
    }
    EVK_CUDA(cudaMalloc(&p->oob_dev, sizeof(unsigned long long)));
    EVK_CUDA(cudaMallocHost(&p->oob_pinned, sizeof(unsigned long long)));
    *out = p;
    return EVK_OK;
}

void evk_pipeline_destroy(evk_pipeline_t *p)
{
    if (!p) return;
    for (int s = 0; s < 2; ++s) {
        for (int a = 0; a < 4; ++a) cudaFree(p->stage[s][a]);
        if (p->copied[s]) cudaEventDestroy(p->copied[s]);
        if (p->consumed[s]) cudaEventDestroy(p->consumed[s]);
    }
    if (p->copy) cudaStreamDestroy(p->copy);
    if (p->compute) cudaStreamDestroy(p->compute);
    cudaFree(p->grid);
    cudaFree(p->ws);
    cudaFree(p->oob_dev);
    cudaFreeHost(p->oob_pinned);
    for (int s = 0; s < 2; ++s)
        for (int a = 0; a < 4; ++a) cudaFreeHost(p->bounce[s][a]);
    free(p);
}

int evk_voxel_host_f32(evk_pipeline_t *p, const float *x, const float *y, const float *t, const float *pol,
                       int64_t n, float t0, float dt, int B, int H, int W, unsigned flags, float *out_host,
                       unsigned long long *oob_host)
{
    using namespace evk;
    if (!p || !out_host || n < 0 || B < 1 || H < 1 || W < 1 || (n > 0 && (!x || !y || !t || !pol))) {
        set_error("evk_voxel_host_f32: bad arguments");
        return EVK_E_ARG;
    }
    const size_t grid_bytes = (size_t)B * H * W * sizeof(float);
    if (p->grid_bytes < grid_bytes) {
        cudaFree(p->grid);
        p->grid = nullptr; p->grid_bytes = 0;
        EVK_CUDA(cudaMalloc(&p->grid, grid_bytes));
        p->grid_bytes = grid_bytes;
    }
    const size_t ws_bytes = evk_voxel_workspace_bytes(B, H, W, flags);
    if (p->ws_bytes < ws_bytes) {
        cudaFree(p->ws);
        p->ws = nullptr; p->ws_bytes = 0;
        EVK_CUDA(cudaMalloc(&p->ws, ws_bytes));
        p->ws_bytes = ws_bytes;
    }
    EVK_CUDA(cudaMemsetAsync(p->oob_dev, 0, sizeof(unsigned long long), p->compute));
    EVK_CUDA(cudaMemsetAsync(p->grid, 0, grid_bytes, p->compute));
    const float *src[4] = {x, y, t, pol};
    int64_t done = 0;
    int k = 0;
    // ordinary (pageable) host arrays -- what the reference's callers hand over -- go through pinned bounce buffers that
    // a few host threads fill while the previous chunk is on the wire
    const bool bounce = n > 0 && (is_pageable(x) || is_pageable(y) || is_pageable(t) || is_pageable(pol));
    if (bounce) { int rc = ensure_bounce(p); if (rc) return rc; }
    // EVK_AUTO_SPAN: the span of the WHOLE stream, read here from the host arrays; a chunk's kernel would take its own
    if ((flags & EVK_AUTO_SPAN) && n > 0) {
        t0 = t[0];
        dt = t[n - 1] - t[0];
    }
    // every chunk accumulates into the same grid; chunk 0 has already been zeroed above
    const unsigned cflags = (flags & ~(EVK_VARIANT_MASK | EVK_AUTO_SPAN)) | EVK_ACCUMULATE | EVK_VARIANT_GLOBAL_RED;
    while (done < n) {
        const int s = k & 1;
        // pageable sources: a quarter-size first chunk, so that the wire starts after a quarter of a chunk's staging copy
        const int64_t cap = (bounce && k == 0) ? ((p->chunk / 4 + 3) & ~(int64_t)3) : p->chunk;
        const int64_t m = (n - done < cap) ? (n - done) : cap;
        const float *from[4] = {src[0] + done, src[1] + done, src[2] + done, src[3] + done};
        if (bounce) {
            if (k >= 2) EVK_CUDA(cudaEventSynchronize(p->copied[s]));      // the bounce slot's previous H2D has left it
            void *dst4[4] = {p->bounce[s][0], p->bounce[s][1], p->bounce[s][2], p->bounce[s][3]};
            const void *src4[4] = {from[0], from[1], from[2], from[3]};
            const size_t bytes4[4] = {(size_t)m * 4, (size_t)m * 4, (size_t)m * 4, (size_t)m * 4};
            parallel_copy(dst4, src4, 4, bytes4);
            for (int a = 0; a < 4; ++a) from[a] = (const float *)p->bounce[s][a];
        }
        if (k >= 2) EVK_CUDA(cudaStreamWaitEvent(p->copy, p->consumed[s], 0));
        for (int a = 0; a < 4; ++a)
            EVK_CUDA(cudaMemcpyAsync(p->stage[s][a], from[a], (size_t)m * sizeof(float), cudaMemcpyHostToDevice, p->copy));
        EVK_CUDA(cudaEventRecord(p->copied[s], p->copy));
        EVK_CUDA(cudaStreamWaitEvent(p->compute, p->copied[s], 0));
        int rc = evk_voxel_f32(p->stage[s][0], p->stage[s][1], p->stage[s][2], p->stage[s][3], m, t0, dt, B, H, W,
                               cflags, p->grid, nullptr, 0, p->oob_dev, p->compute);
        if (rc) return rc;
        EVK_CUDA(cudaEventRecord(p->consumed[s], p->compute));
        done += m;
        ++k;
    }
    EVK_CUDA(cudaMemcpyAsync(out_host, p->grid, grid_bytes, cudaMemcpyDefault, p->compute));  // out may be host or device
    EVK_CUDA(cudaMemcpyAsync(p->oob_pinned, p->oob_dev, sizeof(unsigned long long), cudaMemcpyDeviceToHost, p->compute));
    EVK_CUDA(cudaStreamSynchronize(p->compute));
    if (oob_host) *oob_host = *p->oob_pinned;
    return EVK_OK;
}

// Plain upload of k host arrays into device buffers the caller allocated (the event set of a contrast-maximisation run,
// numpy inputs of the image functions).  Pageable sources go through the pipeline's pinned bounce slots, four 16 MB
// pieces per round filled by the worker pool while the previous round is on the wire (cudaMemcpyAsync from pageable
// memory is a single-threaded staged copy inside the driver); pinned / registered sources are copied directly.
// Returns when the data is on the device (the copy stream has been synchronised).
int evk_host_upload(evk_pipeline_t *p, void *const *dst_dev, const void *const *src_host, int k, const size_t *nbytes)
{
    using namespace evk;
    if (!p || k < 0 || (k > 0 && (!dst_dev || !src_host || !nbytes))) { set_error("evk_host_upload: bad arguments"); return EVK_E_ARG; }
    for (int a = 0; a < k; ++a)
        if (nbytes[a] && (!dst_dev[a] || !src_host[a])) { set_error("evk_host_upload: null array %d", a); return EVK_E_ARG; }
    const size_t piece = (size_t)p->chunk * 4;          // every bounce buffer holds at least this
    int round = 0;
    void *bdst[4]; const void *bsrc[4]; void *ddst[4]; size_t bbytes[4];
    int filled = 0;
    auto flush_round = [&]() -> int {
        if (!filled) return EVK_OK;
        const int s = round & 1;
        if (round >= 2) EVK_CUDA(cudaEventSynchronize(p->copied[s]));        // the slot's previous H2D has left it
        for (int i = 0; i < filled; ++i) bdst[i] = p->bounce[s][i];
        parallel_copy(bdst, bsrc, filled, bbytes);
        for (int i = 0; i < filled; ++i) EVK_CUDA(cudaMemcpyAsync(ddst[i], bdst[i], bbytes[i], cudaMemcpyHostToDevice, p->copy));
        EVK_CUDA(cudaEventRecord(p->copied[s], p->copy));
        ++round;
        filled = 0;
        return EVK_OK;
    };
    for (int a = 0; a < k; ++a) {
        if (!nbytes[a]) continue;
        if (!is_pageable(src_host[a])) {
            EVK_CUDA(cudaMemcpyAsync(dst_dev[a], src_host[a], nbytes[a], cudaMemcpyHostToDevice, p->copy));
            continue;
        }
        { int rc = ensure_bounce(p); if (rc) return rc; }
        for (size_t off = 0; off < nbytes[a]; off += piece) {
            bsrc[filled] = (const char *)src_host[a] + off;
            ddst[filled] = (char *)dst_dev[a] + off;
            bbytes[filled] = (nbytes[a] - off < piece) ? nbytes[a] - off : piece;
            if (++filled == 4) { int rc = flush_round(); if (rc) return rc; }
        }
    }
    { int rc = flush_round(); if (rc) return rc; }
    EVK_CUDA(cudaStreamSynchronize(p->copy));
    return EVK_OK;
}

// Same pipeline for the storage layout (int16 x, int16 y, float64 t, uint8 p): 13 B/event cross PCIe
// instead of 16, and the casts happen on the device (evk_voxel_packed_f32).
int evk_voxel_host_packed_f32(evk_pipeline_t *p, const int16_t *x, const int16_t *y, const double *t, const uint8_t *pol,
                              int64_t n, double t_first, double t_last, int B, int H, int W, unsigned flags, float *out_host,
                              unsigned long long *oob_host)
{
    using namespace evk;
    if (!p || !out_host || n < 0 || B < 1 || H < 1 || W < 1 || (n > 0 && (!x || !y || !t || !pol))) {
        set_error("evk_voxel_host_packed_f32: bad arguments");
        return EVK_E_ARG;
    }
    const size_t grid_bytes = (size_t)B * H * W * sizeof(float);
    if (p->grid_bytes < grid_bytes) {
        cudaFree(p->grid);
        p->grid = nullptr; p->grid_bytes = 0;
        EVK_CUDA(cudaMalloc(&p->grid, grid_bytes));
        p->grid_bytes = grid_bytes;
    }
    EVK_CUDA(cudaMemsetAsync(p->oob_dev, 0, sizeof(unsigned long long), p->compute));
    EVK_CUDA(cudaMemsetAsync(p->grid, 0, grid_bytes, p->compute));
    // EVK_AUTO_SPAN: first and last stamp of the whole stream, as evk_voxel_packed_f32 takes them on the device
    if ((flags & EVK_AUTO_SPAN) && n > 0) {
        t_first = t[0];
        t_last = t[n - 1];
    }
    const unsigned cflags = (flags & ~(EVK_VARIANT_MASK | EVK_AUTO_SPAN)) | EVK_ACCUMULATE | EVK_VARIANT_GLOBAL_RED;
    int64_t done = 0;
    int k = 0;
    // h5py hands over ordinary pageable arrays: pinned bounce slots filled by the worker pool, as in evk_voxel_host_f32
    const bool bounce = n > 0 && (is_pageable(x) || is_pageable(y) || is_pageable(t) || is_pageable(pol));
    if (bounce) { int rc = ensure_bounce(p); if (rc) return rc; }
    while (done < n) {
        const int s = k & 1;
        const int64_t cap = (bounce && k == 0) ? ((p->chunk / 4 + 3) & ~(int64_t)3) : p->chunk;      // as in evk_voxel_host_f32
        const int64_t m = (n - done < cap) ? (n - done) : cap;
        const void *from[4] = {x + done, y + done, t + done, pol + done};
        const size_t bytes4[4] = {(size_t)m * sizeof(int16_t), (size_t)m * sizeof(int16_t), (size_t)m * sizeof(double), (size_t)m * sizeof(uint8_t)};
        if (bounce) {
            if (k >= 2) EVK_CUDA(cudaEventSynchronize(p->copied[s]));      // the bounce slot's previous H2D has left it
            void *dst4[4] = {p->bounce[s][0], p->bounce[s][1], p->bounce[s][2], p->bounce[s][3]};
            parallel_copy(dst4, from, 4, bytes4);
            for (int a = 0; a < 4; ++a) from[a] = p->bounce[s][a];
        }
        if (k >= 2) EVK_CUDA(cudaStreamWaitEvent(p->copy, p->consumed[s], 0));
        for (int a = 0; a < 4; ++a) EVK_CUDA(cudaMemcpyAsync(p->stage[s][a], from[a], bytes4[a], cudaMemcpyHostToDevice, p->copy));
        EVK_CUDA(cudaEventRecord(p->copied[s], p->copy));
        EVK_CUDA(cudaStreamWaitEvent(p->compute, p->copied[s], 0));
        int rc = evk_voxel_packed_f32((const int16_t *)p->stage[s][0], (const int16_t *)p->stage[s][1], (const double *)p->stage[s][2],
                                      (const uint8_t *)p->stage[s][3], m, t_first, t_last, B, H, W, cflags, p->grid, nullptr, 0,
                                      p->oob_dev, p->compute);
        if (rc) return rc;
        EVK_CUDA(cudaEventRecord(p->consumed[s], p->compute));
        done += m;
        ++k;
    }
    EVK_CUDA(cudaMemcpyAsync(out_host, p->grid, grid_bytes, cudaMemcpyDefault, p->compute));
    EVK_CUDA(cudaMemcpyAsync(p->oob_pinned, p->oob_dev, sizeof(unsigned long long), cudaMemcpyDeviceToHost, p->compute));
    EVK_CUDA(cudaStreamSynchronize(p->compute));
    if (oob_host) *oob_host = *p->oob_pinned;
    return EVK_OK;
}

}  // extern "C"
