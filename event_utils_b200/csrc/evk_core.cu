// evk_core.cu -- error reporting, version and device checks of libevk.so.
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>

#include "evk_common.cuh"

namespace evk {

static thread_local char g_err[512] = "";

void set_error(const char *fmt, ...)
{
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

int cuda_fail(cudaError_t e, const char *what)
{
    set_error("CUDA error %d (%s) in %s", (int)e, cudaGetErrorString(e), what);
    return EVK_E_CUDA;
}

int num_sms()
{
    static thread_local int cached_dev = -1, cached_sms = 132;
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 132;
    if (dev != cached_dev) {
        int sms = 132;
        if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && sms > 0) {
            cached_sms = sms;
            cached_dev = dev;
        }
    }
    return cached_sms;
}

double grid_waves()
{
    static double w = -1.0;
    if (w < 0.0) {
        const char *e = getenv("EVK_GRID_WAVES");
        w = (e && atof(e) > 0.0) ? atof(e) : 4.0;  // 4 waves of small CTAs balance the tail (see DESIGN.md section 6)
    }
    return w;
}

int resident_ctas_per_sm(const void *kernel, int threads, size_t dyn_smem)
{
    struct Entry { const void *k; int threads; size_t smem; int ctas; };
    static thread_local Entry cache[64];
    static thread_local int used = 0;
    for (int i = 0; i < used; ++i)
        if (cache[i].k == kernel && cache[i].threads == threads && cache[i].smem == dyn_smem) return cache[i].ctas;
    int ctas = 1;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ctas, kernel, threads, dyn_smem) != cudaSuccess || ctas < 1) {
        cudaGetLastError();
        ctas = 1;
    }
    if (used < 64) cache[used++] = Entry{kernel, threads, dyn_smem, ctas};
    return ctas;
}

// ---- measurement hooks ---------------------------------------------------------------------
static bool g_prof_on = false;
static long long g_launches = 0;
static const int kProfSlots = 4096;
static cudaEvent_t g_prof_ev[kProfSlots][2];
static int g_prof_used = 0, g_prof_created = 0;

void prof_count(int launches)
{
    if (g_prof_on) g_launches += launches;
}

// scopes nest: only the outermost one is timed (a caller that brackets two alternative kernels -- the probe-selected voxel
// kernels -- wants ONE duration for the pair)
static thread_local int g_prof_depth = 0;

ProfScope::ProfScope(cudaStream_t s) : st(s), slot(-1)
{
    if (g_prof_depth++ > 0) return;
    if (!g_prof_on || g_prof_used >= kProfSlots) return;
    if (g_prof_used >= g_prof_created) {
        if (cudaEventCreate(&g_prof_ev[g_prof_created][0]) != cudaSuccess) return;
        if (cudaEventCreate(&g_prof_ev[g_prof_created][1]) != cudaSuccess) return;
        ++g_prof_created;
    }
    slot = g_prof_used++;
    cudaEventRecord(g_prof_ev[slot][0], st);
}

ProfScope::~ProfScope()
{
    --g_prof_depth;
    if (slot >= 0) cudaEventRecord(g_prof_ev[slot][1], st);
}

// Cross-GPU barrier on the stream, for the fused peer kernels (one process per GPU).  Every rank owns `world` 32-bit slots in
// memory that all ranks have mapped (symmetric memory); rank r signals by storing `epoch` into slot [r] of EVERY rank
// (release, system scope) and waits until all of ITS slots have reached `epoch` (acquire).  Epochs only grow, so one slot
// array serves any number of barriers.  One CTA, one thread per peer: a launch plus one NVLink round trip.
constexpr int kMaxBarrierPeers = 16;
struct PeerFlags {
    unsigned *slots[kMaxBarrierPeers];
};

__global__ void __launch_bounds__(32) peer_barrier_kernel(const PeerFlags F, int world, int rank, unsigned epoch)
{
    const int t = threadIdx.x;
    if (t < world) {
        asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(F.slots[t] + rank), "r"(epoch) : "memory");
        unsigned seen;
        do {
            asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(seen) : "l"(F.slots[rank] + t) : "memory");
        } while ((int)(seen - epoch) < 0);
    }
}

}  // namespace evk

extern "C" {

int evk_peer_barrier(unsigned *const *peer_slots, int world, int rank, unsigned epoch, void *stream)
{
    using namespace evk;
    if (!peer_slots || world < 1 || world > kMaxBarrierPeers || rank < 0 || rank >= world) {
        set_error("evk_peer_barrier: bad arguments (world=%d rank=%d, at most %d peers)", world, rank, kMaxBarrierPeers);
        return EVK_E_ARG;
    }
    PeerFlags F{};
    for (int r = 0; r < world; ++r) {
        if (!peer_slots[r]) { set_error("evk_peer_barrier: peer %d: null pointer", r); return EVK_E_ARG; }
        F.slots[r] = peer_slots[r];
    }
    prof_count(1);
    peer_barrier_kernel<<<1, 32, 0, static_cast<cudaStream_t>(stream)>>>(F, world, rank, epoch);
    EVK_CUDA(cudaGetLastError());
    return EVK_OK;
}

int evk_prof_enable(int on)
{
    evk::g_prof_on = on != 0;
    return EVK_OK;
}

int evk_prof_collect(double *ms, long long *timed, long long *launches)
{
    using namespace evk;
    double total = 0.0;
    for (int i = 0; i < g_prof_used; ++i) {
        EVK_CUDA(cudaEventSynchronize(g_prof_ev[i][1]));
        float f = 0.f;
        EVK_CUDA(cudaEventElapsedTime(&f, g_prof_ev[i][0], g_prof_ev[i][1]));
        total += f;
    }
    if (ms) *ms = total;
    if (timed) *timed = g_prof_used;
    if (launches) *launches = g_launches;
    g_prof_used = 0;
    g_launches = 0;
    return EVK_OK;
}

int evk_version(void) { return EVK_VERSION; }

const char *evk_last_error(void) { return evk::g_err; }

int evk_device_check(void)
{
    int dev = 0, major = 0, minor = 0;
    EVK_CUDA(cudaGetDevice(&dev));
    EVK_CUDA(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev));
    EVK_CUDA(cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev));
    if (major != 9 || minor != 0) {
        evk::set_error("libevk is built for sm_90a only; device %d has compute capability %d.%d", dev, major, minor);
        return EVK_E_DEVICE;
    }
    return EVK_OK;
}

}  // extern "C"
