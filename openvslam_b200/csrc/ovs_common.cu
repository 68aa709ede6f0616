// ovs_common.cu -- error string, launch counter, device selection.
#include "ovs_common.h"

#include <atomic>
#include <sched.h>
#include <string.h>

namespace ovs {

static thread_local char g_err[512] = "";
static std::atomic<uint64_t> g_launches{0};

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

void count_launch(int n) { g_launches.fetch_add((uint64_t)n, std::memory_order_relaxed); }

static std::atomic<int> g_blocking{0};
alignas(64) static std::atomic<uint64_t> g_waits{0};   // its own cache line: every host wait of every thread writes it
bool blocking_waits() { return g_blocking.load(std::memory_order_relaxed) == 1; }
unsigned event_flags() { return blocking_waits() ? (unsigned)cudaEventBlockingSync : (unsigned)cudaEventDefault; }

cudaError_t sync_event(cudaEvent_t ev) {
    g_waits.fetch_add(1, std::memory_order_relaxed);
    if (g_blocking.load(std::memory_order_relaxed) != 2) return cudaEventSynchronize(ev);
    cudaError_t q;
    while ((q = cudaEventQuery(ev)) == cudaErrorNotReady) sched_yield();
    return q;
}

cudaError_t sync_stream(cudaStream_t st) {
    g_waits.fetch_add(1, std::memory_order_relaxed);
    const int mode = g_blocking.load(std::memory_order_relaxed);
    if (mode == 0) return cudaStreamSynchronize(st);
    if (mode == 2) {
        // cooperative polling: near-spin latency while cores are free, fair time slicing once host threads outnumber cores
        cudaError_t q;
        while ((q = cudaStreamQuery(st)) == cudaErrorNotReady) sched_yield();
        return q;
    }
    // one blocking event per host thread and device, created on first use
    constexpr int kMaxDev = 64;
    static thread_local cudaEvent_t ev[kMaxDev] = {};
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    if (dev < 0 || dev >= kMaxDev) return cudaStreamSynchronize(st);
    if (!ev[dev]) {
        e = cudaEventCreateWithFlags(&ev[dev], cudaEventBlockingSync | cudaEventDisableTiming);
        if (e != cudaSuccess) return e;
    }
    e = cudaEventRecord(ev[dev], st);
    if (e != cudaSuccess) return e;
    return cudaEventSynchronize(ev[dev]);
}

int select_device(int device) {
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n == 0) {
        set_error("no CUDA device available (%s); libovs_b200 has no CPU fallback",
                  e == cudaSuccess ? "device count 0" : cudaGetErrorString(e));
        return OVS_ERR_NO_DEVICE;
    }
    if (device < 0 || device >= n) {
        set_error("device ordinal %d out of range (0..%d)", device, n - 1);
        return OVS_ERR_INVALID_ARG;
    }
    cudaDeviceProp prop;
    OVS_CUDA_CHECK(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0) {
        set_error("device %d is sm_%d%d; libovs_b200 is built for sm_90a (H100) only", device, prop.major, prop.minor);
        return OVS_ERR_NO_DEVICE;
    }
    OVS_CUDA_CHECK(cudaSetDevice(device));
    return OVS_OK;
}

}  // namespace ovs

extern "C" const char* ovs_last_error(void) { return ovs::g_err; }
extern "C" const char* ovs_version(void) { return "ovs_b200 0.1 sm_90a"; }
extern "C" uint64_t ovs_kernel_launch_count(void) { return ovs::g_launches.load(); }
extern "C" uint64_t ovs_host_wait_count(void) { return ovs::g_waits.load(); }
extern "C" int ovs_set_wait_mode(int mode) { ovs::g_blocking.store(mode == 1 ? 1 : mode == 2 ? 2 : 0); return OVS_OK; }
