// lib.cu -- library-wide state of libtgn_b200.so: error text, launch counter, device facts.
#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <map>
#include <mutex>
#include <utility>

#include "common.cuh"
#include "tgn_b200.h"

namespace tgn {
namespace {
thread_local char g_err[512] = "";
std::atomic<int> g_launches{0};
}  // namespace

void set_error(const char* fmt, ...)
{
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

int check_launch(const char* what)
{
    g_launches.fetch_add(1, std::memory_order_relaxed);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) {
        set_error("%s: %s", what, cudaGetErrorString(e));
        return TGN_ERR_CUDA;
    }
    return TGN_OK;
}

// cudaFuncAttributeMaxDynamicSharedMemorySize is per (device, kernel): remember the largest value configured for
// each pair (thread-safe) so that a process touching several GPUs configures every one of them.
int ensure_dynamic_smem(const void* func, size_t bytes)
{
    static std::mutex mu;
    static std::map<std::pair<int, const void*>, size_t> configured;
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) { (void)cudaGetLastError(); dev = 0; }
    std::lock_guard<std::mutex> lock(mu);
    size_t& have = configured[{dev, func}];
    if (bytes <= have || bytes <= 48 * 1024) return TGN_OK;
    const cudaError_t e = cudaFuncSetAttribute(func, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(bytes));
    if (e != cudaSuccess) { set_error("cudaFuncSetAttribute(%zu bytes): %s", bytes, cudaGetErrorString(e)); return TGN_ERR_CUDA; }
    have = bytes;
    return TGN_OK;
}

// Stream-ordered scratch (cudaMallocAsync) is used by the bucket FPS and the ball query; keep freed
// blocks in the device's default pool instead of returning them to the OS at every synchronisation.
void keep_async_pool()
{
    static std::atomic<unsigned long long> done{0};      // bit d: device d configured
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) { (void)cudaGetLastError(); return; }
    const unsigned long long bit = 1ull << (dev & 63);
    if (done.load(std::memory_order_relaxed) & bit) return;
    cudaMemPool_t pool;
    if (cudaDeviceGetDefaultMemPool(&pool, dev) == cudaSuccess) {
        unsigned long long thr = ~0ull;
        (void)cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr);
        // A block freed on stream A must not be handed to stream B by making B WAIT for A's free point: chunks of a host
        // pipeline run on several streams and would serialise on each other's scratch.  Opportunistic reuse (the free has
        // already completed) and event-ordered reuse stay on; otherwise the pool grows.
        int off = 0;
        (void)cudaMemPoolSetAttribute(pool, cudaMemPoolReuseAllowInternalDependencies, &off);
    }
    (void)cudaGetLastError();
    done.fetch_or(bit, std::memory_order_relaxed);
}

int sm_count()
{
    static std::atomic<int> cached[64];                   // per device, 0 = unknown
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) { (void)cudaGetLastError(); return 132; }   // H100 SXM
    std::atomic<int>& slot = cached[dev & 63];
    int n = slot.load(std::memory_order_relaxed);
    if (n == 0) {
        if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) { (void)cudaGetLastError(); n = 132; }   // H100 SXM
        slot.store(n, std::memory_order_relaxed);
    }
    return n;
}

}  // namespace tgn

extern "C" {
int tgn_version(void) { return 100; }
const char* tgn_last_error(void) { return tgn::g_err; }
int tgn_launch_count(void) { return tgn::g_launches.load(std::memory_order_relaxed); }
}
