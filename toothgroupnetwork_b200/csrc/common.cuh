// common.cuh -- sm_90a device primitives shared by the kernels of libtgn_b200.so.
// Everything here is inline PTX for Hopper (compile with
// -gencode arch=compute_90a,code=sm_90a); there is no other target.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>

#define TGN_OK 0
#define TGN_ERR_INVALID 1     // argument outside what the path supports (message in tgn_last_error)
#define TGN_ERR_CUDA 2        // a CUDA runtime call or launch failed

namespace tgn {

void set_error(const char* fmt, ...);
int check_launch(const char* what);   // cudaGetLastError -> status (+ message)
int sm_count();                       // of the current device (cached per device)
int ensure_dynamic_smem(const void* func, size_t bytes);   // per (device, kernel) opt-in to > 48 KB of dynamic shared memory
void keep_async_pool();               // configure the default cudaMallocAsync pool to cache freed scratch

// ---------------------------------------------------------------- fp32 pairs
// A pair of floats carried in one 64-bit value.  Each op is two IEEE round-to-nearest fp32 operations, so a
// sequence of pair ops is bit-identical to the same sequence of scalar ops on either half.
__device__ __forceinline__ uint64_t pack2(float lo, float hi) {
    uint64_t r;
    asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(lo), "f"(hi));
    return r;
}
__device__ __forceinline__ void unpack2(uint64_t v, float& lo, float& hi) {
    asm("mov.b64 {%0, %1}, %2;" : "=f"(lo), "=f"(hi) : "l"(v));
}
__device__ __forceinline__ uint64_t sub2(uint64_t a, uint64_t b) {
    float a0, a1, b0, b1;
    unpack2(a, a0, a1);
    unpack2(b, b0, b1);
    return pack2(__fsub_rn(a0, b0), __fsub_rn(a1, b1));
}
__device__ __forceinline__ uint64_t add2(uint64_t a, uint64_t b) {
    float a0, a1, b0, b1;
    unpack2(a, a0, a1);
    unpack2(b, b0, b1);
    return pack2(__fadd_rn(a0, b0), __fadd_rn(a1, b1));
}
__device__ __forceinline__ uint64_t mul2(uint64_t a, uint64_t b) {
    float a0, a1, b0, b1;
    unpack2(a, a0, a1);
    unpack2(b, b0, b1);
    return pack2(__fmul_rn(a0, b0), __fmul_rn(a1, b1));
}
__device__ __forceinline__ uint64_t fma2(uint64_t a, uint64_t b, uint64_t c) {
    float a0, a1, b0, b1, c0, c1;
    unpack2(a, a0, a1);
    unpack2(b, b0, b1);
    unpack2(c, c0, c1);
    return pack2(__fmaf_rn(a0, b0, c0), __fmaf_rn(a1, b1, c1));
}
__device__ __forceinline__ float max3(float a, float b, float c) { return fmaxf(fmaxf(a, b), c); }

// ---------------------------------------------------------------- shared-memory addresses / clusters
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ uint32_t cluster_ctarank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
__device__ __forceinline__ uint32_t map_to_cta(uint32_t local_smem_addr, uint32_t cta) {
    uint32_t r;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(local_smem_addr), "r"(cta));
    return r;
}
__device__ __forceinline__ void cluster_sync_all() {
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}

// ---------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(bar), "r"(parity)
        : "memory");
    return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    while (!mbar_try_wait(bar, parity)) {
    }
}
// Same, but a waiting warp yields its issue slots between probes (for long waits next to busy warps).
__device__ __forceinline__ void mbar_wait_relaxed(uint32_t bar, uint32_t parity) {
    while (!mbar_try_wait(bar, parity)) __nanosleep(64);
}
// Same, but the probe itself may suspend the warp in hardware for up to ~10 ms (no polling instructions
// competing with the warps that have work): for waits on tensor-core completion.
__device__ __forceinline__ void mbar_wait_suspend(uint32_t bar, uint32_t parity) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1, %2;\n\t"
        "@!p bra WAIT_%=;\n\t}"
        ::"r"(bar), "r"(parity), "r"(0x989680u)
        : "memory");
}
// Asynchronous remote store that also completes `bytes` on the destination CTA's mbarrier
// (both addresses are shared::cluster addresses obtained with map_to_cta).
__device__ __forceinline__ void st_async_v4(uint32_t dst, uint32_t a, uint32_t b, uint32_t c, uint32_t d, uint32_t bar) {
    asm volatile("st.async.weak.shared::cluster.mbarrier::complete_tx::bytes.v4.b32 [%0], {%1, %2, %3, %4}, [%5];" ::"r"(dst),
                 "r"(a), "r"(b), "r"(c), "r"(d), "r"(bar)
                 : "memory");
}
__device__ __forceinline__ void st_async_v2(uint32_t dst, uint32_t a, uint32_t b, uint32_t bar) {
    asm volatile("st.async.weak.shared::cluster.mbarrier::complete_tx::bytes.v2.b32 [%0], {%1, %2}, [%3];" ::"r"(dst), "r"(a),
                 "r"(b), "r"(bar)
                 : "memory");
}
__device__ __forceinline__ void st_async_b32(uint32_t dst, uint32_t a, uint32_t bar) {
    asm volatile("st.async.weak.shared::cluster.mbarrier::complete_tx::bytes.b32 [%0], %1, [%2];" ::"r"(dst), "r"(a), "r"(bar)
                 : "memory");
}

// ---------------------------------------------------------------- misc
__device__ __forceinline__ int ilog2_floor(unsigned v) { return 31 - __clz(v); }

}  // namespace tgn
