// tc_common.cuh -- warpgroup-MMA (wgmma) primitives shared by the tensor-core engines of the fused set abstraction
// (sa_mlp_tc.cu: 3xTF32, sa_mlp_tcw.cu: wide layers with bf16x2-split operands) and the batch-statistics layers
// (pw_mlp.cu).  sm_90a inline PTX.
//
// A wgmma is issued by one warpgroup (four consecutive warps, the first a multiple of 4) and computes a 64-row slice
// D[64, N] (+)= A[64, K] * B[N, K]^T with both operands K-major in shared memory and D in registers: thread
// (warp w of the group, lane l) holds rows 16w + l/4 and 16w + l/4 + 8, columns 8i + 2(l%4) and 8i + 2(l%4) + 1 of
// every 8-column block i, as d[4i + 0..1] (first row) and d[4i + 2..3] (second row).
#pragma once
#include <cstdint>

#include "common.cuh"
#include "wgmma_ops.cuh"

namespace tgn {
namespace tc {

constexpr int kTileRows = 128;      // rows of a tile = threads of a tile group (one warpgroup)

// Shared-memory matrix descriptor of a K-major, no-swizzle operand: 8-row x 16-byte core matrices,
// SBO = stride between 8-row groups, LBO = stride between 16-byte K-chunks.
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes = 128) {
    uint64_t d = 0;
    d |= static_cast<uint64_t>((saddr & 0x3FFFFu) >> 4);
    d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFFu) << 16;
    d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFFu) << 32;
    return d;                        // layout type 0 (no swizzle), base offset 0
}
// byte offset -> descriptor increment (the start-address field counts 16-byte units)
__host__ __device__ constexpr uint64_t desc_step(uint32_t bytes) { return bytes >> 4; }

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accesses of an accumulator across the asynchronous MMAs that own it
template <int R>
__device__ __forceinline__ void fence_regs(float (&d)[R]) {
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
__device__ __forceinline__ void proxy_fence_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// named barrier of tile group g (128 threads)
__device__ __forceinline__ void group_sync(int g) { asm volatile("bar.sync %0, %1;" ::"r"(g + 1), "r"(kTileRows) : "memory"); }

// a = hi + lo with hi the tf32 truncation of a (exact split)
__device__ __forceinline__ void split_tf32(float a, uint32_t& hi, uint32_t& lo) {
    hi = __float_as_uint(a) & 0xFFFFE000u;
    lo = __float_as_uint(__fsub_rn(a, __uint_as_float(hi)));
}
__device__ __forceinline__ void st_shared_v4(uint32_t addr, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
    asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}
__device__ __forceinline__ void st_shared_v2(uint32_t addr, uint32_t a, uint32_t b) {
    asm volatile("st.shared.v2.b32 [%0], {%1, %2};" ::"r"(addr), "r"(a), "r"(b) : "memory");
}
__device__ __forceinline__ void st_shared_b32(uint32_t addr, uint32_t a) {
    asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(a) : "memory");
}

// Transposed last layer: d holds D^T[channel, row] of one 64-channel slice, N = 128 tile rows.  Max over each
// neighbourhood of K consecutive rows, then + bias and ReLU (both monotone, so they commute with the max), stored
// channel-first.  `ch0` is this thread's first channel (the second is ch0 + 8).  When K is a multiple of 8 a
// neighbourhood is whole 8-column blocks of the fragment: one running max per thread, flushed at block boundaries.
// Any other K takes one pass over the thread's 32 columns per neighbourhood.
__device__ __forceinline__ void store_neighbourhood_max(const float (&d)[64], int ch0, int cout, const float* __restrict__ bias,
                                                        float* out_b, int S, int s0, int K, int groups)
{
    const int lane = threadIdx.x & 31;
    const bool ok0 = ch0 < cout, ok1 = ch0 + 8 < cout;
    const float b0 = ok0 ? __ldg(bias + ch0) : 0.f, b1 = ok1 ? __ldg(bias + ch0 + 8) : 0.f;
    if (K & 7) {
        const int c0 = 2 * (lane & 3);
        for (int sg = 0; sg < groups; ++sg) {
            const int lo = sg * K, hi = lo + K;
            float m0 = -INFINITY, m1 = -INFINITY;
#pragma unroll
            for (int i = 0; i < 16; ++i) {
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int col = 8 * i + c0 + e;
                    if (col >= lo && col < hi) { m0 = fmaxf(m0, d[4 * i + e]); m1 = fmaxf(m1, d[4 * i + 2 + e]); }
                }
            }
            m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, 1));
            m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, 2));
            m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, 1));
            m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, 2));
            if ((lane & 3) == 0) {
                if (ok0) out_b[static_cast<size_t>(ch0) * S + s0 + sg] = fmaxf(m0 + b0, 0.f);
                if (ok1) out_b[static_cast<size_t>(ch0 + 8) * S + s0 + sg] = fmaxf(m1 + b1, 0.f);
            }
        }
        return;
    }
    const int blocks_per_group = K >> 3;
    float m0 = -INFINITY, m1 = -INFINITY;
    int sg = 0, nb = 0;
#pragma unroll
    for (int i = 0; i < 16; ++i) {
        m0 = fmaxf(m0, fmaxf(d[4 * i], d[4 * i + 1]));
        m1 = fmaxf(m1, fmaxf(d[4 * i + 2], d[4 * i + 3]));
        if (++nb == blocks_per_group) {                      // warp-uniform
            m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, 1));
            m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, 2));
            m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, 1));
            m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, 2));
            if ((lane & 3) == 0 && sg < groups) {
                if (ok0) out_b[static_cast<size_t>(ch0) * S + s0 + sg] = fmaxf(m0 + b0, 0.f);
                if (ok1) out_b[static_cast<size_t>(ch0 + 8) * S + s0 + sg] = fmaxf(m1 + b1, 0.f);
            }
            m0 = m1 = -INFINITY;
            nb = 0;
            ++sg;
        }
    }
}

}  // namespace tc
}  // namespace tgn
