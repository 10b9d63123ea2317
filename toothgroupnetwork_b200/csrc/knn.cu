// knn.cu -- segment-aware k nearest neighbours for sm_90a.
//
// Replaces pointops/src/knnquery/knnquery_cuda_kernel.cu:65-116 of the reference (one THREAD
// per query, a 100-entry max-heap in local memory -- 800 B of stack per thread -- and a
// divergent sift-down inside the scan loop).
//
// Design: one WARP per query, WARPS queries per CTA, the segment's coordinates staged as SoA
// tiles in shared memory.  The k+1 best candidates live in registers as a list sorted across
// the lanes (EPL entries per lane); a step tests 32 points against the current threshold and
// only lanes that beat it are inserted (ballot, shuffle-shift).  Distances use the reference's
// SASS sequence (FMUL dy*dy, FFMA dx*dx+., FFMA dz*dz+.), so values are bit-identical.
//
// Exact tie semantics.  With distinct distances the k smallest in ascending order are unique and
// the list IS the reference's answer.  When two candidates among the k+1 best have EQUAL
// distance, which one the reference keeps and where its in-place heap sort puts it depends on
// its heap history (knnquery_cuda_kernel.cu:21-48, strict '<' at :97).  Such a query (rare on
// real clouds, systematic on meshes with duplicated vertices) is re-run by the same warp with an
// exact emulation of that heap in shared memory: lanes still scan 32 points per step, lane 0
// performs the sift-downs in the reference's order.  Trailing slots of a segment shorter than k
// keep (segment start, 1e10) exactly as the reference leaves them (:88-91).
#include <algorithm>

#include "common.cuh"
#include "tgn_b200.h"

// The reference's launchers return void: a rejected call cannot be signalled to the caller, so say it on stderr
// instead of returning with the outputs untouched (ADVICE r1).
#ifndef TGN_REPORT
#include <cstdio>
#define TGN_REPORT(call) do { if ((call) != TGN_OK) std::fprintf(stderr, "libtgn_b200: %s\n", tgn_last_error()); } while (0)
#endif

namespace tgn {
namespace {

constexpr int kWarps = 8;
constexpr int kTilePts = 1024;
constexpr int kMaxK = 128;          // the reference's own limit is 100 (best_dist[100])
constexpr unsigned FULL = 0xffffffffu;

__device__ __forceinline__ float sq_dist_direct(float qx, float qy, float qz, float x, float y, float z) {
    const float dx = qx - x, dy = qy - y, dz = qz - z;
    float d = __fmul_rn(dy, dy);
    d = __fmaf_rn(dx, dx, d);
    return __fmaf_rn(dz, dz, d);
}

// Reference heap, restated (see oracle/pointops_oracle.c sift_down): executed by lane 0 only.
__device__ __forceinline__ void heap_sift_down(float* d, int* id, int len) {
    int parent = 0;
    for (;;) {
        int kid = 2 * parent + 1;
        if (kid >= len) return;
        if (kid + 1 < len && d[kid + 1] > d[kid]) ++kid;
        if (d[parent] > d[kid]) return;
        const float fd = d[parent]; d[parent] = d[kid]; d[kid] = fd;
        const int fi = id[parent]; id[parent] = id[kid]; id[kid] = fi;
        parent = kid;
    }
}

template <int EPL>
__global__ void __launch_bounds__(kWarps * 32)
knn_warp_kernel(int b, int m, int k, const float* __restrict__ xyz, const float* __restrict__ new_xyz,
                const int* __restrict__ offset, const int* __restrict__ new_offset, int* __restrict__ idx,
                float* __restrict__ dist2)
{
    __shared__ float sx[kTilePts], sy[kTilePts], sz[kTilePts];
    __shared__ float hd[kWarps][kMaxK];
    __shared__ int hi[kWarps][kMaxK];
    __shared__ int range[2];

    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int q = blockIdx.x * kWarps + warp;
    const bool live = q < m;
    int start = 0, end = 0;
    float qx = 0.f, qy = 0.f, qz = 0.f;
    if (live) {
        int seg = 0;
        while (seg < b - 1 && q >= __ldg(new_offset + seg)) ++seg;     // knnquery_cuda_kernel.cu:51-62
        start = seg ? __ldg(offset + seg - 1) : 0;
        end = __ldg(offset + seg);
        qx = __ldg(new_xyz + 3 * static_cast<size_t>(q));
        qy = __ldg(new_xyz + 3 * static_cast<size_t>(q) + 1);
        qz = __ldg(new_xyz + 3 * static_cast<size_t>(q) + 2);
    }
    // union of the point ranges needed by this CTA's queries
    if (threadIdx.x == 0) { range[0] = INT_MAX; range[1] = 0; }
    __syncthreads();
    if (live && lane == 0) { atomicMin(&range[0], start); atomicMax(&range[1], end); }
    __syncthreads();
    const int lo = range[0], hi_end = range[1];

    // sorted list across lanes: entry e = lane * EPL + i, ascending in e
    float ld[EPL];
    int li[EPL];
#pragma unroll
    for (int i = 0; i < EPL; ++i) { ld[i] = 1e10f; li[i] = start; }
    const int kth_lane = k / EPL, kth_sub = k % EPL;       // entry k (0-based) = the (k+1)-th best
    float tau = 1e10f;                                     // insert only when d < tau

    for (int base = lo; base < hi_end; base += kTilePts) {
        const int tile = min(kTilePts, hi_end - base);
        __syncthreads();
        for (int i = threadIdx.x; i < tile; i += kWarps * 32) {
            const size_t p = 3 * static_cast<size_t>(base + i);
            sx[i] = __ldg(xyz + p); sy[i] = __ldg(xyz + p + 1); sz[i] = __ldg(xyz + p + 2);
        }
        __syncthreads();
        if (!live) continue;
        const int t0 = max(start - base, 0), t1 = min(end - base, tile);
        for (int o = t0 & ~31; o < t1; o += 32) {
            const int i = o + lane;
            float d = 1e30f;
            if (i >= t0 && i < t1) d = sq_dist_direct(qx, qy, qz, sx[i], sy[i], sz[i]);
            unsigned mask = __ballot_sync(FULL, d < tau);
            while (mask) {
                const int src = __ffs(mask) - 1;
                mask &= mask - 1;
                const float cd = __shfl_sync(FULL, d, src);
                if (cd < tau) {                            // tau may have dropped since the ballot
                    const int ci = base + o + src;
                    // position = number of entries <= cd (new entry goes after equal ones)
                    int below = 0;
#pragma unroll
                    for (int e = 0; e < EPL; ++e) below += (ld[e] <= cd) ? 1 : 0;
                    const unsigned full_lanes = __ballot_sync(FULL, below == EPL);
                    const int plane = __popc(full_lanes);  // lane that receives the new entry
                    // shift everything at or after the insertion point up by one entry
                    const float up_d = __shfl_up_sync(FULL, ld[EPL - 1], 1);
                    const int up_i = __shfl_up_sync(FULL, li[EPL - 1], 1);
                    if (lane > plane) {
#pragma unroll
                        for (int e = EPL - 1; e > 0; --e) { ld[e] = ld[e - 1]; li[e] = li[e - 1]; }
                        ld[0] = up_d; li[0] = up_i;
                    } else if (lane == plane) {
#pragma unroll
                        for (int e = EPL - 1; e > 0; --e) {
                            if (e > below) { ld[e] = ld[e - 1]; li[e] = li[e - 1]; }
                        }
#pragma unroll
                        for (int e = 0; e < EPL; ++e)
                            if (e == below) { ld[e] = cd; li[e] = ci; }
                    }
                    float tl = ld[0];
#pragma unroll
                    for (int e = 1; e < EPL; ++e) tl = (kth_sub == e) ? ld[e] : tl;
                    tau = __shfl_sync(FULL, tl, kth_lane);
                }
            }
        }
    }
    if (!live) return;

    // ---- tie check over entries 0..k (sentinel entries are identical, not ties) ---------------
    bool tie = false;
    {
        const float prev_last = __shfl_up_sync(FULL, ld[EPL - 1], 1);
#pragma unroll
        for (int e = 0; e < EPL; ++e) {
            const int ent = lane * EPL + e;
            const float prev = e ? ld[e - 1] : prev_last;
            if (ent >= 1 && ent <= k && ld[e] == prev && ld[e] < 1e10f) tie = true;
        }
        tie = __any_sync(FULL, tie);
    }
    int* orow = idx + static_cast<size_t>(q) * k;
    float* drow = dist2 + static_cast<size_t>(q) * k;
    if (!tie) {
#pragma unroll
        for (int e = 0; e < EPL; ++e) {
            const int ent = lane * EPL + e;
            if (ent < k) { orow[ent] = li[e]; drow[ent] = ld[e]; }
        }
        return;
    }

    // ---- exact emulation of the reference heap for this query ---------------------------------
    float* d_heap = hd[warp];
    int* i_heap = hi[warp];
    for (int e = lane; e < k; e += 32) { d_heap[e] = 1e10f; i_heap[e] = start; }
    __syncwarp();
    for (int o = start; o < end; o += 32) {
        const int i = o + lane;
        float d = 1e30f;
        if (i < end) d = sq_dist_direct(qx, qy, qz, __ldg(xyz + 3 * static_cast<size_t>(i)), __ldg(xyz + 3 * static_cast<size_t>(i) + 1),
                                        __ldg(xyz + 3 * static_cast<size_t>(i) + 2));
        unsigned mask = __ballot_sync(FULL, d < d_heap[0]);
        while (mask) {
            const int src = __ffs(mask) - 1;
            mask &= mask - 1;
            const float cd = __shfl_sync(FULL, d, src);
            if (lane == 0 && cd < d_heap[0]) {
                d_heap[0] = cd; i_heap[0] = o + src;
                heap_sift_down(d_heap, i_heap, k);
            }
            __syncwarp();
        }
    }
    if (lane == 0) {
        for (int last = k - 1; last > 0; --last) {           // knnquery_cuda_kernel.cu:39-48
            const float fd = d_heap[0]; d_heap[0] = d_heap[last]; d_heap[last] = fd;
            const int fi = i_heap[0]; i_heap[0] = i_heap[last]; i_heap[last] = fi;
            heap_sift_down(d_heap, i_heap, last);
        }
    }
    __syncwarp();
    for (int e = lane; e < k; e += 32) { orow[e] = i_heap[e]; drow[e] = d_heap[e]; }
}

}  // namespace
}  // namespace tgn

extern "C" {

int tgn_knnquery(int b, int m, int nsample, const float* xyz, const float* new_xyz, const int* offset, const int* new_offset,
                 int* idx, float* dist2, void* stream)
{
    using namespace tgn;
    if (m <= 0 || nsample <= 0) return TGN_OK;
    if (nsample > kMaxK - 1) { set_error("knnquery: nsample=%d exceeds %d", nsample, kMaxK - 1); return TGN_ERR_INVALID; }
    if (b <= 0) { set_error("knnquery: b must be positive"); return TGN_ERR_INVALID; }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int grid = (m + kWarps - 1) / kWarps;
    const int epl = (nsample + 1 + 31) / 32;
    switch (epl) {
        case 1: knn_warp_kernel<1><<<grid, kWarps * 32, 0, st>>>(b, m, nsample, xyz, new_xyz, offset, new_offset, idx, dist2); break;
        case 2: knn_warp_kernel<2><<<grid, kWarps * 32, 0, st>>>(b, m, nsample, xyz, new_xyz, offset, new_offset, idx, dist2); break;
        case 3: knn_warp_kernel<3><<<grid, kWarps * 32, 0, st>>>(b, m, nsample, xyz, new_xyz, offset, new_offset, idx, dist2); break;
        default: knn_warp_kernel<4><<<grid, kWarps * 32, 0, st>>>(b, m, nsample, xyz, new_xyz, offset, new_offset, idx, dist2); break;
    }
    return check_launch("knn_warp_kernel");
}

// Reference signature: no segment count, so the segment search walks new_offset until it finds
// the query's segment exactly like get_bt_idx (knnquery_cuda_kernel.cu:51-62); INT_MAX disables
// the bound (the caller guarantees m <= new_offset[last], as the reference requires).
void knnquery_cuda_launcher(int m, int nsample, const float* xyz, const float* new_xyz, const int* offset,
                            const int* new_offset, int* idx, float* dist2)
{
    TGN_REPORT(tgn_knnquery(INT_MAX, m, nsample, xyz, new_xyz, offset, new_offset, idx, dist2, nullptr));
}

}  // extern "C"
