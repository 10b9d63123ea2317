// crop_knn.cu -- the k = 3072 nearest points of a handful of query centres (crop extraction), on the GPU.
//
// Between the two stages of every two-stage model the reference copies the cloud to the host, builds a sklearn KDTree
// and queries it for the crop_sample_size = 3072 nearest vertices of each predicted / ground-truth tooth centroid
// (ops_utils.get_nearest_neighbor_idx ops_utils.py:146-161, called at grouping_network_module.py:71-73 and
// tsegnet.py:73), then gathers the crops back on the GPU (:198-218).  That is a k = 3072 selection for <= 16 queries:
// far beyond a register-resident top-k, tiny for a whole CTA.
//
// One CTA per query:
//   1. exact RADIX SELECT of the k-th smallest squared distance: 8 passes over 8-bit digits of the 64-bit key, most
//      significant first; every pass re-evaluates the distances (24 000 points / 1024 threads: ~24 each) and histograms the
//      digit of the keys that still match the prefix in shared memory;
//   2. COMPACTION of the k selected (key, index) pairs into shared memory: everything below the threshold, plus as many
//      threshold-equal points as are needed, lowest index first: when more points tie at the threshold than are taken,
//      sweeps over ascending blocks of 1024 indices rank the equal keys with a block scan, so however many tie, the choice
//      does not depend on scheduling;
//   3. BITONIC SORT of the k pairs (padded to a power of two) by (distance, index), written out in ascending order -- the
//      order KDTree.query(sort_results=True) returns and the second-stage network depends on (its FPS starts at crop row 0).
// Distances are evaluated in float64 on the float32 coordinates, ((dx*dx + dy*dy) + dz*dz) unfused, like sklearn's
// DistanceMetric on the float64 copy it makes of the data: two points swap only if their float64 distances tie exactly.
#include <algorithm>

#include "common.cuh"
#include "tgn_b200.h"

namespace tgn {
namespace {

constexpr int kT = 1024;
constexpr int kMaxK = 4096;
static_assert(kT == 32 * 32, "the compaction's block scan takes one warp total per lane");

__device__ __forceinline__ unsigned long long dist_key(const float* __restrict__ p, double qx, double qy, double qz) {
    const double dx = static_cast<double>(__ldg(p)) - qx, dy = static_cast<double>(__ldg(p + 1)) - qy, dz = static_cast<double>(__ldg(p + 2)) - qz;
    const double d = __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
    return static_cast<unsigned long long>(__double_as_longlong(d));      // d >= 0: the bit pattern orders like the value
}

template <typename IdxT>
__global__ void __launch_bounds__(kT) crop_knn_kernel(int N, int Q, int k, int kpad, const float* __restrict__ xyz,
                                                      const float* __restrict__ centres, IdxT* __restrict__ out)
{
    extern __shared__ __align__(16) unsigned char dyn[];
    unsigned long long* skey = reinterpret_cast<unsigned long long*>(dyn);            // [kpad]
    int* sidx = reinterpret_cast<int*>(skey + kpad);                                  // [kpad]
    __shared__ unsigned hist[256];
    __shared__ unsigned s_wcnt[2][kT / 32];                                           // threshold-equal keys per warp
    __shared__ unsigned long long s_prefix;
    __shared__ int s_need, s_count, s_eq;

    const int tid = threadIdx.x;
    const int b = blockIdx.y, q = blockIdx.x;
    const float* pts = xyz + 3 * static_cast<size_t>(b) * N;
    const float* c = centres + 3 * (static_cast<size_t>(b) * Q + q);
    const double qx = static_cast<double>(__ldg(c)), qy = static_cast<double>(__ldg(c + 1)), qz = static_cast<double>(__ldg(c + 2));
    const int kk = min(k, N);

    // ---- 1. radix select: after the loop s_prefix is the kk-th smallest key, s_need how many keys EQUAL to it are taken and
    //         s_eq how many there are ----
    if (tid == 0) { s_prefix = 0ull; s_need = kk; s_count = 0; }
    __syncthreads();
    for (int pass = 0; pass < 8; ++pass) {
        const int shift = 56 - 8 * pass;
        for (int i = tid; i < 256; i += kT) hist[i] = 0;
        __syncthreads();
        const unsigned long long prefix = s_prefix;
        const unsigned long long hi_mask = pass == 0 ? 0ull : (~0ull << (shift + 8));
        for (int j = tid; j < N; j += kT) {
            const unsigned long long key = dist_key(pts + 3 * static_cast<size_t>(j), qx, qy, qz);
            if ((key & hi_mask) == prefix) atomicAdd(&hist[(key >> shift) & 0xFF], 1u);
        }
        __syncthreads();
        if (tid == 0) {
            int need = s_need;
            unsigned d = 0;
            for (; d < 256; ++d) {
                if (static_cast<int>(hist[d]) >= need) break;
                need -= static_cast<int>(hist[d]);
            }
            s_prefix = prefix | (static_cast<unsigned long long>(d) << shift);
            s_need = need;                                   // still to be found inside digit d
            s_eq = static_cast<int>(hist[d]);                // keys inside digit d; after the last pass, keys == the kk-th
        }
        __syncthreads();
    }
    const unsigned long long thr = s_prefix;
    const int need_eq = s_need;                              // number of keys == thr that belong to the answer
    const bool all_eq = s_eq == need_eq;                     // all of them: nothing to choose

    // ---- 2. compaction ----------------------------------------------------------------------------------------------
    // The kk - need_eq keys below thr, and the threshold-equal keys when all of them are taken, go to [0, kk) in arrival
    // order (the sort orders them).
    for (int j = tid; j < N; j += kT) {
        const unsigned long long key = dist_key(pts + 3 * static_cast<size_t>(j), qx, qy, qz);
        if (key < thr || (all_eq && key == thr)) {
            const int pos = atomicAdd(&s_count, 1);
            skey[pos] = key; sidx[pos] = j;
        }
    }
    // More keys equal thr than are taken: the need_eq of lowest index go to [kk - need_eq, kk).  Each sweep covers kT
    // consecutive indices, one per thread, and a block scan (a ballot per warp, then the warp totals) gives every equal key
    // the number of equal keys at lower indices; the sweeps stop once need_eq are placed.
    if (!all_eq) {
        const int lane = tid & 31, warp = tid >> 5;
        int taken = 0;                                       // equal keys at lower indices than this sweep (block-uniform)
        for (int base = 0, sweep = 0; base < N && taken < need_eq; base += kT, ++sweep) {
            const int j = base + tid;
            const bool eq = j < N && dist_key(pts + 3 * static_cast<size_t>(j), qx, qy, qz) == thr;
            const unsigned m = __ballot_sync(0xffffffffu, eq);
            unsigned* wcnt = s_wcnt[sweep & 1];              // alternate: the previous sweep's totals may still be read
            if (lane == 0) wcnt[warp] = __popc(m);
            __syncthreads();
            const unsigned c = wcnt[lane];                   // one warp total per lane (kT / 32 == 32 warps)
            unsigned incl = c;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const unsigned t = __shfl_up_sync(0xffffffffu, incl, o);
                if (lane >= o) incl += t;
            }
            const int rank = taken + static_cast<int>(__shfl_sync(0xffffffffu, incl - c, warp)) + __popc(m & ((1u << lane) - 1u));
            if (eq && rank < need_eq) { skey[kk - need_eq + rank] = thr; sidx[kk - need_eq + rank] = j; }
            taken += static_cast<int>(__shfl_sync(0xffffffffu, incl, 31));
        }
    }
    for (int i = kk + tid; i < kpad; i += kT) { skey[i] = ~0ull; sidx[i] = INT_MAX; }      // padding sorts last
    __syncthreads();

    // ---- 3. bitonic sort by (key, index) -------------------------------------------------------------------------------
    for (int size = 2; size <= kpad; size <<= 1) {
        for (int stride = size >> 1; stride > 0; stride >>= 1) {
            for (int t = tid; t < kpad / 2; t += kT) {
                const int lo = 2 * t - (t & (stride - 1));
                const int hi = lo + stride;
                const bool up = (lo & size) == 0;
                const unsigned long long ka = skey[lo], kb = skey[hi];
                const int ia = sidx[lo], ib = sidx[hi];
                const bool a_gt_b = ka > kb || (ka == kb && ia > ib);
                if (a_gt_b == up) { skey[lo] = kb; skey[hi] = ka; sidx[lo] = ib; sidx[hi] = ia; }
            }
            __syncthreads();
        }
    }
    IdxT* row = out + (static_cast<size_t>(b) * Q + q) * k;
    for (int i = tid; i < k; i += kT) row[i] = static_cast<IdxT>(i < kk ? sidx[i] : 0);
}

}  // namespace
}  // namespace tgn

extern "C" {

int tgn_crop_knn(int B, int N, int Q, int k, const float* xyz, const float* centres, void* out_idx, int idx64, void* stream)
{
    using namespace tgn;
    if (B <= 0 || Q <= 0 || k <= 0) return TGN_OK;
    if (N <= 0 || !xyz || !centres || !out_idx) { set_error("crop_knn: bad arguments"); return TGN_ERR_INVALID; }
    if (k > kMaxK) { set_error("crop_knn: k=%d exceeds %d", k, kMaxK); return TGN_ERR_INVALID; }
    if (B > 65535) { set_error("crop_knn: B=%d exceeds gridDim.y", B); return TGN_ERR_INVALID; }
    int kpad = 2;
    while (kpad < k) kpad <<= 1;
    const size_t smem = static_cast<size_t>(kpad) * (sizeof(unsigned long long) + sizeof(int));
    int rc = idx64 ? ensure_dynamic_smem(reinterpret_cast<const void*>(crop_knn_kernel<long long>), smem)
                   : ensure_dynamic_smem(reinterpret_cast<const void*>(crop_knn_kernel<int>), smem);
    if (rc != TGN_OK) return rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    dim3 grid(Q, B);
    if (idx64) crop_knn_kernel<long long><<<grid, kT, smem, st>>>(N, Q, k, kpad, xyz, centres, static_cast<long long*>(out_idx));
    else crop_knn_kernel<int><<<grid, kT, smem, st>>>(N, Q, k, kpad, xyz, centres, static_cast<int*>(out_idx));
    return check_launch("crop_knn_kernel");
}

}  // extern "C"
