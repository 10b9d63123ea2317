// knn_feat.cu -- exact feature-space k nearest neighbours of DGCNN (models/modules/dgcnn.py:4-10) without the N x N matrix
// (DESIGN §3.11).
//
// The reference computes, per cloud,
//     inner = -2*matmul(x^T, x);  xx = sum(x**2, dim=1);  pairwise_distance = -xx - inner - xx^T;  topk(k, dim=-1)
// and its neighbour sets are partly decided by float32 rounding, so this kernel reproduces each step bitwise:
//
//   * dot_ij: the FFMA chain of cuBLAS's FP32 GEMM, dot = +0, then dot = fma(x_ic, x_jc, dot) for c = 0..C-1 in order (pinned
//     on the H100 by scripts/diag_dgcnn_knn.py; starting from +0 rather than from the first product makes an all -0 sum +0);
//   * v_ij = fl(fl(-xx_j - fl(-2*dot)) - xx_i): the reference's two element-wise subtractions (-2*dot is exact); xx is an input,
//     computed by the caller with the reference's own torch expression;
//   * selection: the k largest by topk's radix key of v (order-preserving on the bits, -0 < +0, every NaN largest), the lower
//     column index first among equal keys -- the order radix select takes them in;
//   * output order: that of topk's sort of the selection.  topk gathers the selection in index order, the entries above the k-th
//     key first, and sorts them by value (a > b, NaN largest, so +0 == -0) with a bitonic network of 32 that is not stable:
//     equal values come out in an order set by the network, which the kernel reproduces step by step (pinned on the H100 by
//     scripts/diag_dgcnn_knn.py).
//
// Layout: a CTA owns 64 query rows of one cloud (16 per warp), staged in shared memory as [c][row]; candidate tiles of 64 columns
// stream through double-buffered shared memory by 4-byte cp.async, so any (b, c, n) strides are read in place (the permuted
// (B, N, C) view of the first layer needs no copy).  Each lane accumulates a 16 x 2 register tile.  Each row's current top k
// lives across the warp's lanes (entry e in lane e, sorted); a candidate is inserted only when it beats the row's k-th entry,
// which after the first tiles is rare.
#include <climits>

#include "common.cuh"
#include "tgn_b200.h"

namespace tgn {
namespace {

constexpr int kWarps = 4;
constexpr int kRowsPerWarp = 16;
constexpr int kRows = kWarps * kRowsPerWarp;      // query rows per CTA
constexpr int kCols = 64;                         // candidate columns per tile, two per lane
constexpr int kThreads = kWarps * 32;
constexpr int kMaxC = 64;
constexpr int kMaxK = 32;
constexpr unsigned FULL = 0xffffffffu;
static_assert(kRows == kCols, "the query rows are staged by load_cols");

__device__ __forceinline__ void cp_async4(float* dst, const float* src, bool valid)
{
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(smem_u32(dst)), "l"(src), "r"(valid ? 4 : 0) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// topk's radix key of a float (TopKTypeConfig<float>::convert)
__device__ __forceinline__ uint32_t radix_key(float v)
{
    const uint32_t b = __float_as_uint(v);
    return v != v ? 0xffffffffu : b ^ ((b & 0x80000000u) ? 0xffffffffu : 0x80000000u);
}
__device__ __forceinline__ float key_value(uint32_t key)
{
    return __uint_as_float((key & 0x80000000u) ? key ^ 0x80000000u : ~key);
}
// (key descending, index ascending): true when entry a comes before entry b
__device__ __forceinline__ bool precedes(uint32_t ka, int ia, uint32_t kb, int ib) { return ka > kb || (ka == kb && ia < ib); }

// columns [col0, col0 + kCols) of cloud x (element (c, n) at c*sc + n*sn) into dst[c][col]; columns >= n are zero-filled
template <int CT>
__device__ __forceinline__ void load_cols(float* dst, const float* x, int C, int n, int col0, long long sc, long long sn)
{
    const int total = C * kCols;
    for (int e = threadIdx.x; e < total; e += kThreads) {
        int c, j;
        if (sn == 1) { c = e / kCols; j = e % kCols; }     // consecutive threads along n
        else         { j = e / C;     c = e % C;     }     // consecutive threads along c (the permuted view)
        const int col = col0 + j;
        cp_async4(dst + c * kCols + j, x + c * sc + static_cast<long long>(col < n ? col : 0) * sn, col < n);
    }
}

__device__ __forceinline__ void load_xx(float* dst, const float* xx, int n, int col0)
{
    for (int j = threadIdx.x; j < kCols; j += kThreads)
        cp_async4(dst + j, xx + (col0 + j < n ? col0 + j : 0), col0 + j < n);
}

// one entry of a row's sorted top-k list per lane (lanes >= k unused): insert (ck, cj) if it ranks among the k best
__device__ __forceinline__ void insert(uint32_t& lk, int& li, uint32_t ck, int cj, int k, int lane)
{
    const int p = __popc(__ballot_sync(FULL, lane < k && precedes(lk, li, ck, cj)));
    const uint32_t uk = __shfl_up_sync(FULL, lk, 1);
    const int ui = __shfl_up_sync(FULL, li, 1);
    if (p < k) {
        if (lane > p) { lk = uk; li = ui; }
        if (lane == p) { lk = ck; li = cj; }
    }
}

// topk sorts its k <= 32 selected entries (in gather order, padded to 32 with invalid entries) by a bitonic network of 32 with
// the comparator a > b (NaN largest), which is not stable: reproduced here with entry e in lane e.
__device__ __forceinline__ bool gt_nan(float a, float b) { return (a != a && b == b) || a > b; }
__device__ __forceinline__ void bitonic_step(float& v, int& id, bool& ok, int lane, int stride, bool dir)
{
    const float ov = __shfl_xor_sync(FULL, v, stride);
    const int oi = __shfl_xor_sync(FULL, id, stride);
    const bool ook = __shfl_xor_sync(FULL, static_cast<int>(ok), stride) != 0;
    const bool is_a = (lane & stride) == 0;
    const bool swap = (gt_nan(is_a ? v : ov, is_a ? ov : v) && (is_a ? ok : ook)) || !(is_a ? ook : ok);
    if (swap == dir) { v = ov; id = oi; ok = ook; }
}
__device__ __forceinline__ void topk_bitonic_sort(float& v, int& id, bool& ok, int lane)
{
#pragma unroll
    for (int size = 2; size < 32; size *= 2)
#pragma unroll
        for (int stride = size / 2; stride > 0; stride /= 2) bitonic_step(v, id, ok, lane, stride, (lane & size) != 0);
#pragma unroll
    for (int stride = 16; stride > 0; stride /= 2) bitonic_step(v, id, ok, lane, stride, false);
}

template <int CT>
__global__ void __launch_bounds__(kThreads, 4)
knn_feat_kernel(int n, int C, int k, const float* __restrict__ x, long long sb, long long sc, long long sn,
                const float* __restrict__ xx, long long* __restrict__ idx, float* __restrict__ val)
{
    extern __shared__ __align__(16) float smem[];
    float* As = smem;                                  // [CT][kRows]
    float* Bs = As + CT * kRows;                       // [2][CT][kCols]
    float* xxj = Bs + 2 * CT * kCols;                  // [2][kCols]
    float* xxi = xxj + 2 * kCols;                      // [kRows]

    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int b = blockIdx.y, row0 = blockIdx.x * kRows;
    x += b * sb;
    xx += static_cast<long long>(b) * n;

    load_cols<CT>(As, x, C, n, row0, sc, sn);          // the query rows, [c][row] like a candidate tile of kRows = kCols
    for (int r = threadIdx.x; r < kRows; r += kThreads)
        cp_async4(xxi + r, xx + (row0 + r < n ? row0 + r : 0), row0 + r < n);
    load_cols<CT>(Bs, x, C, n, 0, sc, sn);
    load_xx(xxj, xx, n, 0);
    cp_async_commit();

    uint32_t lk[kRowsPerWarp];
    int li[kRowsPerWarp];
#pragma unroll
    for (int r = 0; r < kRowsPerWarp; ++r) { lk[r] = 0u; li[r] = INT_MAX; }   // below every real key (key 0 is never made)

    const int tiles = (n + kCols - 1) / kCols;
    for (int t = 0; t < tiles; ++t) {
        const int buf = t & 1;
        if (t + 1 < tiles) {
            load_cols<CT>(Bs + (buf ^ 1) * CT * kCols, x, C, n, (t + 1) * kCols, sc, sn);
            load_xx(xxj + (buf ^ 1) * kCols, xx, n, (t + 1) * kCols);
            cp_async_commit();
            cp_async_wait<1>();
        } else {
            cp_async_wait<0>();
        }
        __syncthreads();

        const float* B = Bs + buf * CT * kCols;
        float acc[kRowsPerWarp][2];
#pragma unroll
        for (int c = 0; c < CT; ++c) {
            if (c >= C) break;
            const float4* a4 = reinterpret_cast<const float4*>(As + c * kRows + warp * kRowsPerWarp);
            const float2 bv = *reinterpret_cast<const float2*>(B + c * kCols + 2 * lane);
            float a[kRowsPerWarp];
#pragma unroll
            for (int q = 0; q < kRowsPerWarp / 4; ++q) {
                const float4 v = a4[q];
                a[4 * q] = v.x; a[4 * q + 1] = v.y; a[4 * q + 2] = v.z; a[4 * q + 3] = v.w;
            }
#pragma unroll
            for (int r = 0; r < kRowsPerWarp; ++r) {
                acc[r][0] = __fmaf_rn(a[r], bv.x, c == 0 ? 0.0f : acc[r][0]);
                acc[r][1] = __fmaf_rn(a[r], bv.y, c == 0 ? 0.0f : acc[r][1]);
            }
        }

        const int j0 = t * kCols + 2 * lane, j1 = j0 + 1;
        const float nxj0 = -xxj[buf * kCols + 2 * lane], nxj1 = -xxj[buf * kCols + 2 * lane + 1];
#pragma unroll
        for (int r = 0; r < kRowsPerWarp; ++r) {
            const float xi = xxi[warp * kRowsPerWarp + r];
            const uint32_t k0 = radix_key(__fsub_rn(__fsub_rn(nxj0, __fmul_rn(-2.0f, acc[r][0])), xi));
            const uint32_t k1 = radix_key(__fsub_rn(__fsub_rn(nxj1, __fmul_rn(-2.0f, acc[r][1])), xi));
            const uint32_t tk = __shfl_sync(FULL, lk[r], k - 1);
            const int ti = __shfl_sync(FULL, li[r], k - 1);
            unsigned m0 = __ballot_sync(FULL, j0 < n && precedes(k0, j0, tk, ti));
            unsigned m1 = __ballot_sync(FULL, j1 < n && precedes(k1, j1, tk, ti));
            while (m0 | m1) {
                const bool first = m0 != 0;
                const int src = __ffs(first ? m0 : m1) - 1;
                if (first) m0 &= m0 - 1; else m1 &= m1 - 1;
                const uint32_t ck = __shfl_sync(FULL, first ? k0 : k1, src);
                const int cj = __shfl_sync(FULL, first ? j0 : j1, src);
                insert(lk[r], li[r], ck, cj, k, lane);
            }
        }
        __syncthreads();                               // buffer buf is refilled by the next iteration's prefetch
    }

#pragma unroll
    for (int r = 0; r < kRowsPerWarp; ++r) {
        const int row = row0 + warp * kRowsPerWarp + r;
        // gather order: the entries above the k-th key in index order, then those equal to it (already in index order)
        const uint32_t kth = __shfl_sync(FULL, lk[r], k - 1);
        const unsigned above = __ballot_sync(FULL, lane < k && lk[r] > kth);
        int g = lane;
        if (above & (above - 1)) {
            int rank = 0;
            for (int m = 0; m < 32; ++m) {
                const int im = __shfl_sync(FULL, li[r], m);
                rank += ((above >> m) & 1u) && im < li[r];
            }
            if ((above >> lane) & 1u) g = rank;
            int from = lane;
            for (int m = 0; m < 32; ++m)
                if (__shfl_sync(FULL, g, m) == lane) from = m;
            lk[r] = __shfl_sync(FULL, lk[r], from);
            li[r] = __shfl_sync(FULL, li[r], from);
        }
        float v = lane < k ? key_value(lk[r]) : 0.0f;
        int id = lane < k ? li[r] : 0;
        bool ok = lane < k;
        topk_bitonic_sort(v, id, ok, lane);
        if (row < n && lane < k) {
            const long long o = (static_cast<long long>(b) * n + row) * k + lane;
            idx[o] = id;
            if (val) val[o] = v;
        }
    }
}

template <int CT>
int launch(int b, int n, int c, int k, const float* x, long long sb, long long sc, long long sn, const float* xx, long long* idx,
           float* val, cudaStream_t st)
{
    const size_t smem = sizeof(float) * (CT * kRows + 2 * CT * kCols + 2 * kCols + kRows);
    const int rc = ensure_dynamic_smem(reinterpret_cast<const void*>(&knn_feat_kernel<CT>), smem);
    if (rc != TGN_OK) return rc;
    const dim3 grid((n + kRows - 1) / kRows, b);
    knn_feat_kernel<CT><<<grid, kThreads, smem, st>>>(n, c, k, x, sb, sc, sn, xx, idx, val);
    return check_launch("knn_feat_kernel");
}

}  // namespace
}  // namespace tgn

extern "C" {

int tgn_knn_feat(int b, int n, int c, int k, const float* x, long long stride_b, long long stride_c, long long stride_n,
                 const float* xx, long long* idx, float* val, void* stream)
{
    using namespace tgn;
    if (b < 0 || c < 1 || c > kMaxC || k < 1 || k > kMaxK || n < k || n > INT_MAX / 2) {
        set_error("knn_feat: need b >= 0, 1 <= c <= %d, 1 <= k <= %d, n >= k (b=%d n=%d c=%d k=%d)", kMaxC, kMaxK, b, n, c, k);
        return TGN_ERR_INVALID;
    }
    if (b == 0) return TGN_OK;
    if (!x || !xx || !idx) { set_error("knn_feat: null argument"); return TGN_ERR_INVALID; }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (c <= 8) return launch<8>(b, n, c, k, x, stride_b, stride_c, stride_n, xx, idx, val, st);
    return launch<kMaxC>(b, n, c, k, x, stride_b, stride_c, stride_n, xx, idx, val, st);
}

}  // extern "C"
