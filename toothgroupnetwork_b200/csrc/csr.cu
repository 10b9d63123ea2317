// csr.cu -- deterministic, ORDER-EXACT scatter-add backwards of the gather family.
//
// The reference's live callers gather with torch advanced indexing (pointops.queryandgroup pointops.py:94-99,
// pointops.interpolation :177-179, pointnet2_utils.index_points :44-61), whose backward is
// index_put_(accumulate=True): torch sorts the flat indices (stable) and every destination row adds its
// contributions SEQUENTIALLY IN ASCENDING SOURCE POSITION.  A scatter with atomics adds the same numbers in a
// different, run-dependent order; through training-mode BatchNorm those last-bit differences are amplified into
// visibly different parameter gradients (1e-2 relative on gradients that are sums with heavy cancellation), and the
// result is not reproducible run to run.
//
// Here the inverse index is built once per index tensor -- CSR: row_start[n_rows + 1] and, per destination row, the
// source positions in ascending order -- and the backward is a gather: one thread per (row, channel) walks the row's
// list and adds in exactly torch's order.  Bit-identical gradients to the reference's autograd, deterministic, no
// atomics on the value path (the CSR build itself uses integer atomics only for counting / slot assignment, and each
// row's slots are then rank-sorted, so the result does not depend on their order either).
#include <algorithm>

#include "common.cuh"
#include "tgn_b200.h"

namespace tgn {
namespace {

constexpr unsigned FULL = 0xffffffffu;

struct CsrWs {
    int* row_start;     // [n_rows + 1]
    int* cursor;        // [n_rows]
    int* order;         // [M] source positions, ascending inside each row
    int* scratch;       // [M] unsorted slots
};

size_t carve(long long M, int n_rows, CsrWs* ws, unsigned char* base)
{
    size_t off = 0;
    auto take = [&](size_t bytes) { const size_t o = off; off = (off + bytes + 255) & ~static_cast<size_t>(255); return o; };
    const size_t o_rs = take((static_cast<size_t>(n_rows) + 1) * sizeof(int)), o_cur = take(static_cast<size_t>(n_rows) * sizeof(int)),
                 o_ord = take(static_cast<size_t>(M) * sizeof(int)), o_scr = take(static_cast<size_t>(M) * sizeof(int));
    if (ws) {
        ws->row_start = reinterpret_cast<int*>(base + o_rs);
        ws->cursor = reinterpret_cast<int*>(base + o_cur);
        ws->order = reinterpret_cast<int*>(base + o_ord);
        ws->scratch = reinterpret_cast<int*>(base + o_scr);
    }
    return off;
}

__global__ void __launch_bounds__(256) csr_count_kernel(long long M, int n_rows, const int* __restrict__ keys, int* __restrict__ count)
{
    for (long long p = blockIdx.x * 256LL + threadIdx.x; p < M; p += 256LL * gridDim.x) {
        const int r = __ldg(keys + p);
        if (r >= 0 && r < n_rows) atomicAdd(count + r, 1);
    }
}

// exclusive scan of count[0..n) by ONE CTA of 1024 threads (n up to a few 1e5: ~20 us); count -> row_start, cursor = 0
__global__ void __launch_bounds__(1024) csr_scan_kernel(int n_rows, int* __restrict__ row_start, int* __restrict__ cursor)
{
    __shared__ int warp_tot[32];
    __shared__ int carry_s;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) carry_s = 0;
    __syncthreads();
    for (int base = 0; base < n_rows; base += 1024) {
        const int i = base + tid;
        const int v = i < n_rows ? cursor[i] : 0;            // counts were accumulated in `cursor`
        int incl = v;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const int t = __shfl_up_sync(FULL, incl, d);
            if (lane >= d) incl += t;
        }
        if (lane == 31) warp_tot[warp] = incl;
        __syncthreads();
        if (warp == 0) {
            int w = warp_tot[lane];
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const int t = __shfl_up_sync(FULL, w, d);
                if (lane >= d) w += t;
            }
            warp_tot[lane] = w;
        }
        __syncthreads();
        const int carry = carry_s;
        const int excl = carry + (incl - v) + (warp ? warp_tot[warp - 1] : 0);
        if (i < n_rows) { row_start[i] = excl; cursor[i] = 0; }
        __syncthreads();
        if (tid == 1023) carry_s = carry + warp_tot[31];
        __syncthreads();
    }
    if (tid == 0) row_start[n_rows] = carry_s;
}

__global__ void __launch_bounds__(256) csr_fill_kernel(long long M, int n_rows, const int* __restrict__ keys, CsrWs ws)
{
    for (long long p = blockIdx.x * 256LL + threadIdx.x; p < M; p += 256LL * gridDim.x) {
        const int r = __ldg(keys + p);
        if (r >= 0 && r < n_rows) ws.scratch[ws.row_start[r] + atomicAdd(ws.cursor + r, 1)] = static_cast<int>(p);
    }
}

// rank sort of every row's slots (distinct integers): one warp per row, O(d^2 / 32)
__global__ void __launch_bounds__(256) csr_sort_rows_kernel(int n_rows, CsrWs ws)
{
    const int lane = threadIdx.x & 31;
    const int row = blockIdx.x * 8 + (threadIdx.x >> 5);
    if (row >= n_rows) return;
    const int s = ws.row_start[row], e = ws.row_start[row + 1];
    const int d = e - s;
    if (d <= 32) {
        const int v = lane < d ? ws.scratch[s + lane] : INT_MAX;
        int rank = 0;
        for (int j = 0; j < d; ++j) rank += __shfl_sync(FULL, v, j) < v ? 1 : 0;
        if (lane < d) ws.order[s + rank] = v;
        return;
    }
    for (int i = lane; i < d; i += 32) {
        const int v = ws.scratch[s + i];
        int rank = 0;
        for (int j = 0; j < d; ++j) rank += __ldg(ws.scratch + s + j) < v ? 1 : 0;
        ws.order[s + rank] = v;
    }
}

// grad_in[r, :] = sum over the row's source positions p (ascending) of grad_out[p, :]      (index_put accumulate order)
__global__ void __launch_bounds__(256) gather_sum_det_kernel(int n_rows, int c, const int* __restrict__ row_start,
                                                             const int* __restrict__ order, const float* __restrict__ grad_out,
                                                             float* __restrict__ grad_in)
{
    const size_t total = static_cast<size_t>(n_rows) * c;
    for (size_t e = static_cast<size_t>(blockIdx.x) * 256 + threadIdx.x; e < total; e += static_cast<size_t>(gridDim.x) * 256) {
        const int r = static_cast<int>(e / c), ch = static_cast<int>(e - static_cast<size_t>(r) * c);
        float acc = 0.f;
        const int s = __ldg(row_start + r), t = __ldg(row_start + r + 1);
        for (int q = s; q < t; ++q) acc = __fadd_rn(acc, __ldg(grad_out + static_cast<size_t>(__ldg(order + q)) * c + ch));
        grad_in[e] = acc;
    }
}

// Backward of  out[n,:] = sum_i in[idx[n,i],:] * w[n,i]  as the reference's torch loop builds it (pointops.py:177-179):
// k separate index_put accumulations G_i (ascending n, product rounded then added), summed by autograd in the order the
// engine runs them, i = k-1 first:  ((G_{k-1} + G_{k-2}) + ...) + G_0.   Source position p = n*k + i.
template <int KMAX>
// single != 0: ONE index_put over all (n, i) pairs in ascending p -- the backward of
// torch.sum(index_points(points2, idx) * weight, dim=2) (pointnet2_utils.py:340).
__global__ void __launch_bounds__(256) weighted_gather_bwd_det_kernel(int n_rows, int c, int k, int single, const int* __restrict__ row_start,
                                                                      const int* __restrict__ order, const float* __restrict__ grad_out,
                                                                      const float* __restrict__ w, float* __restrict__ grad_in)
{
    const size_t total = static_cast<size_t>(n_rows) * c;
    for (size_t e = static_cast<size_t>(blockIdx.x) * 256 + threadIdx.x; e < total; e += static_cast<size_t>(gridDim.x) * 256) {
        const int r = static_cast<int>(e / c), ch = static_cast<int>(e - static_cast<size_t>(r) * c);
        float acc[KMAX];
        bool any[KMAX];
#pragma unroll
        for (int i = 0; i < KMAX; ++i) { acc[i] = 0.f; any[i] = false; }
        const int s = __ldg(row_start + r), t = __ldg(row_start + r + 1);
        for (int q = s; q < t; ++q) {
            const int p = __ldg(order + q);
            const int n = p / k, i = single ? 0 : p - n * k;
            const float term = __fmul_rn(__ldg(grad_out + static_cast<size_t>(n) * c + ch), __ldg(w + p));
#pragma unroll
            for (int u = 0; u < KMAX; ++u)
                if (u == i) { acc[u] = __fadd_rn(acc[u], term); any[u] = true; }
        }
        (void)any;
        float tot = 0.f;
        bool first = true;
#pragma unroll
        for (int i = KMAX - 1; i >= 0; --i) {
            if (i < (single ? 1 : k)) {
                tot = first ? acc[i] : __fadd_rn(tot, acc[i]);
                first = false;
            }
        }
        grad_in[e] = tot;
    }
}

// c == 1: torch's index_put takes another kernel for slices of one element (indexing_backward_kernel_stride_1, ATen
// Indexing.cu).  For a destination row with d contributions t_0 .. t_{d-1} (ascending source position) and F = 32*floor(d/32):
// lane L sums t_L, t_{32+L}, ... below F sequentially, the 32 lane sums are reduced by shfl_down (offsets 16, 8, 4, 2, 1),
// then lane 0 adds t_F .. t_{d-1} sequentially; d < 32 is the plain sequential sum.  One warp per row reproduces that.
// The weighted form applies it to every index_put (each i, or all positions at once when `single`); w == nullptr is the
// plain gather backward (term = grad_out[p]).  A row's list is walked twice in chunks of 32: once to count every index_put's
// d, once to hand each term to the lane that adds it (through shared memory) or to lane 0's tail.
template <int KMAX>
__global__ void __launch_bounds__(256) gather_c1_det_kernel(int n_rows, int k, int single, const int* __restrict__ row_start,
                                                            const int* __restrict__ order, const float* __restrict__ grad_out,
                                                            const float* __restrict__ w, float* __restrict__ grad_in)
{
    __shared__ float xch_s[8][32];
    __shared__ float tail_s[8][KMAX][32];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const int row = blockIdx.x * 8 + wid;
    if (row >= n_rows) return;
    const int nk = single ? 1 : k;
    const int s = __ldg(row_start + row), t = __ldg(row_start + row + 1);
    const unsigned lt = (1u << lane) - 1u;
    int d[KMAX];
#pragma unroll
    for (int u = 0; u < KMAX; ++u) d[u] = 0;
    if (nk == 1) {
        d[0] = t - s;
    } else {
        for (int q0 = s; q0 < t; q0 += 32) {
            const int q = q0 + lane;
            const int i = q < t ? __ldg(order + q) % k : -1;
#pragma unroll
            for (int u = 0; u < KMAX; ++u) d[u] += __popc(__ballot_sync(FULL, i == u));
        }
    }
    float acc[KMAX];
    int cnt[KMAX];
#pragma unroll
    for (int u = 0; u < KMAX; ++u) { acc[u] = 0.f; cnt[u] = 0; }
    for (int q0 = s; q0 < t; q0 += 32) {
        const int q = q0 + lane;
        int i = -1;
        float term = 0.f;
        if (q < t) {
            const int p = __ldg(order + q);
            if (w) {
                const int n = p / k;
                i = single ? 0 : p - n * k;
                term = __fmul_rn(__ldg(grad_out + n), __ldg(w + p));
            } else {
                i = 0;
                term = __ldg(grad_out + p);
            }
        }
#pragma unroll
        for (int u = 0; u < KMAX; ++u) {
            if (u >= nk) break;
            const unsigned mask = __ballot_sync(FULL, i == u);
            const int full = d[u] & ~31;
            if (i == u) {
                const int j = cnt[u] + __popc(mask & lt);
                if (j < full) xch_s[wid][j & 31] = term;
                else tail_s[wid][u][j - full] = term;
            }
            __syncwarp();
            const int want = cnt[u] + ((lane - cnt[u]) & 31);       // the rank this lane adds, if this chunk holds it
            if (want < cnt[u] + __popc(mask) && want < full) acc[u] = __fadd_rn(acc[u], xch_s[wid][lane]);
            __syncwarp();
            cnt[u] += __popc(mask);
        }
    }
    float tot = 0.f;
#pragma unroll
    for (int u = KMAX - 1; u >= 0; --u) {
        if (u >= nk) continue;
        float g = acc[u];
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) g = __fadd_rn(g, __shfl_down_sync(FULL, g, off));
        for (int j = d[u] & ~31; j < d[u]; ++j) g = __fadd_rn(g, tail_s[wid][u][j - (d[u] & ~31)]);
        g = __fadd_rn(0.f, g);                                      // index_put adds into the zero-filled gradient
        tot = u == nk - 1 ? g : __fadd_rn(tot, g);
    }
    if (lane == 0) grad_in[row] = tot;
}

int grid_for_elems(size_t n) { return static_cast<int>(std::min<size_t>((n + 255) / 256, 16 * static_cast<size_t>(sm_count()))); }

}  // namespace
}  // namespace tgn

extern "C" {

size_t tgn_csr_bytes(long long M, int n_rows) { return tgn::carve(M, n_rows, nullptr, nullptr); }

int tgn_csr_build(long long M, int n_rows, const int* keys, void* workspace, void* stream)
{
    using namespace tgn;
    if (n_rows <= 0) return TGN_OK;
    if (!workspace || (M > 0 && !keys)) { set_error("csr_build: null argument"); return TGN_ERR_INVALID; }
    if (M > INT_MAX) { set_error("csr_build: %lld source positions exceed int32", M); return TGN_ERR_INVALID; }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    CsrWs ws{};
    carve(M < 0 ? 0 : M, n_rows, &ws, static_cast<unsigned char*>(workspace));
    if (M <= 0) {           // empty index: every row is empty, and both backwards then write zeros
        if (cudaMemsetAsync(ws.row_start, 0, (static_cast<size_t>(n_rows) + 1) * sizeof(int), st) != cudaSuccess) {
            set_error("csr_build: memset failed: %s", cudaGetErrorString(cudaGetLastError()));
            return TGN_ERR_CUDA;
        }
        return TGN_OK;
    }
    if (cudaMemsetAsync(ws.cursor, 0, static_cast<size_t>(n_rows) * sizeof(int), st) != cudaSuccess) {
        set_error("csr_build: memset failed: %s", cudaGetErrorString(cudaGetLastError()));
        return TGN_ERR_CUDA;
    }
    csr_count_kernel<<<grid_for_elems(static_cast<size_t>(M)), 256, 0, st>>>(M, n_rows, keys, ws.cursor);
    int rc = check_launch("csr_count_kernel");
    if (rc != TGN_OK) return rc;
    csr_scan_kernel<<<1, 1024, 0, st>>>(n_rows, ws.row_start, ws.cursor);
    if ((rc = check_launch("csr_scan_kernel")) != TGN_OK) return rc;
    csr_fill_kernel<<<grid_for_elems(static_cast<size_t>(M)), 256, 0, st>>>(M, n_rows, keys, ws);
    if ((rc = check_launch("csr_fill_kernel")) != TGN_OK) return rc;
    csr_sort_rows_kernel<<<(n_rows + 7) / 8, 256, 0, st>>>(n_rows, ws);
    return check_launch("csr_sort_rows_kernel");
}

int tgn_gather_backward_det(long long M, int n_rows, int c, const void* workspace, const float* grad_out, float* grad_in, void* stream)
{
    using namespace tgn;
    if (n_rows <= 0 || c <= 0) return TGN_OK;
    CsrWs ws{};
    carve(M, n_rows, &ws, const_cast<unsigned char*>(static_cast<const unsigned char*>(workspace)));
    if (c == 1) {
        gather_c1_det_kernel<1><<<(n_rows + 7) / 8, 256, 0, static_cast<cudaStream_t>(stream)>>>(n_rows, 1, 1, ws.row_start, ws.order,
                                                                                                  grad_out, nullptr, grad_in);
        return check_launch("gather_c1_det_kernel");
    }
    gather_sum_det_kernel<<<grid_for_elems(static_cast<size_t>(n_rows) * c), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        n_rows, c, ws.row_start, ws.order, grad_out, grad_in);
    return check_launch("gather_sum_det_kernel");
}

int tgn_weighted_gather_backward_det(long long M, int n_rows, int c, int k, int single, const void* workspace, const float* grad_out,
                                     const float* weight, float* grad_in, void* stream)
{
    using namespace tgn;
    if (n_rows <= 0 || c <= 0) return TGN_OK;
    if (k < 1 || k > 8) { set_error("weighted_gather_backward_det: k=%d outside [1, 8]", k); return TGN_ERR_INVALID; }
    CsrWs ws{};
    carve(M, n_rows, &ws, const_cast<unsigned char*>(static_cast<const unsigned char*>(workspace)));
    const int grid = grid_for_elems(static_cast<size_t>(n_rows) * c);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (c == 1) {
        const int blocks = (n_rows + 7) / 8;
        if (k <= 1 || single) gather_c1_det_kernel<1><<<blocks, 256, 0, st>>>(n_rows, k, single, ws.row_start, ws.order, grad_out, weight, grad_in);
        else if (k <= 3) gather_c1_det_kernel<3><<<blocks, 256, 0, st>>>(n_rows, k, 0, ws.row_start, ws.order, grad_out, weight, grad_in);
        else gather_c1_det_kernel<8><<<blocks, 256, 0, st>>>(n_rows, k, 0, ws.row_start, ws.order, grad_out, weight, grad_in);
        return check_launch("gather_c1_det_kernel");
    }
    if (k <= 1 || single) weighted_gather_bwd_det_kernel<1><<<grid, 256, 0, st>>>(n_rows, c, k, single, ws.row_start, ws.order, grad_out, weight, grad_in);
    else if (k <= 3) weighted_gather_bwd_det_kernel<3><<<grid, 256, 0, st>>>(n_rows, c, k, 0, ws.row_start, ws.order, grad_out, weight, grad_in);
    else weighted_gather_bwd_det_kernel<8><<<grid, 256, 0, st>>>(n_rows, c, k, 0, ws.row_start, ws.order, grad_out, weight, grad_in);
    return check_launch("weighted_gather_bwd_det_kernel");
}

}  // extern "C"
