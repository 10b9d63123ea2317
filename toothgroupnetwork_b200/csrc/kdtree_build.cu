// kdtree_build.cu -- scikit-learn 1.9's KDTree(X, leaf_size) built on the device, bit for bit (DESIGN §3.16): idx_array,
// node_data (idx_start, idx_end, is_leaf; the radius is the host's, tgn_kdtree_radius) and node_bounds of float64 (n,3) points.
//
// scikit-learn builds depth first: init_node (bounds), find_node_split_dim (the first dimension with the largest spread) and
// partition_node_indices, which is libstdc++'s std::nth_element on idx_array[start:end) with the comparator (x[split], index)
// to the midpoint start + n_points / 2.  Node ranges depend on n alone, and a node only reorders its own range, so the nodes
// of one level are independent: here one launch per level runs every node of that level, one CTA per node.
//
//   * bounds: a min/max reduction in float64.  The compiled init_node keeps the running bound when a point equals it, so
//     among equal values (+0.0 / -0.0) the first in idx_array order wins: the reduction carries (value, position).
//   * nth_element: libstdc++'s __introselect, depth limit 2 * floor(log2 n).  Each iteration is __move_median_to_first on
//     one thread, then __unguarded_partition(first + 1, last, pivot = first) done in parallel: with distinct keys and the
//     pivot outside [first + 1, last), the i-th element greater than the pivot counted from the left swaps with the i-th
//     element less than it counted from the right, exactly for the i where the first lies left of the second, and the cut
//     is first + 1 + #(< pivot).  One ranking scan writes the position of every less element at its rank from the left and of
//     every greater element at its rank from the left counted from the slot array's end; one pass swaps the pairs.  The last <= 3 elements are sorted (the
//     insertion sort of a strict total order), and the depth-limit branch (__heap_select + iter_swap) runs on one thread.
//   * memory: a node of at most kSmemElems points works in shared memory (keys, ids, rank slots); a larger one works in the
//     workspace in global memory.  Small nodes get one warp, large ones up to 1024 threads.
#include <climits>
#include <cmath>

#include "common.cuh"
#include "tgn_b200.h"

namespace tgn {
namespace {

constexpr int kSmemElems = 4096;           // 16 bytes per point: 64 KB of keys, ids and rank slots
constexpr int kItems = 4;                  // consecutive positions per thread in a ranking scan chunk
constexpr int kMaxThreads = 1024;

struct KdWs {
    int* id;                               // [n] the permutation being built (idx_array as int32)
    double* key;                           // [n] split-coordinate keys, global-memory nodes
    int* slot;                             // [n] rank slots, global-memory nodes
};

size_t carve(int n, KdWs* ws, unsigned char* base)
{
    size_t off = 0;
    auto take = [&](size_t bytes) { const size_t o = off; off = (off + bytes + 255) & ~static_cast<size_t>(255); return o; };
    const size_t o_id = take(static_cast<size_t>(n) * sizeof(int));
    const size_t o_key = take(static_cast<size_t>(n) * sizeof(double));
    const size_t o_slot = take(static_cast<size_t>(n) * sizeof(int));
    if (ws) {
        ws->id = reinterpret_cast<int*>(base + o_id);
        ws->key = reinterpret_cast<double*>(base + o_key);
        ws->slot = reinterpret_cast<int*>(base + o_slot);
    }
    return off;
}

// n_levels = int(log2(max(1, (n - 1) / leaf_size)) + 1): 1 + the largest k with leaf_size * 2^k <= n - 1 (0 when none).
// For n < 2^31 the float quotient is never within a rounding of a power of two it does not reach, so this is the same.
int tree_levels(int n, int leaf_size)
{
    int k = 0;
    while (static_cast<long long>(leaf_size) << (k + 1) <= static_cast<long long>(n) - 1) ++k;
    return k + 1;
}

struct LevelArgs {
    int n, n_nodes, level;
    const double* xyz;
    long long* idx_out;
    long long* node_data;                  // (n_nodes, 4) 8-byte fields: idx_start, idx_end, is_leaf, radius
    double* bounds;                        // (2, n_nodes, 3)
    KdWs ws;
};

__device__ __forceinline__ bool less_key(double ka, int ia, double kb, int ib)
{
    return ka == kb ? ia < ib : ka < kb;
}

// (value, position) reductions: the smaller / larger value, the earlier position among equal values
__device__ __forceinline__ void take_min(double& v, int& p, double v2, int p2)
{
    if (v2 < v || (v2 == v && p2 < p)) { v = v2; p = p2; }
}
__device__ __forceinline__ void take_max(double& v, int& p, double v2, int p2)
{
    if (v2 > v || (v2 == v && p2 < p)) { v = v2; p = p2; }
}

// exclusive prefix of v over the block (blockDim.x a multiple of 32), total in `total`; s_warp holds 32 ints
__device__ int block_exclusive_scan(int v, int& total, int* s_warp)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    int incl = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += t;
    }
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    if (warp == 0) {
        int w = lane < nw ? s_warp[lane] : 0;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int t = __shfl_up_sync(0xffffffffu, w, o);
            if (lane >= o) w += t;
        }
        if (lane < nw) s_warp[lane] = w;
    }
    __syncthreads();
    const int off = warp ? s_warp[warp - 1] : 0;
    total = s_warp[nw - 1];
    __syncthreads();
    return off + incl - v;
}

// libstdc++ __adjust_heap + __push_heap on (K, I)[first, first + len)
__device__ void adjust_heap(double* K, int* I, int first, int hole, int len, double vk, int vi)
{
    const int top = hole;
    int second = hole;
    while (second < (len - 1) / 2) {
        second = 2 * (second + 1);
        if (less_key(K[first + second], I[first + second], K[first + second - 1], I[first + second - 1])) --second;
        K[first + hole] = K[first + second];
        I[first + hole] = I[first + second];
        hole = second;
    }
    if ((len & 1) == 0 && second == (len - 2) / 2) {
        second = 2 * (second + 1);
        K[first + hole] = K[first + second - 1];
        I[first + hole] = I[first + second - 1];
        hole = second - 1;
    }
    int parent = (hole - 1) / 2;
    while (hole > top && less_key(K[first + parent], I[first + parent], vk, vi)) {
        K[first + hole] = K[first + parent];
        I[first + hole] = I[first + parent];
        hole = parent;
        parent = (hole - 1) / 2;
    }
    K[first + hole] = vk;
    I[first + hole] = vi;
}

// libstdc++ __heap_select(first, middle, last) followed by iter_swap(first, nth), one thread
__device__ void heap_select_swap(double* K, int* I, int first, int nth, int last)
{
    const int middle = nth + 1, len = middle - first;
    if (len >= 2) {
        for (int parent = (len - 2) / 2;; --parent) {
            adjust_heap(K, I, first, parent, len, K[first + parent], I[first + parent]);
            if (parent == 0) break;
        }
    }
    for (int i = middle; i < last; ++i) {
        if (less_key(K[i], I[i], K[first], I[first])) {
            const double vk = K[i];
            const int vi = I[i];
            K[i] = K[first];
            I[i] = I[first];
            adjust_heap(K, I, first, 0, len, vk, vi);
        }
    }
    const double tk = K[first]; K[first] = K[nth]; K[nth] = tk;
    const int ti = I[first]; I[first] = I[nth]; I[nth] = ti;
}

__device__ __forceinline__ void swap_at(double* K, int* I, int a, int b)
{
    const double tk = K[a]; K[a] = K[b]; K[b] = tk;
    const int ti = I[a]; I[a] = I[b]; I[b] = ti;
}

// std::nth_element(first, nth, last) on (K, I)[0, len) with the whole block; S holds len ints of scratch
__device__ void block_nth_element(double* K, int* I, int* S, int len, int nth, int* s_warp)
{
    int first = 0, last = len;
    int depth = 2 * (31 - __clz(len));
    bool heap = false;
    while (last - first > 3) {
        if (depth == 0) { heap = true; break; }
        --depth;
        if (threadIdx.x == 0) {                                   // __move_median_to_first(first, first+1, mid, last-1)
            const int a = first + 1, b = first + (last - first) / 2, c = last - 1;
            int s;
            if (less_key(K[a], I[a], K[b], I[b])) {
                if (less_key(K[b], I[b], K[c], I[c])) s = b;
                else if (less_key(K[a], I[a], K[c], I[c])) s = c;
                else s = a;
            } else if (less_key(K[a], I[a], K[c], I[c])) s = a;
            else if (less_key(K[b], I[b], K[c], I[c])) s = c;
            else s = b;
            swap_at(K, I, first, s);
        }
        __syncthreads();
        const double kp = K[first];
        const int ip = I[first];
        // ranking scan over [a, last): less elements to S[rank from the left], greater ones to S[n - 1 - rank from the left]
        const int a = first + 1, n = last - a;
        int run_less = 0;
        for (int base = 0; base < n; base += kItems * blockDim.x) {
            const int p0 = base + kItems * threadIdx.x;
            unsigned flags = 0;
            int cnt = 0, valid = 0;
#pragma unroll
            for (int j = 0; j < kItems; ++j) {
                const int p = p0 + j;
                if (p < n) {
                    ++valid;
                    if (less_key(K[a + p], I[a + p], kp, ip)) { flags |= 1u << j; ++cnt; }
                }
            }
            int chunk_less;
            int before = run_less + block_exclusive_scan(cnt, chunk_less, s_warp);
#pragma unroll
            for (int j = 0; j < kItems; ++j) {
                if (j < valid) {
                    const int p = p0 + j;
                    if (flags >> j & 1u) S[before++] = a + p;
                    else S[n - 1 - (p - before)] = a + p;
                }
            }
            run_less += chunk_less;
        }
        __syncthreads();
        // swap pass: the r-th greater from the left with the r-th less from the right while the first lies left of the second
        const int n_less = run_less, pairs = min(n_less, n - n_less);
        for (int r = threadIdx.x; r < pairs; r += blockDim.x) {
            const int pg = S[n - 1 - r], pl = S[n_less - 1 - r];
            if (pg < pl) swap_at(K, I, pg, pl);
        }
        __syncthreads();
        const int cut = a + n_less;
        if (cut <= nth) first = cut;
        else last = cut;
    }
    if (threadIdx.x == 0) {
        if (heap) {
            heap_select_swap(K, I, first, nth, last);
        } else {
            for (int i = first + 1; i < last; ++i)                // insertion sort of <= 3 elements
                for (int j = i; j > first && less_key(K[j], I[j], K[j - 1], I[j - 1]); --j) swap_at(K, I, j, j - 1);
        }
    }
    __syncthreads();
}

__global__ void __launch_bounds__(kMaxThreads) kdtree_level_kernel(LevelArgs a, int smem_mode)
{
    extern __shared__ __align__(16) unsigned char s_dyn[];
    __shared__ int s_warp[32];
    __shared__ double s_v[32][6];
    __shared__ int s_p[32][6];
    __shared__ int s_dim;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nw = blockDim.x >> 5;
    const int node = (1 << a.level) - 1 + blockIdx.x;
    int s = 0, e = a.n;
    for (int b = a.level - 1; b >= 0; --b) {
        const int mid = s + (e - s) / 2;
        if ((blockIdx.x >> b) & 1) s = mid;
        else e = mid;
    }
    const int len = e - s;
    const bool leaf = 2 * node + 1 >= a.n_nodes;
    int* gid = a.ws.id + s;

    // bounds: v[0..2] lower, v[3..5] upper, with the position of the first point that holds them
    double v[6];
    int p[6];
#pragma unroll
    for (int j = 0; j < 3; ++j) { v[j] = INFINITY; v[3 + j] = -INFINITY; p[j] = p[3 + j] = INT_MAX; }
    for (int t = tid; t < len; t += blockDim.x) {
        const int id = a.level == 0 ? t : gid[t];
        const double* x = a.xyz + 3 * static_cast<size_t>(id);
#pragma unroll
        for (int j = 0; j < 3; ++j) {
            const double c = x[j];
            take_min(v[j], p[j], c, t);
            take_max(v[3 + j], p[3 + j], c, t);
        }
    }
#pragma unroll
    for (int j = 0; j < 6; ++j)
        for (int o = 16; o; o >>= 1) {
            const double v2 = __shfl_xor_sync(0xffffffffu, v[j], o);
            const int p2 = __shfl_xor_sync(0xffffffffu, p[j], o);
            if (j < 3) take_min(v[j], p[j], v2, p2);
            else take_max(v[j], p[j], v2, p2);
        }
    if (lane == 0)
#pragma unroll
        for (int j = 0; j < 6; ++j) { s_v[warp][j] = v[j]; s_p[warp][j] = p[j]; }
    __syncthreads();
    if (tid == 0) {
        for (int w = 1; w < nw; ++w)
#pragma unroll
            for (int j = 0; j < 6; ++j) {
                if (j < 3) take_min(v[j], p[j], s_v[w][j], s_p[w][j]);
                else take_max(v[j], p[j], s_v[w][j], s_p[w][j]);
            }
        int dim = 0;
        double best = 0.0;
        for (int j = 0; j < 3; ++j) {
            a.bounds[3 * static_cast<size_t>(node) + j] = v[j];
            a.bounds[3 * (static_cast<size_t>(a.n_nodes) + node) + j] = v[3 + j];
            const double spread = __dsub_rn(v[3 + j], v[j]);
            if (spread > best) { best = spread; dim = j; }
        }
        long long* nd = a.node_data + 4 * static_cast<size_t>(node);
        nd[0] = s; nd[1] = e; nd[2] = leaf ? 1 : 0;
        nd[3] = 0x7ff8000000000000ll;                         // radius: NaN until tgn_kdtree_radius fills it
        s_dim = dim;
    }
    if (leaf) {
        for (int t = tid; t < len; t += blockDim.x) a.idx_out[s + t] = a.level == 0 ? t : gid[t];
        return;
    }
    __syncthreads();
    const int dim = s_dim;
    double* K;
    int* I;
    int* S;
    if (smem_mode) {
        K = reinterpret_cast<double*>(s_dyn);
        I = reinterpret_cast<int*>(K + len);
        S = I + len;
    } else {
        K = a.ws.key + s;
        I = gid;
        S = a.ws.slot + s;
    }
    for (int t = tid; t < len; t += blockDim.x) {
        const int id = a.level == 0 ? t : gid[t];
        K[t] = a.xyz[3 * static_cast<size_t>(id) + dim];
        I[t] = id;
    }
    __syncthreads();
    block_nth_element(K, I, S, len, len / 2, s_warp);
    if (smem_mode)
        for (int t = tid; t < len; t += blockDim.x) gid[t] = I[t];
}

}  // namespace
}  // namespace tgn

extern "C" {

int tgn_kdtree_nodes(int n, int leaf_size)
{
    if (n < 1 || leaf_size < 1 || n > (1 << 30)) return -1;
    return (1 << tgn::tree_levels(n, leaf_size)) - 1;
}

size_t tgn_kdtree_bytes(int n, int leaf_size)
{
    (void)leaf_size;
    return tgn::carve(n > 0 ? n : 1, nullptr, nullptr);
}

int tgn_kdtree_build(int n, int leaf_size, const double* xyz, long long* idx_array, long long* node_data, double* node_bounds,
                     void* workspace, void* stream)
{
    using namespace tgn;
    if (n < 1 || leaf_size < 1 || n > (1 << 30)) {
        set_error("kdtree_build: need 1 <= n <= 2^30 and leaf_size >= 1 (n=%d, leaf_size=%d)", n, leaf_size);
        return TGN_ERR_INVALID;
    }
    if (!xyz || !idx_array || !node_data || !node_bounds || !workspace) {
        set_error("kdtree_build: null argument");
        return TGN_ERR_INVALID;
    }
    const int levels = tree_levels(n, leaf_size);
    LevelArgs a;
    a.n = n; a.n_nodes = (1 << levels) - 1;
    a.xyz = xyz; a.idx_out = idx_array; a.node_data = node_data; a.bounds = node_bounds;
    carve(n, &a.ws, static_cast<unsigned char*>(workspace));
    if (ensure_dynamic_smem(reinterpret_cast<const void*>(kdtree_level_kernel), kSmemElems * 16) != TGN_OK) return TGN_ERR_CUDA;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    for (int level = 0; level < levels; ++level) {
        a.level = level;
        const int nodes = 1 << level;
        const int max_len = static_cast<int>((static_cast<long long>(n) + nodes - 1) / nodes);
        const bool leaf_level = level == levels - 1;
        const int smem_mode = !leaf_level && max_len <= kSmemElems;
        int threads = kMaxThreads;
        if (max_len <= 128) threads = 32;
        else if (max_len <= 1024) threads = 128;
        else if (max_len <= kSmemElems) threads = 256;
        const size_t smem = smem_mode ? static_cast<size_t>(max_len) * 16 : 0;
        kdtree_level_kernel<<<nodes, threads, smem, st>>>(a, smem_mode);
        const int rc = check_launch("kdtree_build");
        if (rc != TGN_OK) return rc;
    }
    return TGN_OK;
}

void tgn_kdtree_radius(int n_nodes, const double* node_bounds, double* node_data)
{
    // init_node's radius: pow(sum_j pow(0.5 * |hi_j - lo_j|, p), 1 / p) with p = 2 held at run time, as in scikit-learn,
    // so that the compiler calls the C library's pow rather than folding it into a multiplication or a square root.
    volatile double p_runtime = 2.0;
    const double p = p_runtime;
    for (int i = 0; i < n_nodes; ++i) {
        double rad = 0.0;
        for (int j = 0; j < 3; ++j)
            rad += pow(0.5 * fabs(node_bounds[3 * (size_t)(n_nodes + i) + j] - node_bounds[3 * (size_t)i + j]), p);
        node_data[4 * (size_t)i + 3] = pow(rad, 1.0 / p);
    }
}

}  // extern "C"
