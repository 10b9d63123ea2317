// kdtree_query.cu -- scikit-learn 1.9's KDTree.query(X, k) (single tree, depth first, sorted) on the device, one warp per
// query row, over the arrays tgn_kdtree_build writes (DESIGN §3.17).  Used for the label transfers' rows whose nearest
// distances tie, where the answer depends on the order of scikit-learn's walk.
//
// What scikit-learn computes for one row, and how it is kept here:
//   * _query_single_depthfirst(node, LB): trim when LB > heap.largest (LB computed by the parent, compared with the heap as
//     it is on entry); a leaf pushes idx_array[idx_start:idx_end] in that order; an inner node visits child 2i+1 first iff
//     LB1 <= LB2.  Here an explicit stack of (node, LB, exact) entries, entry s held by lane s (depth <= n_levels <= 31).
//   * min_rdist: h_j = max(lo_j - q_j, q_j - hi_j, 0) exactly, rdist = ((0 + pow(h0,2)) + pow(h1,2)) + pow(h2,2) with the
//     C library's pow.  The device squares with h*h, which equals pow(h, 2) whenever the product is exact and is within one
//     ulp of it otherwise.  A bound is `exact` when fma(h, h, -h*h) == 0 for all three axes: it is then scikit-learn's bit
//     for bit, and any other bound is within a few ulps.  A row is flagged when a trim or child-order decision involves an
//     inexact bound and its two operands lie within a relative 2^-40: every decision of an unflagged row is scikit-learn's.
//   * leaf distances ((0 + dx*dx) + dy*dy) + dz*dz, computed by the lanes; heap_push (a fixed-size max-heap: rejected when
//     val >= root, the left child taken when values[l] >= values[r]) applied by lane 0 in leaf order, every candidate
//     re-checked against the root after the previous push.
//   * simultaneous_sort: the 2-way introsort (maxd = 2 * floor(log2 k), median of three, Hoare-style partition, heapsort at
//     the depth limit, insertion sort at <= 15 elements) on lane 0.  Its subranges are disjoint, so an explicit task stack
//     in place of the recursion sorts them to the same permutation.
// Every rounding is an explicit __d*_rn / __fma_rn, so nvcc contracts nothing.
#include <climits>
#include <cmath>

#include "common.cuh"
#include "tgn_b200.h"

namespace tgn {
namespace {

constexpr int kWarpsPerBlock = 4;
constexpr int kMaxK = 63;
constexpr int kSortTasks = 16;             // introsort tasks pending: < 2 * floor(log2 63) + 1
constexpr double kBand = 0x1p-40;          // flag margin, relative to the larger operand
constexpr unsigned kFull = 0xffffffffu;

struct QueryArgs {
    int n_nodes, k, m, n_rows;
    const double* xyz;                     // (n,3) points in their original order
    const long long* idx_array;            // (n) tree position -> point
    const long long* node_data;            // (n_nodes,4) idx_start, idx_end, is_leaf, radius (unused)
    const double* bounds;                  // (2,n_nodes,3) lower corners, then upper corners
    const double* queries;                 // (m,3)
    const long long* rows;                 // (n_rows) rows to answer, or NULL for all m
    long long* idx;                        // (m,k)
    double* dist;                          // (m,k) or NULL
    unsigned char* flag;                   // (m)
};

// min_rdist of node for q, with h*h for pow(h, 2); exact = every square is exact
__device__ __forceinline__ double min_rdist(const double* bounds, int n_nodes, int node, const double q[3], bool& exact)
{
    const double* lo = bounds + 3 * static_cast<size_t>(node);
    const double* hi = bounds + 3 * (static_cast<size_t>(n_nodes) + node);
    double r = 0.0;
    exact = true;
#pragma unroll
    for (int j = 0; j < 3; ++j) {
        const double h = fmax(fmax(__dsub_rn(lo[j], q[j]), __dsub_rn(q[j], hi[j])), 0.0);
        const double hh = __dmul_rn(h, h);
        exact &= __fma_rn(h, h, -hh) == 0.0;
        r = __dadd_rn(r, hh);
    }
    return r;
}

// whether a decision between a and b (finite, >= 0) could go the other way under a few ulps of error in one operand
__device__ __forceinline__ bool close(double a, double b)
{
    return b < INFINITY && fabs(__dsub_rn(a, b)) <= __dmul_rn(kBand, fmax(a, b));
}

// utils/_heap.pyx heap_push after its rejection test (val < v[0])
__device__ __forceinline__ void heap_push(double* v, int* ix, int size, double val, int vi)
{
    int cur = 0;
    while (true) {
        const int l = 2 * cur + 1, r = l + 1;
        int sw;
        if (l >= size) break;
        if (r >= size) {
            if (v[l] > val) sw = l;
            else break;
        } else if (v[l] >= v[r]) {
            if (val < v[l]) sw = l;
            else break;
        } else {
            if (val < v[r]) sw = r;
            else break;
        }
        v[cur] = v[sw];
        ix[cur] = ix[sw];
        cur = sw;
    }
    v[cur] = val;
    ix[cur] = vi;
}

__device__ __forceinline__ void swap_at(double* v, int* ix, int a, int b)
{
    const double t = v[a]; v[a] = v[b]; v[b] = t;
    const int u = ix[a]; ix[a] = ix[b]; ix[b] = u;
}

// utils/_sorting.pyx sift_down / heapsort / insertion_sort / inplace_median3
__device__ __forceinline__ void sift_down(double* v, int* ix, int start, int end)
{
    int root = start;
    while (true) {
        const int child = 2 * root + 1;
        int maxind = root;
        if (child < end && v[maxind] < v[child]) maxind = child;
        if (child + 1 < end && v[maxind] < v[child + 1]) maxind = child + 1;
        if (maxind == root) break;
        swap_at(v, ix, root, maxind);
        root = maxind;
    }
}

__device__ __forceinline__ void heapsort(double* v, int* ix, int n)
{
    for (int start = (n - 2) / 2;; --start) {
        sift_down(v, ix, start, n);
        if (start == 0) break;
    }
    for (int end = n - 1; end > 0; --end) {
        swap_at(v, ix, 0, end);
        sift_down(v, ix, 0, end);
    }
}

__device__ __forceinline__ void insertion_sort(double* v, int* ix, int n)
{
    for (int i = 1; i < n; ++i) {
        const double tv = v[i];
        const int ti = ix[i];
        int j = i;
        while (j > 0 && v[j - 1] > tv) {
            v[j] = v[j - 1];
            ix[j] = ix[j - 1];
            --j;
        }
        v[j] = tv;
        ix[j] = ti;
    }
}

__device__ __forceinline__ double median3(double* v, int* ix, int n)
{
    const int p = n / 2;
    if (v[0] > v[n - 1]) swap_at(v, ix, 0, n - 1);
    if (v[n - 1] > v[p]) {
        swap_at(v, ix, n - 1, p);
        if (v[0] > v[n - 1]) swap_at(v, ix, 0, n - 1);
    }
    return v[n - 1];
}

// simultaneous_sort(v, ix, n) with introsort_2way; tasks: kSortTasks ints of scratch (offset | len << 8 | maxd << 16)
__device__ __forceinline__ void simultaneous_sort(double* v, int* ix, int n, int* tasks)
{
    int top = 0;
    tasks[top++] = n << 8 | (2 * (31 - __clz(n))) << 16;
    while (top) {
        const int t = tasks[--top];
        int off = t & 0xff, len = t >> 8 & 0xff, maxd = t >> 16;
        bool sorted = false;
        while (len > 15) {
            if (maxd <= 0) {
                heapsort(v + off, ix + off, len);
                sorted = true;
                break;
            }
            --maxd;
            double* w = v + off;
            int* wi = ix + off;
            const double pivot = median3(w, wi, len);
            int i = 1, j = len - 2;
            while (true) {
                while (i <= j && w[i] < pivot) ++i;
                while (i <= j && w[j] > pivot) --j;
                if (i >= j) break;
                swap_at(w, wi, i, j);
                ++i;
                --j;
            }
            swap_at(w, wi, i, len - 1);
            tasks[top++] = off | i << 8 | maxd << 16;          // the left part [0, i), sorted later: disjoint ranges
            off += i + 1;
            len -= i + 1;
        }
        if (!sorted) insertion_sort(v + off, ix + off, len);
    }
}

__global__ void __launch_bounds__(kWarpsPerBlock * 32) kdtree_query_kernel(QueryArgs a)
{
    __shared__ double s_val[kWarpsPerBlock][kMaxK];
    __shared__ int s_ind[kWarpsPerBlock][kMaxK];
    __shared__ int s_task[kWarpsPerBlock][kSortTasks];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const long long j = static_cast<long long>(blockIdx.x) * kWarpsPerBlock + w;
    if (j >= (a.rows ? a.n_rows : a.m)) return;                // whole warps leave together
    const long long row = a.rows ? a.rows[j] : j;
    if (row < 0 || row >= a.m) return;
    const int k = a.k;
    double* hv = s_val[w];                                     // the heap: lane 0 alone reads and writes it
    int* hi = s_ind[w];
    if (lane == 0)
        for (int t = 0; t < k; ++t) { hv[t] = INFINITY; hi[t] = 0; }
    const double q[3] = {a.queries[3 * row], a.queries[3 * row + 1], a.queries[3 * row + 2]};

    bool ex;
    double st_lb = min_rdist(a.bounds, a.n_nodes, 0, q, ex);   // lane s holds stack entry s
    int st_node = 0;
    bool st_ex = ex;
    int sp = 1;
    double largest = INFINITY;                                 // the heap's root, uniform over the warp
    bool flagged = false;
    while (sp > 0) {
        --sp;
        const int node = __shfl_sync(kFull, st_node, sp);
        const double lb = __shfl_sync(kFull, st_lb, sp);
        const bool lb_ex = __shfl_sync(kFull, static_cast<int>(st_ex), sp);
        flagged |= !lb_ex && close(lb, largest);
        if (lb > largest) continue;                            // trimmed
        const long long* nd = a.node_data + 4 * static_cast<size_t>(node);
        if (nd[2]) {
            const int end = static_cast<int>(nd[1]);
            for (int base = static_cast<int>(nd[0]); base < end; base += 32) {
                const int p = base + lane;
                double rd = INFINITY;
                int id = 0;
                if (p < end) {
                    id = static_cast<int>(a.idx_array[p]);
                    const double* x = a.xyz + 3 * static_cast<size_t>(id);
                    const double dx = __dsub_rn(q[0], x[0]), dy = __dsub_rn(q[1], x[1]), dz = __dsub_rn(q[2], x[2]);
                    rd = __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
                }
                unsigned cand = __ballot_sync(kFull, rd < largest);
                while (cand) {                                 // leaf order
                    const int b = __ffs(cand) - 1;
                    cand &= cand - 1;
                    const double v = __shfl_sync(kFull, rd, b);
                    const int vi = __shfl_sync(kFull, id, b);
                    if (v < largest) {
                        double root = 0.0;
                        if (lane == 0) {
                            heap_push(hv, hi, k, v, vi);
                            root = hv[0];
                        }
                        largest = __shfl_sync(kFull, root, 0);
                    }
                }
            }
        } else {
            const int i1 = 2 * node + 1, i2 = i1 + 1;
            bool ex1, ex2;
            const double lb1 = min_rdist(a.bounds, a.n_nodes, i1, q, ex1);
            const double lb2 = min_rdist(a.bounds, a.n_nodes, i2, q, ex2);
            flagged |= !(ex1 && ex2) && close(lb1, lb2);
            const bool first1 = lb1 <= lb2;
            if (lane == sp) {                                  // visited second: pushed first
                st_node = first1 ? i2 : i1; st_lb = first1 ? lb2 : lb1; st_ex = first1 ? ex2 : ex1;
            } else if (lane == sp + 1) {
                st_node = first1 ? i1 : i2; st_lb = first1 ? lb1 : lb2; st_ex = first1 ? ex1 : ex2;
            }
            sp += 2;
        }
    }
    if (lane == 0) {
        simultaneous_sort(hv, hi, k, s_task[w]);
        a.flag[row] = flagged ? 1 : 0;
    }
    __syncwarp();
    long long* out_idx = a.idx + row * k;
    for (int t = lane; t < k; t += 32) out_idx[t] = hi[t];
    if (a.dist) {
        double* out_dist = a.dist + row * k;
        for (int t = lane; t < k; t += 32) out_dist[t] = __dsqrt_rn(hv[t]);
    }
}

}  // namespace
}  // namespace tgn

extern "C" {

int tgn_kdtree_query(int n, int n_nodes, int k, const double* xyz, const long long* idx_array, const long long* node_data,
                     const double* node_bounds, int m, const double* queries, const long long* rows, int n_rows, long long* idx,
                     double* dist, unsigned char* flag, void* stream)
{
    using namespace tgn;
    // a tree of n_levels <= 31 levels, every leaf holding a point: the walk's stack fits one entry per lane
    if (n < 1 || n > (1 << 30) || n_nodes < 1 || (n_nodes & (n_nodes + 1)) != 0 || (n_nodes + 1) / 2 > n) {
        set_error("kdtree_query: need 1 <= n <= 2^30 and n_nodes = 2^L - 1 with 2^(L-1) <= n (n=%d, n_nodes=%d)", n, n_nodes);
        return TGN_ERR_INVALID;
    }
    if (k < 1 || k > kMaxK || k > n) {
        set_error("kdtree_query: need 1 <= k <= min(n, %d) (k=%d, n=%d)", kMaxK, k, n);
        return TGN_ERR_INVALID;
    }
    if (m < 0 || (rows && n_rows < 0)) {
        set_error("kdtree_query: bad row counts m=%d n_rows=%d", m, n_rows);
        return TGN_ERR_INVALID;
    }
    const int count = rows ? n_rows : m;
    if (count == 0 || m == 0) return TGN_OK;
    if (!xyz || !idx_array || !node_data || !node_bounds || !queries || !idx || !flag) {
        set_error("kdtree_query: null argument");
        return TGN_ERR_INVALID;
    }
    QueryArgs a;
    a.n_nodes = n_nodes; a.k = k; a.m = m; a.n_rows = n_rows;
    a.xyz = xyz; a.idx_array = idx_array; a.node_data = node_data; a.bounds = node_bounds;
    a.queries = queries; a.rows = rows; a.idx = idx; a.dist = dist; a.flag = flag;
    const int blocks = (count + kWarpsPerBlock - 1) / kWarpsPerBlock;
    kdtree_query_kernel<<<blocks, kWarpsPerBlock * 32, 0, static_cast<cudaStream_t>(stream)>>>(a);
    return check_launch("kdtree_query");
}

}  // extern "C"
