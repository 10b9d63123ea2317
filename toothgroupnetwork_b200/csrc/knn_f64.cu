// knn_f64.cu -- exact float64 k nearest neighbours over a uniform grid, with a fused label vote (DESIGN §3.9).
//
// InferencePipeLine.get_boundary_sampled_feats (inference_pipeline_tgn.py:289-330) asks a scikit-learn KDTree built on the
// 24 000 sampled points for the 40 nearest of every original vertex (1e5 - 2e5 of them), all in float64, and then only needs
// two things per vertex: the label of the nearest point and how many of the 40 share it.  This file answers the query
// exactly as the KDTree does and computes those two numbers in the warp, so the (m, 40) index matrix never reaches HBM.
//
//   * distance: d2 = (dx*dx + dy*dy) + dz*dz in float64, every operation rounded on its own (no contraction) -- the order of
//     scikit-learn's Euclidean reduced distance; the reported distance is the correctly rounded sqrt(d2), which is what
//     KDTree.query returns;
//   * order: the key (d2, index) is a strict total order, so ties go to the lower index and the k best do not depend on the
//     order in which candidates are visited;
//   * grid: a counting sort of the points into about two points per cell (at most kCellsMax cells), cell-sorted records
//     (x, y, z, index);
//   * query: one warp per query keeps the k best in a register list sorted across the lanes and visits growing cubes of cells
//     around the query's (clamped) cell.  After the cube of radius R, a point not yet visited lies beyond one of the cube's
//     faces that is not a face of the grid; its distance is at least the distance L from the query to the nearest such face,
//     computed per axis from the query's own coordinates (so queries outside the points' box are handled like any other).
//     L is shrunk by a slack far larger than the rounding of the cell assignment and of L itself, and the search stops when
//     d2[k-th best] < L^2 * (1 - 1e-12) -- strictly below every d2 an unvisited point can produce -- or when the cube covers
//     the grid.  Stopping later only costs time.
//   * build once, query many times: tgn_knn_f64_build writes the grid into a caller-owned workspace and tgn_knn_f64_query only
//     reads it, so one point set serves any number of query sets and k;
//   * tie flag (optional): the warp keeps the min(k+1, n) best keys and flags the query when two adjacent ones have equal d2.
//     An unflagged query's k neighbours, and their order, are the same under every tie-break rule, so scikit-learn's KDTree
//     (which keeps whichever tied point its walk meets first) returns exactly them; flagged rows are for the caller to resolve.
#include <climits>
#include <cmath>

#include "common.cuh"
#include "tgn_b200.h"

namespace tgn {
namespace {

constexpr int kWarps = 8;                 // queries per CTA, one warp each
constexpr int kMaxK = 64;                 // two list entries per lane
constexpr int kCellsMax = 32768;
constexpr int kScanThreads = 1024;
constexpr unsigned FULL = 0xffffffffu;

struct F64Grid {
    double org[3];
    double cs, inv_cs;
    int dim[3];
};

struct F64Ws {                            // all arrays live in one caller-provided workspace
    F64Grid* grid;
    int* cell_start;                      // [kCellsMax + 1]
    int* cursor;                          // [kCellsMax]: counts, then scatter cursors
    int* cell_of;                         // [n]
    double4* sorted;                      // [n] (x, y, z, original index as long long bits), cell-sorted
};

size_t carve(int n, F64Ws* ws, unsigned char* base)
{
    size_t off = 0;
    auto take = [&](size_t bytes) { const size_t o = off; off = (off + bytes + 255) & ~static_cast<size_t>(255); return o; };
    const size_t o_grid = take(sizeof(F64Grid));
    const size_t o_start = take(static_cast<size_t>(kCellsMax + 1) * sizeof(int));
    const size_t o_cur = take(static_cast<size_t>(kCellsMax) * sizeof(int));
    const size_t o_cell = take(static_cast<size_t>(n) * sizeof(int));
    const size_t o_sorted = take(static_cast<size_t>(n) * sizeof(double4));
    if (ws) {
        ws->grid = reinterpret_cast<F64Grid*>(base + o_grid);
        ws->cell_start = reinterpret_cast<int*>(base + o_start);
        ws->cursor = reinterpret_cast<int*>(base + o_cur);
        ws->cell_of = reinterpret_cast<int*>(base + o_cell);
        ws->sorted = reinterpret_cast<double4*>(base + o_sorted);
    }
    return off;
}

// Cell of a coordinate along one axis, clamped into the grid (NaN lands in cell 0 and can never be a neighbour).
__device__ __forceinline__ int cell_coord(double v, double org, double inv_cs, int dim)
{
    const double t = floor(__dmul_rn(__dsub_rn(v, org), inv_cs));
    return static_cast<int>(fmin(fmax(t, 0.0), static_cast<double>(dim - 1)));
}

// ---- 1. bounding box, cell size, zeroed counters: one CTA ---------------------------------------------------------------
__global__ void __launch_bounds__(kScanThreads) knn_f64_setup_kernel(int n, const double* __restrict__ xyz, F64Ws ws)
{
    __shared__ double s_lo[3][32], s_hi[3][32];
    __shared__ int s_cells;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    double lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
    for (int i = tid; i < n; i += kScanThreads)
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            const double v = xyz[3 * static_cast<size_t>(i) + a];
            lo[a] = fmin(lo[a], v);
            hi[a] = fmax(hi[a], v);
        }
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        for (int o = 16; o; o >>= 1) {
            lo[a] = fmin(lo[a], __shfl_xor_sync(FULL, lo[a], o));
            hi[a] = fmax(hi[a], __shfl_xor_sync(FULL, hi[a], o));
        }
        if (lane == 0) { s_lo[a][warp] = lo[a]; s_hi[a][warp] = hi[a]; }
    }
    __syncthreads();
    if (tid == 0) {
        F64Grid g;
        double ext[3], emax = 0.0;
        bool finite = true;
        for (int a = 0; a < 3; ++a) {
            double l = s_lo[a][0], h = s_hi[a][0];
            for (int w = 1; w < kScanThreads / 32; ++w) { l = fmin(l, s_lo[a][w]); h = fmax(h, s_hi[a][w]); }
            finite = finite && isfinite(l) && isfinite(h);
            g.org[a] = isfinite(l) ? l : 0.0;
            ext[a] = h - l;
            g.dim[a] = 1;
        }
        for (int a = 0; a < 3; ++a) emax = fmax(emax, finite ? ext[a] : 0.0);
        g.cs = 1.0;
        if (emax > 0.0) {
            // about two points per cell of the bounding box, never more than kCellsMax cells (as csrc/knn_grid.cu)
            const double target = fmin(fmax(0.5 * n, 1.0), static_cast<double>(kCellsMax));
            double vol = 1.0;
            for (int a = 0; a < 3; ++a) vol *= fmax(ext[a], 1e-3 * emax);
            double cs = cbrt(vol / target);
            for (int it = 0; it < 200; ++it) {
                const double fx = ext[0] / cs, fy = ext[1] / cs, fz = ext[2] / cs;
                if (fx < 2048.0 && fy < 2048.0 && fz < 2048.0) {
                    g.dim[0] = static_cast<int>(fx) + 1; g.dim[1] = static_cast<int>(fy) + 1; g.dim[2] = static_cast<int>(fz) + 1;
                    if (static_cast<long long>(g.dim[0]) * g.dim[1] * g.dim[2] <= kCellsMax) break;
                }
                g.dim[0] = g.dim[1] = g.dim[2] = 1;
                cs *= 1.26;
            }
            g.cs = cs;
        }
        g.inv_cs = 1.0 / g.cs;
        *ws.grid = g;
        s_cells = g.dim[0] * g.dim[1] * g.dim[2];
    }
    __syncthreads();
    for (int c = tid; c < s_cells; c += kScanThreads) ws.cursor[c] = 0;
}

// ---- 2. histogram ----------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) knn_f64_count_kernel(int n, const double* __restrict__ xyz, F64Ws ws)
{
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i >= n) return;
    const F64Grid g = *ws.grid;
    const double* p = xyz + 3 * static_cast<size_t>(i);
    const int c = (cell_coord(p[2], g.org[2], g.inv_cs, g.dim[2]) * g.dim[1] + cell_coord(p[1], g.org[1], g.inv_cs, g.dim[1])) * g.dim[0]
                  + cell_coord(p[0], g.org[0], g.inv_cs, g.dim[0]);
    ws.cell_of[i] = c;
    atomicAdd(ws.cursor + c, 1);
}

// ---- 3. exclusive scan of the counters: one CTA, kCellsMax / 1024 consecutive cells per thread ----------------------------
__global__ void __launch_bounds__(kScanThreads) knn_f64_scan_kernel(int n, F64Ws ws)
{
    __shared__ int warp_tot[32];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const F64Grid g = *ws.grid;
    const int cells = g.dim[0] * g.dim[1] * g.dim[2];
    constexpr int kPer = kCellsMax / kScanThreads;
    int v[kPer], sum = 0;
#pragma unroll
    for (int i = 0; i < kPer; ++i) {
        const int c = tid * kPer + i;
        v[i] = c < cells ? ws.cursor[c] : 0;
        sum += v[i];
    }
    int incl = sum;
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
    int run = (incl - sum) + (warp ? warp_tot[warp - 1] : 0);
#pragma unroll
    for (int i = 0; i < kPer; ++i) {
        const int c = tid * kPer + i;
        if (c < cells) { ws.cell_start[c] = run; ws.cursor[c] = run; }
        run += v[i];
    }
    if (tid == kScanThreads - 1) ws.cell_start[cells] = n;
}

// ---- 4. scatter --------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) knn_f64_scatter_kernel(int n, const double* __restrict__ xyz, F64Ws ws)
{
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i >= n) return;
    const int pos = atomicAdd(ws.cursor + ws.cell_of[i], 1);
    if (pos < 0 || pos >= n) return;          // cannot happen: the counts of step 2 sum to n
    const double* p = xyz + 3 * static_cast<size_t>(i);
    ws.sorted[pos] = make_double4(p[0], p[1], p[2], __longlong_as_double(static_cast<long long>(i)));
}

// ---- 5. query ----------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ double sq_dist(double qx, double qy, double qz, const double4& p)
{
    const double dx = __dsub_rn(qx, p.x), dy = __dsub_rn(qy, p.y), dz = __dsub_rn(qz, p.z);
    return __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
}

__device__ __forceinline__ bool key_less(double d, int i, double od, int oi) { return d < od || (d == od && i < oi); }

// One warp per query.  TIE: the list holds keep = min(k+1, n) entries instead of k and tie[q] reports an equal adjacent pair of d2.
template <int EPL, bool TIE>
__device__ __forceinline__ void knn_f64_query(int n, int m, int k, const double* __restrict__ queries, const F64Ws& ws,
                                              const int* __restrict__ labels, long long* __restrict__ idx, double* __restrict__ dist,
                                              int* __restrict__ nn0, int* __restrict__ agree, unsigned char* __restrict__ tie)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int q = blockIdx.x * kWarps + warp;
    if (q >= m) return;                                   // warps are independent: no block-level barriers below
    const F64Grid g = *ws.grid;
    const double qc[3] = {queries[3 * static_cast<size_t>(q)], queries[3 * static_cast<size_t>(q) + 1], queries[3 * static_cast<size_t>(q) + 2]};
    const int* __restrict__ cst = ws.cell_start;

    // list entry lane * EPL + e, ascending by (d2, index); empty slots (+inf, INT_MAX) sort last
    double ld[EPL];
    int li[EPL];
#pragma unroll
    for (int e = 0; e < EPL; ++e) { ld[e] = INFINITY; li[e] = INT_MAX; }
    const int keep = TIE ? min(k + 1, n) : k;
    const int kth_lane = (keep - 1) / EPL, kth_sub = (keep - 1) % EPL;
    double tau_d = INFINITY;                              // key of the keep-th entry
    int tau_i = INT_MAX;

    auto scan_range = [&](int p0, int p1) {               // candidates sorted[p0, p1)
        for (int o = p0; o < p1; o += 32) {
            const int s = o + lane;
            double d = INFINITY;
            int ci = INT_MAX;
            if (s < p1) {
                const double4 c = ws.sorted[s];
                d = sq_dist(qc[0], qc[1], qc[2], c);
                ci = static_cast<int>(__double_as_longlong(c.w));
            }
            unsigned mask = __ballot_sync(FULL, key_less(d, ci, tau_d, tau_i));
            while (mask) {
                const int src = __ffs(mask) - 1;
                mask &= mask - 1;
                const double cd = __shfl_sync(FULL, d, src);
                const int cid = __shfl_sync(FULL, ci, src);
                if (!key_less(cd, cid, tau_d, tau_i)) continue;           // warp-uniform: tau is shared
                int below = 0;
#pragma unroll
                for (int e = 0; e < EPL; ++e) below += key_less(ld[e], li[e], cd, cid) ? 1 : 0;
                const int plane = __popc(__ballot_sync(FULL, below == EPL));     // lanes entirely before the candidate
                const double up_d = __shfl_up_sync(FULL, ld[EPL - 1], 1);
                const int up_i = __shfl_up_sync(FULL, li[EPL - 1], 1);
                if (lane > plane) {
#pragma unroll
                    for (int e = EPL - 1; e > 0; --e) { ld[e] = ld[e - 1]; li[e] = li[e - 1]; }
                    ld[0] = up_d; li[0] = up_i;
                } else if (lane == plane) {
#pragma unroll
                    for (int e = EPL - 1; e > 0; --e)
                        if (e > below) { ld[e] = ld[e - 1]; li[e] = li[e - 1]; }
#pragma unroll
                    for (int e = 0; e < EPL; ++e)
                        if (e == below) { ld[e] = cd; li[e] = cid; }
                }
                double td = ld[0];
                int ti = li[0];
#pragma unroll
                for (int e = 1; e < EPL; ++e)
                    if (kth_sub == e) { td = ld[e]; ti = li[e]; }
                tau_d = __shfl_sync(FULL, td, kth_lane);
                tau_i = __shfl_sync(FULL, ti, kth_lane);
            }
        }
    };

    int c[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) c[a] = cell_coord(qc[a], g.org[a], g.inv_cs, g.dim[a]);
    const int nx = g.dim[0], ny = g.dim[1], nz = g.dim[2];
    // covers the rounding of the cell assignment and of the bound itself (a few ulps of these magnitudes)
    const double slack = 1e-9 * (fmax(fmax(fabs(qc[0]), fabs(qc[1])), fabs(qc[2])) + fmax(fmax(fabs(g.org[0]), fabs(g.org[1])), fabs(g.org[2]))
                                 + (max(max(nx, ny), nz) + 1) * g.cs);
    for (int R = 0;; ++R) {
        const int z0 = max(c[2] - R, 0), z1 = min(c[2] + R, nz - 1), y0 = max(c[1] - R, 0), y1 = min(c[1] + R, ny - 1);
        const int x0 = max(c[0] - R, 0), x1 = min(c[0] + R, nx - 1);
        for (int z = z0; z <= z1; ++z) {
            const bool z_old = R > 0 && abs(z - c[2]) < R;
            for (int y = y0; y <= y1; ++y) {
                const int row = (z * ny + y) * nx;
                if (!(z_old && abs(y - c[1]) < R)) {
                    scan_range(cst[row + x0], cst[row + x1 + 1]);
                } else {                                  // rows of the previous cube: only its two x-faces are new
                    if (c[0] - R >= 0) scan_range(cst[row + c[0] - R], cst[row + c[0] - R + 1]);
                    if (c[0] + R <= nx - 1) scan_range(cst[row + c[0] + R], cst[row + c[0] + R + 1]);
                }
            }
        }
        // lower bound on the distance of any unvisited point: the nearest cube face that is not a grid face
        double bound = INFINITY;
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            if (c[a] - R > 0) bound = fmin(bound, qc[a] - (g.org[a] + (c[a] - R) * g.cs) - slack);
            if (c[a] + R < g.dim[a] - 1) bound = fmin(bound, (g.org[a] + (c[a] + R + 1) * g.cs) - qc[a] - slack);
        }
        if (bound == INFINITY) break;                                       // the cube covers the grid
        if (bound > 0.0 && tau_d < bound * bound * (1.0 - 1e-12)) break;    // every unvisited point sorts after the k-th
    }

#pragma unroll
    for (int e = 0; e < EPL; ++e) {
        const int ent = lane * EPL + e;
        if (ent < k) {
            if (idx) idx[static_cast<size_t>(q) * k + ent] = li[e];
            if (dist) dist[static_cast<size_t>(q) * k + ent] = __dsqrt_rn(ld[e]);
        }
    }
    const int first = __shfl_sync(FULL, li[0], 0);
    if (labels) {
        const bool valid = first >= 0 && first < n;       // always, for finite coordinates
        const int l0 = valid ? labels[first] : 0;
        int count = 0;
#pragma unroll
        for (int e = 0; e < EPL; ++e) {
            const int ent = lane * EPL + e;
            const bool same = valid && ent < k && li[e] >= 0 && li[e] < n && labels[li[e]] == l0;
            count += __popc(__ballot_sync(FULL, same));
        }
        if (lane == 0 && agree) agree[q] = count;
    }
    if (lane == 0 && nn0) nn0[q] = first;
    if constexpr (TIE) {
        const double prev = __shfl_up_sync(FULL, ld[EPL - 1], 1);           // the entry before this lane's first
        bool eq = false;
#pragma unroll
        for (int e = 0; e < EPL; ++e) {
            const int ent = lane * EPL + e;
            if (ent >= 1 && ent < keep) eq |= (e ? ld[e - 1] : prev) == ld[e];  // d2 >= +0 and finite: == is bitwise equality
        }
        const bool any = __any_sync(FULL, eq);
        if (lane == 0) tie[q] = any ? 1 : 0;
    }
}

template <int EPL>
__global__ void __launch_bounds__(kWarps * 32, 4)      // four CTAs per SM: ptxas then keeps everything in registers
knn_f64_query_kernel(int n, int m, int k, const double* __restrict__ queries, const F64Ws ws, const int* __restrict__ labels,
                     long long* __restrict__ idx, double* __restrict__ dist, int* __restrict__ nn0, int* __restrict__ agree)
{
    knn_f64_query<EPL, false>(n, m, k, queries, ws, labels, idx, dist, nn0, agree, nullptr);
}

template <int EPL>
__global__ void __launch_bounds__(kWarps * 32, 4)
knn_f64_tie_query_kernel(int n, int m, int k, const double* __restrict__ queries, const F64Ws ws, const int* __restrict__ labels,
                         long long* __restrict__ idx, double* __restrict__ dist, int* __restrict__ nn0, int* __restrict__ agree,
                         unsigned char* __restrict__ tie)
{
    knn_f64_query<EPL, true>(n, m, k, queries, ws, labels, idx, dist, nn0, agree, tie);
}

}  // namespace
}  // namespace tgn

extern "C" {

size_t tgn_knn_f64_bytes(int n)
{
    return tgn::carve(n > 0 ? n : 1, nullptr, nullptr);
}

int tgn_knn_f64_build(int n, const double* xyz, void* workspace, void* stream)
{
    using namespace tgn;
    if (n < 1) { set_error("knn_f64_build: need n >= 1 (n=%d)", n); return TGN_ERR_INVALID; }
    if (!xyz || !workspace) { set_error("knn_f64_build: null argument"); return TGN_ERR_INVALID; }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    F64Ws ws{};
    carve(n, &ws, static_cast<unsigned char*>(workspace));
    knn_f64_setup_kernel<<<1, kScanThreads, 0, st>>>(n, xyz, ws);
    int rc = check_launch("knn_f64_setup_kernel");
    if (rc != TGN_OK) return rc;
    const int blocks = (n + 255) / 256;
    knn_f64_count_kernel<<<blocks, 256, 0, st>>>(n, xyz, ws);
    if ((rc = check_launch("knn_f64_count_kernel")) != TGN_OK) return rc;
    knn_f64_scan_kernel<<<1, kScanThreads, 0, st>>>(n, ws);
    if ((rc = check_launch("knn_f64_scan_kernel")) != TGN_OK) return rc;
    knn_f64_scatter_kernel<<<blocks, 256, 0, st>>>(n, xyz, ws);
    return check_launch("knn_f64_scatter_kernel");
}

int tgn_knn_f64_query(int n, int m, int k, const double* xyz, const double* queries, const void* workspace, const int* labels,
                      long long* idx, double* dist, int* nn0, int* agree, unsigned char* tie, void* stream)
{
    using namespace tgn;
    const int max_k = tie ? kMaxK - 1 : kMaxK;            // the tie flag needs one more list entry
    if (n < 1 || m < 0 || k < 1 || k > max_k || k > n) {
        set_error("knn_f64_query: need 1 <= k <= min(n, %d)%s, m >= 0 (n=%d m=%d k=%d)", max_k, tie ? " with tie" : "", n, m, k);
        return TGN_ERR_INVALID;
    }
    if (m == 0) return TGN_OK;
    if (!xyz || !queries || !workspace) { set_error("knn_f64_query: null argument"); return TGN_ERR_INVALID; }
    if (agree && !labels) { set_error("knn_f64_query: agree needs labels"); return TGN_ERR_INVALID; }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    F64Ws ws{};
    carve(n, &ws, static_cast<unsigned char*>(const_cast<void*>(workspace)));   // read only below
    const int grid = (m + kWarps - 1) / kWarps;
    if (tie) {
        if (k + 1 <= 32)
            knn_f64_tie_query_kernel<1><<<grid, kWarps * 32, 0, st>>>(n, m, k, queries, ws, labels, idx, dist, nn0, agree, tie);
        else
            knn_f64_tie_query_kernel<2><<<grid, kWarps * 32, 0, st>>>(n, m, k, queries, ws, labels, idx, dist, nn0, agree, tie);
        return check_launch("knn_f64_tie_query_kernel");
    }
    if (k <= 32)
        knn_f64_query_kernel<1><<<grid, kWarps * 32, 0, st>>>(n, m, k, queries, ws, labels, idx, dist, nn0, agree);
    else
        knn_f64_query_kernel<2><<<grid, kWarps * 32, 0, st>>>(n, m, k, queries, ws, labels, idx, dist, nn0, agree);
    return check_launch("knn_f64_query_kernel");
}

int tgn_knn_f64(int n, int m, int k, const double* xyz, const double* queries, void* workspace, const int* labels, long long* idx,
                double* dist, int* nn0, int* agree, void* stream)
{
    using namespace tgn;
    if (n < 1 || m < 0 || k < 1 || k > kMaxK || k > n) {
        set_error("knn_f64: need 1 <= k <= min(n, %d), m >= 0 (n=%d m=%d k=%d)", kMaxK, n, m, k);
        return TGN_ERR_INVALID;
    }
    if (m == 0) return TGN_OK;
    if (!xyz || !queries || !workspace) { set_error("knn_f64: null argument"); return TGN_ERR_INVALID; }
    if (agree && !labels) { set_error("knn_f64: agree needs labels"); return TGN_ERR_INVALID; }
    const int rc = tgn_knn_f64_build(n, xyz, workspace, stream);
    if (rc != TGN_OK) return rc;
    return tgn_knn_f64_query(n, m, k, xyz, queries, workspace, labels, idx, dist, nn0, agree, nullptr, stream);
}

}  // extern "C"
