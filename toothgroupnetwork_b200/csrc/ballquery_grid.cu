// ballquery_grid.cu -- ball query through a uniform grid binned by index window, for clouds whose balls are sparse (sm_90a).
//
// query_ball_point (external_libs/pointnet2_utils/pointnet2_utils.py:120-144) returns, per query, the
// nsample SMALLEST point indices whose expanded-form distance satisfies !(d > r2), padded with the
// first of them (N everywhere when the ball is empty).  The tile kernel in ballquery.cu scans the cloud
// in index order until a query is full; when a ball holds well under 1 % of the cloud (SA1 of the
// reference networks: r = 0.1 on a 24 000-vertex arch, ~350 members) that scan reads a tenth of the
// cloud per query.  Here:
//   * bq_grid_build_kernel (one CTA per cloud) bins the points by KEY = window * cells + cell, where
//     window = j / Wsz is the point's index window (Wsz a power of two, 1024 ... 8192) and cell one of the
//     cubic cells no smaller than the query radius (counting sort with shared-memory atomics; at most
//     kMaxCells keys).  A sorted point is one 16-byte record (x, y, z, bits of j); |p|^2 is recomputed at
//     test time with the same rounding.  A tiny estimate kernel decides per cloud beforehand whether the
//     grid pays;
//   * ball_query_grid_kernel (one warp per query) visits the index windows in increasing order.  In a
//     window it tests the points of the cells that intersect the query's box (each x-run of cells is one
//     contiguous segment of the window), spread over the lanes, and records members in a per-warp BITMAP
//     of the window's Wsz indices in shared memory.  The set bits, read in order, are the window's members
//     in ascending index order; the query stops in the first window where it has nsample of them.
// Membership is decided by the computed d alone, so the result is bit-identical to the scan as long as
// no member is left unvisited: the visited box is inflated by a bound on the rounding error of the
// expanded form (|d_fp - |a-b|^2| <= 2^-19 (|a|^2 + |b|^2), generous by > 2x) plus a few ulps of the
// coordinates, and cell indices are monotone functions of the coordinates.
// Clouds flagged "dense" are left to the tile kernel (it skips the flagged-sparse ones and vice versa).
#include <algorithm>
#include <climits>

#include "ballquery.cuh"
#include "common.cuh"
#include "tgn_b200.h"

namespace tgn {
namespace {

constexpr int kBT = 1024;            // build kernel threads
constexpr int kBNW = kBT / 32;
constexpr int kMaxCells = 8192;      // (window, cell) keys: 32 KB of shared-memory counters
constexpr int kMinWinLog = 10;       // index windows of 1024 ...
constexpr int kMaxWinLog = 13;       // ... 8192 points (a 1 KB bitmap per query warp)
constexpr int kQW = 16;              // query warps per CTA
constexpr unsigned FULL = 0xffffffffu;

__device__ __forceinline__ int float_ordered(float f) {
    const int i = __float_as_int(f);
    return i ^ ((i >> 31) & 0x7FFFFFFF);
}
__device__ __forceinline__ float ordered_float(int i) { return __int_as_float(i ^ ((i >> 31) & 0x7FFFFFFF)); }

// Radius of the box a query has to visit: members satisfy |a-b|^2 <= r2 + E with E the rounding bound.
__device__ __forceinline__ float safe_radius(float r2, float an, float bn_max, float cmax) {
    const float e = 1.9073486e-6f * (an + bn_max);                 // 2^-19 (|a|^2 + max |b|^2)
    return sqrtf(fmaxf(r2, 0.f) + e) * 1.000001f + 4.0f * 1.1920929e-7f * cmax;
}
__device__ __forceinline__ int cell_of(float v, float origin, float inv, int dim) {
    return min(dim - 1, max(0, static_cast<int>(floorf((v - origin) * inv))));
}

// Per cloud: does the grid pay?  A subsample of <= kEstPoints points is binned into cells of the
// query radius; the mean population of a point's 27-cell neighbourhood (scaled back to the full cloud)
// estimates the candidates `cand` near a query.  About kBallFrac of them are members, so the index-order
// scan needs L = nsample * N / (kBallFrac * cand) points to fill a query, and the grid kernel visits the
// windows up to L (plus one 2048-point window), i.e. a fraction f = min(1, (L + 2048) / N) of the cloud.
// Cost models in ns per query, fitted on an H100 80GB HBM3 (700 W) with scripts/ball_sweep.py (DESIGN 3.2):
//   tile = kTile * nsample * N / cand (at most the full scan, kTileFull * N)
//   grid = kGBuild * N / S + kGSeg * 9 * f * N / 2048 + kGTest * f * cand
// (the build shared by the cloud's S queries, 9 x-runs of cells per window, f * cand points tested).  Least squares over
// the 63 sweep shapes; the cheaper model wins, and it picks the faster kernel on all of them but two within 10 %.
constexpr float kBallFrac = 0.28f, kTile = 4.3e-3f, kTileFull = 5.6e-4f;
constexpr float kGBuild = 0.071f, kGSeg = 0.040f, kGTest = 5.7e-4f;
constexpr int kET = 256;
constexpr int kEstPoints = 4096;
constexpr int kEstCells = 4096;

__global__ void __launch_bounds__(kET)
bq_grid_estimate_kernel(int N, int S, float r2, int nsample, int force, const float* __restrict__ xyz, BqGridWs ws)
{
    __shared__ int cnt[kEstCells];
    __shared__ int red[6][kET / 32];
    __shared__ float4 s_org;
    __shared__ int4 s_dim;
    __shared__ float s_cost[kET / 32];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int b = blockIdx.x;
    if (force) { if (tid == 0) ws.flag[b] = 1; return; }
    const float* pts = xyz + 3 * static_cast<size_t>(b) * N;
    // sample: runs of 8 consecutive points (three 32-byte sectors) spread evenly over the cloud
    const int nchunk = min(kEstPoints / 8, N / 8);
    const int ns = nchunk > 0 ? nchunk * 8 : N;
    const int cstride = nchunk > 0 ? N / nchunk : 1;
    auto sample = [&](int i) { return nchunk > 0 ? (i >> 3) * cstride + (i & 7) : i; };

    float mn[3] = {INFINITY, INFINITY, INFINITY}, mx[3] = {-INFINITY, -INFINITY, -INFINITY};
    for (int i = tid; i < ns; i += kET) {
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            const float v = __ldg(pts + 3 * static_cast<size_t>(sample(i)) + a);
            mn[a] = fminf(mn[a], v); mx[a] = fmaxf(mx[a], v);
        }
    }
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const int lo = __reduce_min_sync(FULL, float_ordered(mn[a])), hi = __reduce_max_sync(FULL, float_ordered(mx[a]));
        if (lane == 0) { red[a][warp] = lo; red[3 + a][warp] = hi; }
    }
    for (int c = tid; c < kEstCells; c += kET) cnt[c] = 0;
    __syncthreads();
    if (tid == 0) {
        float lo[3], hi[3];
        for (int a = 0; a < 3; ++a) {
            int l = red[a][0], h = red[3 + a][0];
            for (int w = 1; w < kET / 32; ++w) { l = min(l, red[a][w]); h = max(h, red[3 + a][w]); }
            lo[a] = ordered_float(l); hi[a] = ordered_float(h);
        }
        float cs = fmaxf(sqrtf(fmaxf(r2, 0.f)), 1e-30f);
        int nx = 0, ny = 0, nz = 0;
        // bounded search (1e-30 * 1.26^700 > FLT_MAX); a non-finite extent (inf / NaN coordinates) never satisfies
        // the exit test, so such a cloud is left to the tile kernel instead of spinning forever
        bool found = false;
        for (int it = 0; it < 700 && !found; ++it) {
            const float fx = (hi[0] - lo[0]) / cs, fy = (hi[1] - lo[1]) / cs, fz = (hi[2] - lo[2]) / cs;
            if (fx < 4096.f && fy < 4096.f && fz < 4096.f) {
                nx = static_cast<int>(fx) + 1; ny = static_cast<int>(fy) + 1; nz = static_cast<int>(fz) + 1;
                if (static_cast<long long>(nx) * ny * nz <= kEstCells) found = true;
            }
            if (!found) cs *= 1.26f;
        }
        if (!found) { nx = ny = nz = 0; ws.flag[b] = 0; }
        s_org = make_float4(lo[0], lo[1], lo[2], 1.0f / cs);
        s_dim = make_int4(nx, ny, nz, nx * ny * nz);
    }
    __syncthreads();
    if (s_dim.w == 0) return;                        // block-uniform: flag[b] = 0 was written above
    const float4 org = s_org;
    const int4 dim = s_dim;
    for (int i = tid; i < ns; i += kET) {
        const float* q = pts + 3 * static_cast<size_t>(sample(i));
        const int c = (cell_of(__ldg(q + 2), org.z, org.w, dim.z) * dim.y + cell_of(__ldg(q + 1), org.y, org.w, dim.y)) * dim.x +
                      cell_of(__ldg(q), org.x, org.w, dim.x);
        atomicAdd(&cnt[c], 1);
    }
    __syncthreads();
    float cost = 0.f;
    for (int c = tid; c < dim.w; c += kET) {
        const int own = cnt[c];
        if (own == 0) continue;
        const int cx = c % dim.x, cy = (c / dim.x) % dim.y, cz = c / (dim.x * dim.y);
        int nb = 0;
        for (int dz = max(cz - 1, 0); dz <= min(cz + 1, dim.z - 1); ++dz)
            for (int dy = max(cy - 1, 0); dy <= min(cy + 1, dim.y - 1); ++dy)
                for (int dx = max(cx - 1, 0); dx <= min(cx + 1, dim.x - 1); ++dx) nb += cnt[(dz * dim.y + dy) * dim.x + dx];
        cost += static_cast<float>(own) * static_cast<float>(nb);
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) cost += __shfl_xor_sync(FULL, cost, o);
    if (lane == 0) s_cost[warp] = cost;
    __syncthreads();
    if (tid == 0) {
        float tot = 0.f;
        for (int w = 0; w < kET / 32; ++w) tot += s_cost[w];
        const float fn = static_cast<float>(N);
        const float cand = fmaxf(tot / static_cast<float>(ns) * (fn / static_cast<float>(ns)), 1.f);
        const float tile_ns = fminf(kTile * static_cast<float>(nsample) * fn / cand, kTileFull * fn);
        const float f = fminf(1.f, (static_cast<float>(nsample) * fn / (kBallFrac * cand) + 2048.f) / fn);
        const float grid_ns = kGBuild * fn / static_cast<float>(S) + kGSeg * 9.f * f * fn / 2048.f + kGTest * f * cand;
        ws.flag[b] = grid_ns < tile_ns ? 1 : 0;
    }
}

__global__ void __launch_bounds__(kBT)
bq_grid_build_kernel(int N, float r2, const float* __restrict__ xyz, BqGridWs ws)
{
    __shared__ int cnt[kMaxCells];
    __shared__ int red[6][kBNW];
    __shared__ int warp_tot[kBNW];
    __shared__ float4 s_org;          // origin x, y, z, 1 / cell size
    __shared__ int4 s_dim;            // nx, ny, nz, log2 window size
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int b = blockIdx.x;
    if (!ws.flag[b]) return;          // the estimate left this cloud to the tile kernel
    const float* pts = xyz + 3 * static_cast<size_t>(b) * N;

    // ---- bounding box ---------------------------------------------------------------------------------
    float mn[3] = {INFINITY, INFINITY, INFINITY}, mx[3] = {-INFINITY, -INFINITY, -INFINITY};
    for (int j = tid; j < N; j += kBT) {
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            const float v = __ldg(pts + 3 * static_cast<size_t>(j) + a);
            mn[a] = fminf(mn[a], v); mx[a] = fmaxf(mx[a], v);
        }
    }
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const int lo = __reduce_min_sync(FULL, float_ordered(mn[a])), hi = __reduce_max_sync(FULL, float_ordered(mx[a]));
        if (lane == 0) { red[a][warp] = lo; red[3 + a][warp] = hi; }
    }
    for (int c = tid; c < kMaxCells; c += kBT) cnt[c] = 0;
    __syncthreads();
    if (tid == 0) {
        float lo[3], hi[3];
        for (int a = 0; a < 3; ++a) {
            int l = red[a][0], h = red[3 + a][0];
            for (int w = 1; w < kBNW; ++w) { l = min(l, red[a][w]); h = max(h, red[3 + a][w]); }
            lo[a] = ordered_float(l); hi[a] = ordered_float(h);
        }
        float cmax = 0.f, bn_max = 0.f;
        for (int a = 0; a < 3; ++a) {
            const float m = fmaxf(fabsf(lo[a]), fabsf(hi[a]));
            cmax = fmaxf(cmax, m);
            bn_max += m * m;
        }
        bn_max *= 1.000001f;
        // cells no smaller than the radius a query inside the cloud has to cover; coarser if the cells times the
        // windows of the largest window size overflow the table
        const int cell_cap = kMaxCells / (((N - 1) >> kMaxWinLog) + 1);
        float cs = fmaxf(safe_radius(r2, bn_max, bn_max, cmax), 1e-30f);
        int nx = 0, ny = 0, nz = 0;
        bool found = false;                          // bounded like the estimate's search; see there
        for (int it = 0; it < 700 && !found; ++it) {
            const float fx = (hi[0] - lo[0]) / cs, fy = (hi[1] - lo[1]) / cs, fz = (hi[2] - lo[2]) / cs;
            if (fx < 4096.f && fy < 4096.f && fz < 4096.f) {
                nx = static_cast<int>(fx) + 1; ny = static_cast<int>(fy) + 1; nz = static_cast<int>(fz) + 1;
                if (static_cast<long long>(nx) * ny * nz <= cell_cap) found = true;
            }
            if (!found) cs *= 1.26f;
        }
        // the smallest window whose (window, cell) keys fit the table (at the latest kMaxWinLog, by cell_cap)
        int wlog = kMinWinLog;
        while (found && (((N - 1) >> wlog) + 1) * nx * ny * nz > kMaxCells) ++wlog;
        if (!found) { nx = ny = nz = 0; ws.flag[b] = 0; }      // non-finite extent: the tile kernel answers this cloud
        s_org = make_float4(lo[0], lo[1], lo[2], 1.0f / cs);
        s_dim = make_int4(nx, ny, nz, wlog);
        ws.org[b] = s_org;
        ws.dim[b] = s_dim;
        ws.bnd[b] = make_float4(bn_max, cmax, 0.f, 0.f);
    }
    __syncthreads();
    const float4 org = s_org;
    const int4 dim = s_dim;
    const int cells = dim.x * dim.y * dim.z;
    if (cells == 0) return;                          // block-uniform: cloud handed to the tile kernel (flag[b] = 0)
    const int nkeys = (((N - 1) >> dim.w) + 1) * cells;
    auto key_of = [&](int j, float x, float y, float z) {
        return (j >> dim.w) * cells +
               (cell_of(z, org.z, org.w, dim.z) * dim.y + cell_of(y, org.y, org.w, dim.y)) * dim.x + cell_of(x, org.x, org.w, dim.x);
    };

    // ---- histogram --------------------------------------------------------------------------------------
    for (int j = tid; j < N; j += kBT) {
        const float x = __ldg(pts + 3 * static_cast<size_t>(j)), y = __ldg(pts + 3 * static_cast<size_t>(j) + 1),
                    z = __ldg(pts + 3 * static_cast<size_t>(j) + 2);
        atomicAdd(&cnt[key_of(j, x, y, z)], 1);
    }
    __syncthreads();

    // ---- exclusive scan of the counters -> cell_start (global) and scatter cursors (shared) ------------------
    constexpr int kPer = kMaxCells / kBT;      // 8 consecutive keys per thread
    int v[kPer], sum = 0;
#pragma unroll
    for (int k = 0; k < kPer; ++k) { v[k] = cnt[tid * kPer + k]; sum += v[k]; }
    int inc = sum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(FULL, inc, o);
        if (lane >= o) inc += t;
    }
    if (lane == 31) warp_tot[warp] = inc;
    __syncthreads();
    if (warp == 0) {
        int t = warp_tot[lane];
        int i2 = t;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int u = __shfl_up_sync(FULL, i2, o);
            if (lane >= o) i2 += u;
        }
        warp_tot[lane] = i2 - t;
    }
    __syncthreads();
    int run = warp_tot[warp] + inc - sum;
    int* cstart = ws.cell_start + static_cast<size_t>(b) * (kMaxCells + 1);
#pragma unroll
    for (int k = 0; k < kPer; ++k) {
        const int key = tid * kPer + k;
        cnt[key] = run;
        if (key <= nkeys) cstart[key] = run;     // keys past nkeys are empty: cstart[nkeys] = N
        run += v[k];
    }
    if (tid == kBT - 1) cstart[kMaxCells] = run;
    __syncthreads();

    // ---- scatter (order inside a segment is irrelevant: membership goes through the bitmap).  Indices are visited
    //      in ascending order across the CTA, so the writes in flight stay inside one or two windows' output. -------
    float4* rec = ws.rec + static_cast<size_t>(b) * N;
    for (int j = tid; j < N; j += kBT) {
        const float x = __ldg(pts + 3 * static_cast<size_t>(j)), y = __ldg(pts + 3 * static_cast<size_t>(j) + 1),
                    z = __ldg(pts + 3 * static_cast<size_t>(j) + 2);
        const int pos = atomicAdd(&cnt[key_of(j, x, y, z)], 1);
        rec[pos] = make_float4(x, y, z, __int_as_float(j));
    }
}

template <typename IdxT>
__global__ void __launch_bounds__(kQW * 32)
ball_query_grid_kernel(int N, int S, float r2, int nsample, const float* __restrict__ new_xyz, IdxT* __restrict__ group_idx,
                       BqGridWs ws, int qpw, int order)
{
    __shared__ unsigned bm_all[kQW][(1 << kMaxWinLog) / 32];     // per warp: membership bitmap of one index window
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int b = blockIdx.y;
    if (!ws.flag[b]) return;                        // dense cloud: the tile kernel answers it
    unsigned* bm = bm_all[warp];
    const float4 org = ws.org[b];
    const int4 dim = ws.dim[b];
    const float4 bnd = ws.bnd[b];
    const int wlog = dim.w, wrows = 1 << (wlog - 10);            // the window's bitmap: wrows rows of 32 words
    const int cells = dim.x * dim.y * dim.z, nwin = ((N - 1) >> wlog) + 1;
    for (int w = lane; w < 32 * wrows; w += 32) bm[w] = 0u;
    const float4* __restrict__ rec = ws.rec + static_cast<size_t>(b) * N;
    const int* __restrict__ cstart = ws.cell_start + static_cast<size_t>(b) * (kMaxCells + 1);
    __syncwarp();

    for (int qi = 0; qi < qpw; ++qi) {        // qpw queries per warp; the bitmap is cleared while it is read out
        const int q = blockIdx.x * (kQW * qpw) + qi * kQW + warp;
        if (q >= S) break;
        const float* a = new_xyz + 3 * (static_cast<size_t>(b) * S + q);
        const float ax = __ldg(a), ay = __ldg(a + 1), az = __ldg(a + 2);
        const float an = sq_norm_unfused(ax, ay, az, order & 1);
        IdxT* row = group_idx + (static_cast<size_t>(b) * S + q) * nsample;
        const float R = safe_radius(r2, an, bnd.x, fmaxf(bnd.y, fmaxf(fabsf(ax), fmaxf(fabsf(ay), fabsf(az)))));
        const int x0 = cell_of(ax - R, org.x, org.w, dim.x), x1 = cell_of(ax + R, org.x, org.w, dim.x);
        const int y0 = cell_of(ay - R, org.y, org.w, dim.y), y1 = cell_of(ay + R, org.y, org.w, dim.y);
        const int z0 = cell_of(az - R, org.z, org.w, dim.z), z1 = cell_of(az + R, org.z, org.w, dim.z);
        // a run = the cells (x0..x1, y, z) of one window: one contiguous segment of the sorted records
        const int ny_r = y1 - y0 + 1, nruns = ny_r * (z1 - z0 + 1);
        int pos = 0, first = N;                     // N: the sentinel the reference leaves when the ball is empty
        for (int w = 0; w < nwin && pos < nsample; ++w) {
            const int* cs_w = cstart + w * cells;
            for (int rb = 0; rb < nruns; rb += 32) {
                // lane l holds run rb + l; a prefix sum over the segment lengths spreads all tests over the lanes
                int s = 0, len = 0;
                if (rb + lane < nruns) {
                    const int rr = rb + lane;
                    const int c0 = ((z0 + rr / ny_r) * dim.y + y0 + rr % ny_r) * dim.x;
                    s = __ldg(cs_w + c0 + x0);
                    len = __ldg(cs_w + c0 + x1 + 1) - s;
                }
                int incl = len;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) {
                    const int t = __shfl_up_sync(FULL, incl, o);
                    if (lane >= o) incl += t;
                }
                const int total = __shfl_sync(FULL, incl, 31);
                const int off = s - (incl - len);   // sorted position of test t of this run: off + t
                for (int t0 = 0; t0 < total; t0 += 64) {
                    float4 p[2];
#pragma unroll
                    for (int u = 0; u < 2; ++u) {
                        const int t = t0 + 32 * u + lane;
                        int k = 0;                  // run of test t: the number of runs whose inclusive end is <= t
#pragma unroll
                        for (int h = 16; h; h >>= 1)
                            if (__shfl_sync(FULL, incl, k + h - 1) <= t) k += h;
                        const int src = __shfl_sync(FULL, off, k) + t;
                        p[u] = t < total ? __ldg(rec + src) : make_float4(0.f, 0.f, 0.f, 0.f);
                    }
#pragma unroll
                    for (int u = 0; u < 2; ++u) {
                        const float bn = sq_norm_unfused(p[u].x, p[u].y, p[u].z, order & 2);
                        if (t0 + 32 * u + lane < total && !(sq_dist_expanded(ax, ay, az, an, p[u].x, p[u].y, p[u].z, bn) > r2)) {
                            const int j = __float_as_int(p[u].w) & ((1 << wlog) - 1);
                            atomicOr(&bm[j >> 5], 1u << (j & 31));
                        }
                    }
                }
            }
            __syncwarp();
            // ---- the window's first nsample - pos set bits, ascending.  Lane l holds word 32*k + l of row k; rows
            //      are read (and cleared) in order and the read-out stops counting once the query is full. ---------
            const int wbase = w << wlog;
            for (int k = 0; k < wrows; ++k) {
                unsigned word = bm[32 * k + lane];
                bm[32 * k + lane] = 0u;
                if (pos >= nsample) continue;         // warp-uniform: only the clearing is left
                const unsigned nz = __ballot_sync(FULL, word != 0u);
                if (!nz) continue;
                const int c = __popc(word);
                int inc = c;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) {
                    const int t = __shfl_up_sync(FULL, inc, o);
                    if (lane >= o) inc += t;
                }
                if (pos == 0) {
                    const int fl = __ffs(nz) - 1;
                    first = wbase + (32 * k + fl) * 32 + __ffs(__shfl_sync(FULL, word, fl)) - 1;
                }
                int p = pos + inc - c;
                const int base = wbase + (32 * k + lane) * 32;
                while (word && p < nsample) {
                    row[p++] = static_cast<IdxT>(base + __ffs(word) - 1);
                    word &= word - 1;
                }
                pos += __shfl_sync(FULL, inc, 31);
            }
            __syncwarp();
        }
        for (int p = min(pos, nsample) + lane; p < nsample; p += 32) row[p] = static_cast<IdxT>(first);
    }
}

}  // namespace

size_t bq_grid_workspace_bytes(int B, int N, BqGridWs* ws_offsets)
{
    size_t off = 0;
    auto take = [&off](size_t bytes) { const size_t o = off; off = (off + bytes + 255) & ~static_cast<size_t>(255); return o; };
    const size_t o_rec = take(static_cast<size_t>(B) * N * sizeof(float4)),
                 o_cs = take(static_cast<size_t>(B) * (kMaxCells + 1) * sizeof(int)), o_org = take(B * sizeof(float4)),
                 o_dim = take(B * sizeof(int4)), o_bnd = take(B * sizeof(float4)), o_flag = take(B * sizeof(int));
    if (ws_offsets) {
        ws_offsets->rec = reinterpret_cast<float4*>(o_rec);
        ws_offsets->cell_start = reinterpret_cast<int*>(o_cs);
        ws_offsets->org = reinterpret_cast<float4*>(o_org);
        ws_offsets->dim = reinterpret_cast<int4*>(o_dim);
        ws_offsets->bnd = reinterpret_cast<float4*>(o_bnd);
        ws_offsets->flag = reinterpret_cast<int*>(o_flag);
    }
    return off;
}

// Largest cloud the grid takes: with windows of the largest size the table still holds >= 64 cells per window.
int bq_grid_max_points() { return (kMaxCells / 64) << kMaxWinLog; }

int bq_grid_launch(int B, int N, int S, float r2, int nsample, const float* xyz, const float* new_xyz, void* group_idx,
                   bool idx64, int force, int order, const BqGridWs& ws, cudaStream_t st)
{
    bq_grid_estimate_kernel<<<B, kET, 0, st>>>(N, S, r2, nsample, force, xyz, ws);
    int rc = check_launch("bq_grid_estimate_kernel");
    if (rc != TGN_OK) return rc;
    bq_grid_build_kernel<<<B, kBT, 0, st>>>(N, r2, xyz, ws);
    rc = check_launch("bq_grid_build_kernel");
    if (rc != TGN_OK) return rc;
    // queries per warp: 4, more when the batch alone fills the machine (fewer, longer CTAs: clouds the
    // estimate left to the tile kernel cost one early-exit CTA launch per block of queries)
    const long long blocks4 = static_cast<long long>(B) * ((S + kQW * 4 - 1) / (kQW * 4));
    const int qpw = 4 * static_cast<int>(std::max<long long>(1, std::min<long long>(blocks4 / (12LL * sm_count()), 16)));
    dim3 grid((S + kQW * qpw - 1) / (kQW * qpw), B);
    if (idx64) ball_query_grid_kernel<long long><<<grid, kQW * 32, 0, st>>>(N, S, r2, nsample, new_xyz, static_cast<long long*>(group_idx), ws, qpw, order);
    else ball_query_grid_kernel<int><<<grid, kQW * 32, 0, st>>>(N, S, r2, nsample, new_xyz, static_cast<int*>(group_idx), ws, qpw, order);
    return check_launch("ball_query_grid_kernel");
}

}  // namespace tgn
