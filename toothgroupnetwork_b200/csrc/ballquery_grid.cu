// ballquery_grid.cu -- ball query through a uniform grid, for clouds whose balls are sparse (sm_90a).
//
// query_ball_point (external_libs/pointnet2_utils/pointnet2_utils.py:120-144) returns, per query, the
// nsample SMALLEST point indices whose expanded-form distance satisfies !(d > r2), padded with the
// first of them (N everywhere when the ball is empty).  The tile kernel in ballquery.cu scans the cloud
// in index order until a query is full; when a ball holds well under 1 % of the cloud (SA1 of the
// reference networks: r = 0.1 on a 24 000-vertex arch, ~150 members) that scan reads a third of the
// cloud per query.  Here:
//   * bq_grid_build_kernel (one CTA per cloud) bins the points into cubic cells no smaller than the
//     query radius (counting sort with shared-memory atomics; at most kMaxCells cells), writes the
//     cell-sorted points as lane-friendly PAIRS (x0,x1,y0,y1), (z0,z1,|p0|^2,|p1|^2), (j0,j1); a tiny
//     estimate kernel decides per cloud beforehand whether the grid pays (estimated candidates per
//     query against the estimated length of the index-order scan);
//   * ball_query_grid_kernel (one warp per query) visits only the cells that intersect the query's
//     box, evaluates the SAME expanded-form arithmetic as the tile kernel on those candidates, and
//     records members in a per-warp BITMAP over original indices in shared memory; the answer is then
//     the first nsample set bits -- ascending index order for free, independent of the order in which
//     the cells were visited.
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
constexpr int kMaxCells = 8192;      // 32 KB of shared-memory counters
constexpr int kQW = 16;              // query warps per CTA
constexpr unsigned FULL = 0xffffffffu;

__device__ __forceinline__ float sq_norm_unfused(float x, float y, float z, bool alt) {      // see ballquery.cu
    return alt ? __fadd_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(z, z)), __fmul_rn(y, y))
               : __fadd_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)), __fmul_rn(z, z));
}
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
// estimates the candidates a grid query tests, and from it the length of the index-order scan the
// tile kernel needs to collect nsample members.  Cost models in ns per query, to be refitted on
// the target GPU with scripts/ball_sweep.py: tile = 3.7e-3 * nsample * N / cand (at most the full scan, 5.6e-4 * N),
// grid = 1.4 + N * (0.5e-4 + 0.5e-4 * 1024 / S) + 8.6e-4 * cand, with a 15 % bias towards the tile kernel.
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
        const float tile_ns = fminf(3.7e-3f * static_cast<float>(nsample) * fn / cand, 5.6e-4f * fn);
        const float grid_ns = 1.4f + fn * (0.5e-4f + 0.5e-4f * 1024.f / static_cast<float>(S)) + 8.6e-4f * cand;
        ws.flag[b] = 1.15f * grid_ns < tile_ns ? 1 : 0;
    }
}

__global__ void __launch_bounds__(kBT)
bq_grid_build_kernel(int N, float r2, const float* __restrict__ xyz, BqGridWs ws, int order)
{
    __shared__ int cnt[kMaxCells];
    __shared__ int red[6][kBNW];
    __shared__ int warp_tot[kBNW];
    __shared__ float4 s_org;          // origin x, y, z, 1 / cell size
    __shared__ int4 s_dim;            // nx, ny, nz, cells
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
        // cells no smaller than the radius a query inside the cloud has to cover; coarser if the table overflows
        float cs = fmaxf(safe_radius(r2, bn_max, bn_max, cmax), 1e-30f);
        int nx = 0, ny = 0, nz = 0;
        bool found = false;                          // bounded like the estimate's search; see there
        for (int it = 0; it < 700 && !found; ++it) {
            const float fx = (hi[0] - lo[0]) / cs, fy = (hi[1] - lo[1]) / cs, fz = (hi[2] - lo[2]) / cs;
            if (fx < 4096.f && fy < 4096.f && fz < 4096.f) {
                nx = static_cast<int>(fx) + 1; ny = static_cast<int>(fy) + 1; nz = static_cast<int>(fz) + 1;
                if (static_cast<long long>(nx) * ny * nz <= kMaxCells) found = true;
            }
            if (!found) cs *= 1.26f;
        }
        if (!found) { nx = ny = nz = 0; ws.flag[b] = 0; }      // non-finite extent: the tile kernel answers this cloud
        s_org = make_float4(lo[0], lo[1], lo[2], 1.0f / cs);
        s_dim = make_int4(nx, ny, nz, nx * ny * nz);
        ws.org[b] = s_org;
        ws.dim[b] = s_dim;
        ws.bnd[b] = make_float4(bn_max, cmax, 0.f, 0.f);
    }
    __syncthreads();
    const float4 org = s_org;
    const int4 dim = s_dim;
    if (dim.w == 0) return;                          // block-uniform: cloud handed to the tile kernel (flag[b] = 0)

    // ---- histogram --------------------------------------------------------------------------------------
    for (int j = tid; j < N; j += kBT) {
        const float x = __ldg(pts + 3 * static_cast<size_t>(j)), y = __ldg(pts + 3 * static_cast<size_t>(j) + 1),
                    z = __ldg(pts + 3 * static_cast<size_t>(j) + 2);
        const int c = (cell_of(z, org.z, org.w, dim.z) * dim.y + cell_of(y, org.y, org.w, dim.y)) * dim.x + cell_of(x, org.x, org.w, dim.x);
        atomicAdd(&cnt[c], 1);
    }
    __syncthreads();

    // ---- exclusive scan of the counters -> cell_start (global) and scatter cursors (shared) ------------------
    constexpr int kPer = kMaxCells / kBT;      // 8 consecutive cells per thread
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
        cnt[tid * kPer + k] = run;
        cstart[tid * kPer + k] = run;
        run += v[k];
    }
    if (tid == kBT - 1) cstart[kMaxCells] = run;
    __syncthreads();

    // ---- scatter (order inside a cell is irrelevant: membership goes through the bitmap) -------------------
    // Sorted position p lives in pair p / 2, half p % 2: (x0,x1,y0,y1), (z0,z1,|p0|^2,|p1|^2), (j0,j1).
    const size_t npair = static_cast<size_t>(N + 1) / 2;
    float* ga = reinterpret_cast<float*>(ws.ga + static_cast<size_t>(b) * npair);
    float* gb = reinterpret_cast<float*>(ws.gb + static_cast<size_t>(b) * npair);
    int* gj = reinterpret_cast<int*>(ws.gj + static_cast<size_t>(b) * npair);
    if ((N & 1) && tid == 0) {                    // odd N: the unused half can never be a member
        const size_t u = npair - 1;
        ga[4 * u + 1] = 0.f; ga[4 * u + 3] = 0.f; gb[4 * u + 1] = 0.f; gb[4 * u + 3] = INFINITY; gj[2 * u + 1] = 0;
    }
    for (int j = tid; j < N; j += kBT) {
        const float x = __ldg(pts + 3 * static_cast<size_t>(j)), y = __ldg(pts + 3 * static_cast<size_t>(j) + 1),
                    z = __ldg(pts + 3 * static_cast<size_t>(j) + 2);
        const int c = (cell_of(z, org.z, org.w, dim.z) * dim.y + cell_of(y, org.y, org.w, dim.y)) * dim.x + cell_of(x, org.x, org.w, dim.x);
        const int pos = atomicAdd(&cnt[c], 1);
        const size_t u = static_cast<size_t>(pos >> 1);
        const int h = pos & 1;
        ga[4 * u + h] = x; ga[4 * u + 2 + h] = y;
        gb[4 * u + h] = z; gb[4 * u + 2 + h] = sq_norm_unfused(x, y, z, order & 2);
        gj[2 * u + h] = j;
    }
}

template <typename IdxT>
__global__ void __launch_bounds__(kQW * 32)
ball_query_grid_kernel(int N, int S, float r2, int nsample, const float* __restrict__ new_xyz, IdxT* __restrict__ group_idx,
                       BqGridWs ws, int rows, int qpw, int order)
{
    extern __shared__ unsigned bm_all[];            // [kQW][32 * rows] membership bitmaps over original indices
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int b = blockIdx.y;
    if (!ws.flag[b]) return;                        // dense cloud: the tile kernel answers it
    unsigned* bm = bm_all + static_cast<size_t>(warp) * 32 * rows;
    for (int w = lane; w < 32 * rows; w += 32) bm[w] = 0u;
    const float4 org = ws.org[b];
    const int4 dim = ws.dim[b];
    const float4 bnd = ws.bnd[b];
    const size_t npair = static_cast<size_t>(N + 1) / 2;
    const float4* __restrict__ ga = ws.ga + static_cast<size_t>(b) * npair;
    const float4* __restrict__ gb = ws.gb + static_cast<size_t>(b) * npair;
    const int2* __restrict__ gj = ws.gj + static_cast<size_t>(b) * npair;
    const int* __restrict__ cstart = ws.cell_start + static_cast<size_t>(b) * (kMaxCells + 1);
    const uint64_t M2 = pack2(-2.0f, -2.0f);
    __syncwarp();

    for (int qi = 0; qi < qpw; ++qi) {        // qpw queries per warp; the bitmap is cleared while it is read out
        const int q = blockIdx.x * (kQW * qpw) + qi * kQW + warp;
        if (q >= S) break;
        const float* a = new_xyz + 3 * (static_cast<size_t>(b) * S + q);
        const float ax = __ldg(a), ay = __ldg(a + 1), az = __ldg(a + 2);
        const float an = sq_norm_unfused(ax, ay, az, order & 1);
        const uint64_t AX = pack2(ax, ax), AY = pack2(ay, ay), AZ = pack2(az, az), AN = pack2(an, an);
        IdxT* row = group_idx + (static_cast<size_t>(b) * S + q) * nsample;
        const float R = safe_radius(r2, an, bnd.x, fmaxf(bnd.y, fmaxf(fabsf(ax), fmaxf(fabsf(ay), fabsf(az)))));
        const int x0 = cell_of(ax - R, org.x, org.w, dim.x), x1 = cell_of(ax + R, org.x, org.w, dim.x);
        const int y0 = cell_of(ay - R, org.y, org.w, dim.y), y1 = cell_of(ay + R, org.y, org.w, dim.y);
        const int z0 = cell_of(az - R, org.z, org.w, dim.z), z1 = cell_of(az + R, org.z, org.w, dim.z);
        // a run = the cells (x0..x1, y, z): contiguous in the cell-sorted arrays.  A lane tests the pair of
        // ADJACENT sorted points (2u, 2u+1) with packed fp32x2 arithmetic -- the same operation sequence per
        // element as the tile kernel; a pair straddling the run boundary only adds a harmless candidate.
        const int ny_r = y1 - y0 + 1, nruns = ny_r * (z1 - z0 + 1);
        for (int rb = 0; rb < nruns; rb += 32) {
            int u0 = 0, u1 = 0;
            if (rb + lane < nruns) {
                const int rr = rb + lane;
                const int cz = z0 + rr / ny_r, cy = y0 + rr % ny_r;
                const int c0 = (cz * dim.y + cy) * dim.x;
                u0 = __ldg(cstart + c0 + x0) >> 1;
                u1 = (__ldg(cstart + c0 + x1 + 1) + 1) >> 1;
            }
            const int here = min(32, nruns - rb);
            for (int k = 0; k < here; ++k) {
                const int e1 = __shfl_sync(FULL, u1, k);
                for (int u = __shfl_sync(FULL, u0, k) + lane; u < e1; u += 64) {
                    float4 A[2], B[2];
                    A[0] = __ldg(ga + u); B[0] = __ldg(gb + u);
                    const bool two = u + 32 < e1;
                    if (two) { A[1] = __ldg(ga + u + 32); B[1] = __ldg(gb + u + 32); }
#pragma unroll
                    for (int t = 0; t < 2; ++t) {
                        if (t == 1 && !two) break;
                        uint64_t dot = mul2(AX, pack2(A[t].x, A[t].y));
                        dot = fma2(AY, pack2(A[t].z, A[t].w), dot);
                        dot = fma2(AZ, pack2(B[t].x, B[t].y), dot);
                        const uint64_t d = add2(add2(mul2(M2, dot), AN), pack2(B[t].z, B[t].w));
                        float d0, d1;
                        unpack2(d, d0, d1);
                        const bool h0 = !(d0 > r2), h1 = !(d1 > r2);
                        if (h0 || h1) {
                            const int2 J = __ldg(gj + u + 32 * t);
                            if (h0) atomicOr(&bm[J.x >> 5], 1u << (J.x & 31));
                            if (h1) atomicOr(&bm[J.y >> 5], 1u << (J.y & 31));
                        }
                    }
                }
            }
        }
        __syncwarp();
        // ---- the first nsample set bits, ascending.  Lane l holds word 32*k + l of row k; rows are read (and
        //      cleared) in order and the read-out stops counting once the query is full. --------------------------
        int pos = 0, first = N;                     // N: the sentinel the reference leaves when the ball is empty
        for (int k = 0; k < rows; ++k) {
            unsigned word = bm[32 * k + lane];
            bm[32 * k + lane] = 0u;
            if (pos >= nsample) continue;             // warp-uniform: only the clearing is left
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
                first = (32 * k + fl) * 32 + __ffs(__shfl_sync(FULL, word, fl)) - 1;
            }
            int p = pos + inc - c;
            const int base = (32 * k + lane) * 32;
            while (word && p < nsample) {
                row[p++] = static_cast<IdxT>(base + __ffs(word) - 1);
                word &= word - 1;
            }
            pos += __shfl_sync(FULL, inc, 31);
        }
        for (int p = min(pos, nsample) + lane; p < nsample; p += 32) row[p] = static_cast<IdxT>(first);
        __syncwarp();
    }
}

}  // namespace

size_t bq_grid_workspace_bytes(int B, int N, BqGridWs* ws_offsets)
{
    size_t off = 0;
    auto take = [&off](size_t bytes) { const size_t o = off; off = (off + bytes + 255) & ~static_cast<size_t>(255); return o; };
    const size_t pts = static_cast<size_t>(B) * N;
    (void)pts;
    const size_t pairs = static_cast<size_t>(B) * ((static_cast<size_t>(N) + 1) / 2);
    const size_t o_ga = take(pairs * sizeof(float4)), o_gb = take(pairs * sizeof(float4)), o_gj = take(pairs * sizeof(int2)),
                 o_cs = take(static_cast<size_t>(B) * (kMaxCells + 1) * sizeof(int)), o_org = take(B * sizeof(float4)),
                 o_dim = take(B * sizeof(int4)), o_bnd = take(B * sizeof(float4)), o_flag = take(B * sizeof(int));
    if (ws_offsets) {
        ws_offsets->ga = reinterpret_cast<float4*>(o_ga);
        ws_offsets->gb = reinterpret_cast<float4*>(o_gb);
        ws_offsets->gj = reinterpret_cast<int2*>(o_gj);
        ws_offsets->cell_start = reinterpret_cast<int*>(o_cs);
        ws_offsets->org = reinterpret_cast<float4*>(o_org);
        ws_offsets->dim = reinterpret_cast<int4*>(o_dim);
        ws_offsets->bnd = reinterpret_cast<float4*>(o_bnd);
        ws_offsets->flag = reinterpret_cast<int*>(o_flag);
    }
    return off;
}

// Largest cloud whose bitmaps (one per query warp) fit the CTA's shared memory.
int bq_grid_max_points() { return 32 * 32 * ((200 * 1024) / (kQW * 32 * 4)); }

int bq_grid_launch(int B, int N, int S, float r2, int nsample, const float* xyz, const float* new_xyz, void* group_idx,
                   bool idx64, int force, int order, const BqGridWs& ws, cudaStream_t st)
{
    bq_grid_estimate_kernel<<<B, kET, 0, st>>>(N, S, r2, nsample, force, xyz, ws);
    int rc = check_launch("bq_grid_estimate_kernel");
    if (rc != TGN_OK) return rc;
    bq_grid_build_kernel<<<B, kBT, 0, st>>>(N, r2, xyz, ws, order);
    rc = check_launch("bq_grid_build_kernel");
    if (rc != TGN_OK) return rc;
    const int rows = ((N + 31) / 32 + 31) / 32;     // bitmap rows of 32 words
    const size_t smem = static_cast<size_t>(kQW) * 32 * rows * sizeof(unsigned);
    rc = idx64 ? ensure_dynamic_smem(reinterpret_cast<const void*>(ball_query_grid_kernel<long long>), smem)
               : ensure_dynamic_smem(reinterpret_cast<const void*>(ball_query_grid_kernel<int>), smem);
    if (rc != TGN_OK) return rc;
    // queries per warp: 4, more when the batch alone fills the machine (fewer, longer CTAs: clouds the
    // estimate left to the tile kernel cost one early-exit CTA launch per block of queries)
    const long long blocks4 = static_cast<long long>(B) * ((S + kQW * 4 - 1) / (kQW * 4));
    const int qpw = 4 * static_cast<int>(std::max<long long>(1, std::min<long long>(blocks4 / (12LL * sm_count()), 16)));
    dim3 grid((S + kQW * qpw - 1) / (kQW * qpw), B);
    if (idx64) ball_query_grid_kernel<long long><<<grid, kQW * 32, smem, st>>>(N, S, r2, nsample, new_xyz, static_cast<long long*>(group_idx), ws, rows, qpw, order);
    else ball_query_grid_kernel<int><<<grid, kQW * 32, smem, st>>>(N, S, r2, nsample, new_xyz, static_cast<int*>(group_idx), ws, rows, qpw, order);
    return check_launch("ball_query_grid_kernel");
}

}  // namespace tgn
