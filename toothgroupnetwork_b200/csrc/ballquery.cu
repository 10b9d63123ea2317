// ballquery.cu -- ball query and 3-NN on the PointNet++ side, sm_90a.
//
// The reference has no kernel here: query_ball_point materialises an (S,N) fp32 distance
// matrix through a K=3 matmul plus an (S,N) int64 index tensor and SORTS every row
// (external_libs/pointnet2_utils/pointnet2_utils.py:120-144); PointNetFeaturePropagation
// sorts an (N,S) matrix to take three entries (:333-335).  Here both are streaming scans with
// coordinates staged through shared memory, and the ball query stops as soon as a query has
// its nsample hits.
//
// Bit-exact membership: the distance is evaluated in the reference's EXPANDED form and
// rounding order (probed against torch, see oracle/pointops_oracle.c):
//      dot = ax*bx; dot = fma(ay,by,dot); dot = fma(az,bz,dot);
//      d = -2*dot; d += |a|^2; d += |b|^2      with |p|^2 = (x*x + y*y) + z*z, unfused
// and a point is a member iff !(d > r2), r2 = float32(radius**2).
#include <algorithm>
#include <climits>

#include "ballquery.cuh"
#include "common.cuh"
#include "tgn_b200.h"

namespace tgn {
namespace {

constexpr int kTile = 1024;   // points staged per shared-memory tile (16 KB as SoA x,y,z,|p|^2)

// |p|^2 as torch.sum(p ** 2, -1) rounds it ON THE GPU (square_distance :39-40), measured with torch 2.11
// (scripts/diag_sumsq.py): a strided reduction (the permuted views the reference's modules
// pass) accumulates in index order, (x*x + y*y) + z*z -- the same as torch on the CPU; a CONTIGUOUS (..., 3) tensor
// (e.g. new_xyz fresh out of index_points) goes through the vectorised reduce path and comes out as
// (x*x + z*z) + y*y.  `alt` selects the second form; the Python layer derives it from the layout the reference's
// own call would see, per operand.
__device__ __forceinline__ float sq_norm_unfused(float x, float y, float z, bool alt) {
    return alt ? __fadd_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(z, z)), __fmul_rn(y, y))
               : __fadd_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)), __fmul_rn(z, z));
}
__device__ __forceinline__ float sq_dist_expanded(float ax, float ay, float az, float an, float bx, float by, float bz,
                                                  float bn) {
    float dot = __fmul_rn(ax, bx);
    dot = __fmaf_rn(ay, by, dot);
    dot = __fmaf_rn(az, bz, dot);
    float d = __fmul_rn(-2.0f, dot);
    d = __fadd_rn(d, an);
    return __fadd_rn(d, bn);
}

// The same when the reference's matmul has a single column (one dst point per batch, tsegnet.get_ddf): cuBLAS on H100 then
// takes a matrix-vector path that rounds the dot product as fma(ay, by, ax*bx) + az*bz (measured with torch 2.11 / cuBLAS
// for CUDA 12.8; two or more columns round as the fused chain above).
__device__ __forceinline__ float sq_dist_expanded_one_column(float ax, float ay, float az, float an, float bx, float by, float bz,
                                                             float bn) {
    float dot = __fmaf_rn(ay, by, __fmul_rn(ax, bx));
    dot = __fadd_rn(dot, __fmul_rn(az, bz));
    float d = __fmul_rn(-2.0f, dot);
    d = __fadd_rn(d, an);
    return __fadd_rn(d, bn);
}

// Stage points [base, base+cnt) of one cloud into shared SoA arrays (coalesced 12-byte reads).
template <int THREADS>
__device__ __forceinline__ void stage_tile(const float* __restrict__ pts, int base, int cnt, float* sx, float* sy,
                                           float* sz, float* sn, bool alt)
{
    for (int i = threadIdx.x; i < cnt; i += THREADS) {
        const float x = __ldg(pts + 3 * static_cast<size_t>(base + i)), y = __ldg(pts + 3 * static_cast<size_t>(base + i) + 1),
                    z = __ldg(pts + 3 * static_cast<size_t>(base + i) + 2);
        sx[i] = x; sy[i] = y; sz[i] = z; sn[i] = sq_norm_unfused(x, y, z, alt);
    }
    // pad to a multiple of 128 with points at infinite distance (never a member, never a neighbour)
    for (int i = cnt + threadIdx.x; i < ((cnt + 127) & ~127); i += THREADS) {
        sx[i] = 0.f; sy[i] = 0.f; sz[i] = 0.f; sn[i] = INFINITY;
    }
}
__device__ __forceinline__ uint64_t lds_f32x2(uint32_t addr) {      // two adjacent floats as a packed pair
    uint64_t v;
    asm volatile("ld.shared.b64 %0, [%1];" : "=l"(v) : "r"(addr));
    return v;
}

// One warp per query, WARPS queries of one cloud per CTA.  Lanes test 32 consecutive points per
// step; __ballot + popc give each hit its rank in ascending index order.
template <int WARPS, typename IdxT>
__global__ void __launch_bounds__(WARPS * 32)
ball_query_kernel(int N, int S, float r2, int nsample, const float* __restrict__ xyz, const float* __restrict__ new_xyz,
                  IdxT* __restrict__ group_idx, const int* __restrict__ answered, int order)
{
    constexpr unsigned FULL = 0xffffffffu;
    if (answered && answered[blockIdx.y]) return;     // this cloud went through the grid kernel
    __shared__ __align__(16) float sx[kTile], sy[kTile], sz[kTile], sn[kTile];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int b = blockIdx.y;
    const int q = blockIdx.x * WARPS + warp;
    const bool live = q < S;
    const float* pts = xyz + 3 * static_cast<size_t>(b) * N;
    float ax = 0.f, ay = 0.f, az = 0.f, an = 0.f;
    IdxT* row = nullptr;
    if (live) {
        const float* a = new_xyz + 3 * (static_cast<size_t>(b) * S + q);
        ax = __ldg(a); ay = __ldg(a + 1); az = __ldg(a + 2);
        an = sq_norm_unfused(ax, ay, az, order & 1);
        row = group_idx + (static_cast<size_t>(b) * S + q) * nsample;
    }
    int cnt = live ? 0 : nsample;     // dead warps count as finished
    int first = N;                    // sentinel the reference leaves when the ball is empty
    const uint32_t a_x = smem_u32(sx), a_y = smem_u32(sy), a_z = smem_u32(sz), a_n = smem_u32(sn);
    for (int base = 0; base < N; base += kTile) {
        const int tile = min(kTile, N - base);
        __syncthreads();              // previous tile fully consumed
        stage_tile<WARPS * 32>(pts, base, tile, sx, sy, sz, sn, order & 2);
        __syncthreads();
        if (cnt < nsample) {
            // four 32-point steps per trip: 16 shared loads issued together, one early-exit test per 128
            // points (the tile arrays are padded to a multiple of 128 with points that can never hit)
            // Each lane tests the ADJACENT points 2*lane and 2*lane+1 of a 64-point step with packed
            // fp32 pair arithmetic (same IEEE-rn results per element as scalar code); two steps per trip.
            const uint64_t AX = pack2(ax, ax), AY = pack2(ay, ay), AZ = pack2(az, az), AN = pack2(an, an);
            const uint64_t M2 = pack2(-2.0f, -2.0f);
            const unsigned lt = (1u << lane) - 1u;
            for (int o = 0; o < tile && cnt < nsample; o += 128) {
                uint64_t d[2];
#pragma unroll
                for (int u = 0; u < 2; ++u) {
                    const uint32_t off = static_cast<uint32_t>(o + 64 * u + 2 * lane) * 4u;
                    uint64_t dot = mul2(AX, lds_f32x2(a_x + off));
                    dot = fma2(AY, lds_f32x2(a_y + off), dot);
                    dot = fma2(AZ, lds_f32x2(a_z + off), dot);
                    d[u] = add2(add2(mul2(M2, dot), AN), lds_f32x2(a_n + off));
                }
#pragma unroll
                for (int u = 0; u < 2; ++u) {
                    float d0, d1;
                    unpack2(d[u], d0, d1);
                    const bool h0 = !(d0 > r2), h1 = !(d1 > r2);
                    const unsigned m0 = __ballot_sync(FULL, h0), m1 = __ballot_sync(FULL, h1);
                    if (m0 | m1) {
                        const int p0 = base + o + 64 * u;               // index of point (lane 0, half 0)
                        if (cnt == 0) {
                            const int f0 = m0 ? 2 * (__ffs(m0) - 1) : INT_MAX, f1 = m1 ? 2 * (__ffs(m1) - 1) + 1 : INT_MAX;
                            first = p0 + min(f0, f1);
                        }
                        const int before = cnt + __popc(m0 & lt) + __popc(m1 & lt);   // hits at lower indices
                        if (h0 && before < nsample) row[before] = static_cast<IdxT>(p0 + 2 * lane);
                        const int pos1 = before + (h0 ? 1 : 0);
                        if (h1 && pos1 < nsample) row[pos1] = static_cast<IdxT>(p0 + 2 * lane + 1);
                        cnt += __popc(m0) + __popc(m1);
                    }
                }
            }
        }
        if (__syncthreads_and(cnt >= nsample)) break;   // every query of this CTA is full
    }
    if (live) {
        cnt = min(cnt, nsample);
        for (int p = cnt + lane; p < nsample; p += 32) row[p] = static_cast<IdxT>(first);
    }
}

// ---- streaming variant (default) ------------------------------------------------------------------
// pack: (x, y, z) -> (x, y, z, |p|^2) so that the scan needs ONE 16-byte load per point.
__global__ void __launch_bounds__(256)
pack_xyzn_kernel(size_t total, const float* __restrict__ xyz, float4* __restrict__ out, int order)
{
    for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
         i += static_cast<size_t>(gridDim.x) * blockDim.x) {
        const float x = __ldg(xyz + 3 * i), y = __ldg(xyz + 3 * i + 1), z = __ldg(xyz + 3 * i + 2);
        out[i] = make_float4(x, y, z, sq_norm_unfused(x, y, z, order & 2));
    }
}

// One warp per query, warps fully independent (no shared memory, no block barrier): every warp
// scans its cloud from index 0 in steps of 128 points (4 x 16-byte loads in flight per lane) and
// leaves as soon as it has its nsample hits.  All queries of a cloud start at the same addresses,
// so the head of the cloud stays L1-resident.
template <typename IdxT>
__global__ void __launch_bounds__(256)
ball_query_stream_kernel(int N, int S, float r2, int nsample, const float4* __restrict__ pts, const float* __restrict__ new_xyz,
                         IdxT* __restrict__ group_idx, int order)
{
    constexpr unsigned FULL = 0xffffffffu;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int b = blockIdx.y;
    const int q = blockIdx.x * 8 + warp;
    if (q >= S) return;
    const float* a = new_xyz + 3 * (static_cast<size_t>(b) * S + q);
    const float ax = __ldg(a), ay = __ldg(a + 1), az = __ldg(a + 2);
    const float an = sq_norm_unfused(ax, ay, az, order & 1);
    IdxT* row = group_idx + (static_cast<size_t>(b) * S + q) * nsample;
    const float4* P = pts + static_cast<size_t>(b) * N;
    int cnt = 0, first = N;
    for (int o = 0; o < N && cnt < nsample; o += 128) {
        float4 v[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const int i = o + 32 * u + lane;
            v[u] = i < N ? __ldg(P + i) : make_float4(0.f, 0.f, 0.f, INFINITY);
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const bool hit = !(sq_dist_expanded(ax, ay, az, an, v[u].x, v[u].y, v[u].z, v[u].w) > r2);
            const unsigned mask = __ballot_sync(FULL, hit);
            if (mask) {
                if (cnt == 0) first = o + 32 * u + __ffs(mask) - 1;
                const int pos = cnt + __popc(mask & ((1u << lane) - 1));
                if (hit && pos < nsample) row[pos] = static_cast<IdxT>(o + 32 * u + lane);
                cnt += __popc(mask);
            }
        }
    }
    cnt = min(cnt, nsample);
    for (int p = cnt + lane; p < nsample; p += 32) row[p] = static_cast<IdxT>(first);
}

// 3 nearest coarse points per fine point; one thread per fine point, coarse cloud in shared tiles.
// Strict '<' keeps the lower index among equal distances.
template <int THREADS>
__global__ void __launch_bounds__(THREADS)
three_nn_kernel(int N, int S, const float* __restrict__ xyz1, const float* __restrict__ xyz2, float* __restrict__ dist,
                int* __restrict__ idx, int order)
{
    __shared__ float sx[kTile], sy[kTile], sz[kTile], sn[kTile];
    const int b = blockIdx.y;
    const int i = blockIdx.x * THREADS + threadIdx.x;
    const bool live = i < N;
    float ax = 0.f, ay = 0.f, az = 0.f, an = 0.f;
    if (live) {
        const float* a = xyz1 + 3 * (static_cast<size_t>(b) * N + i);
        ax = __ldg(a); ay = __ldg(a + 1); az = __ldg(a + 2);
        an = sq_norm_unfused(ax, ay, az, order & 1);
    }
    float d0 = INFINITY, d1 = INFINITY, d2 = INFINITY;
    int i0 = 0, i1 = 0, i2 = 0;
    const float* pts = xyz2 + 3 * static_cast<size_t>(b) * S;
    for (int base = 0; base < S; base += kTile) {
        const int tile = min(kTile, S - base);
        __syncthreads();
        stage_tile<THREADS>(pts, base, tile, sx, sy, sz, sn, order & 2);
        __syncthreads();
        if (live) {
#pragma unroll 4
            for (int j = 0; j < tile; ++j) {
                const float d = sq_dist_expanded(ax, ay, az, an, sx[j], sy[j], sz[j], sn[j]);
                if (d < d2) {
                    const int g = base + j;
                    if (d < d0) { d2 = d1; i2 = i1; d1 = d0; i1 = i0; d0 = d; i0 = g; }
                    else if (d < d1) { d2 = d1; i2 = i1; d1 = d; i1 = g; }
                    else { d2 = d; i2 = g; }
                }
            }
        }
    }
    if (live) {
        const size_t o = 3 * (static_cast<size_t>(b) * N + i);
        dist[o] = d0; dist[o + 1] = d1; dist[o + 2] = d2;
        idx[o] = i0; idx[o + 1] = i1; idx[o + 2] = i2;
    }
}

// out[b,n,:] = sum_k w_k * points2[b, idx[b,n,k], :],  w = (1/(d+1e-8)) / sum (pointnet2_utils.py:337-340)
__global__ void __launch_bounds__(256)
three_interpolate_kernel(int N, int S, int C, const float* __restrict__ points2, const float* __restrict__ dist,
                         const int* __restrict__ idx, float* __restrict__ out, bool norm_alt)
{
    const int b = blockIdx.y;
    const size_t total = static_cast<size_t>(N) * C;
    const float* p2 = points2 + static_cast<size_t>(b) * S * C;
    for (size_t e = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; e < total;
         e += static_cast<size_t>(gridDim.x) * blockDim.x) {
        const int n = static_cast<int>(e / C), c = static_cast<int>(e % C);
        const size_t o = 3 * (static_cast<size_t>(b) * N + n);
        const float r0 = __fdiv_rn(1.0f, __fadd_rn(dist[o], 1e-8f)), r1 = __fdiv_rn(1.0f, __fadd_rn(dist[o + 1], 1e-8f)),
                    r2 = __fdiv_rn(1.0f, __fadd_rn(dist[o + 2], 1e-8f));
        // torch.sum(dist_recip, dim=2) (:338): dist_recip is a fresh contiguous (B,N,3) tensor, so on CUDA the vectorised
        // reduce applies, (r0 + r2) + r1; on the CPU (and in the committed fixtures) it is (r0 + r1) + r2
        const float norm = norm_alt ? __fadd_rn(__fadd_rn(r0, r2), r1) : __fadd_rn(__fadd_rn(r0, r1), r2);
        const float w0 = __fdiv_rn(r0, norm), w1 = __fdiv_rn(r1, norm), w2 = __fdiv_rn(r2, norm);
        float acc = __fmul_rn(p2[static_cast<size_t>(idx[o]) * C + c], w0);
        acc = __fadd_rn(acc, __fmul_rn(p2[static_cast<size_t>(idx[o + 1]) * C + c], w1));
        acc = __fadd_rn(acc, __fmul_rn(p2[static_cast<size_t>(idx[o + 2]) * C + c], w2));
        out[(static_cast<size_t>(b) * N + n) * C + c] = acc;
    }
}

// out[b, i, j] = expanded squared distance between src[b, i] and dst[b, j] (pointnet2_utils.square_distance :20-41), the
// same arithmetic as the searches above but materialised: the losses (tgn_loss.py / tsg_loss.py) and tsegnet.get_ddf want the
// matrix itself.  One thread per output element, src row staged per block row.
__global__ void __launch_bounds__(256)
square_distance_kernel(int N, int M, const float* __restrict__ src, const float* __restrict__ dst, float* __restrict__ out, int order)
{
    const int b = blockIdx.z, i = blockIdx.y;
    const float* a = src + 3 * (static_cast<size_t>(b) * N + i);
    const float ax = __ldg(a), ay = __ldg(a + 1), az = __ldg(a + 2);
    const float an = sq_norm_unfused(ax, ay, az, order & 1);
    float* row = out + (static_cast<size_t>(b) * N + i) * M;
    for (int j = blockIdx.x * 256 + threadIdx.x; j < M; j += gridDim.x * 256) {
        const float* p = dst + 3 * (static_cast<size_t>(b) * M + j);
        const float bx = __ldg(p), by = __ldg(p + 1), bz = __ldg(p + 2);
        const float bn = sq_norm_unfused(bx, by, bz, order & 2);
        row[j] = M == 1 ? sq_dist_expanded_one_column(ax, ay, az, an, bx, by, bz, bn) : sq_dist_expanded(ax, ay, az, an, bx, by, bz, bn);
    }
}

}  // namespace
}  // namespace tgn

extern "C" {

int tgn_ball_query(int B, int N, int S, float r2, int nsample, const float* xyz, const float* new_xyz, void* group_idx,
                   int idx64, void* stream)
{
    using namespace tgn;
    if (B <= 0 || S <= 0 || nsample <= 0) return TGN_OK;
    if (N <= 0) { set_error("ball_query: N must be positive"); return TGN_ERR_INVALID; }
    if (B > 65535) { set_error("ball_query: B=%d exceeds gridDim.y", B); return TGN_ERR_INVALID; }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int order = (idx64 >> 4) & 3;      // bit 4: |new_xyz|^2 in the contiguous-reduce order, bit 5: |xyz|^2 likewise
    // Streaming variant (pack once into stream-ordered scratch, then fully independent warps).  Measured
    // it ties with the shared-memory tile kernel at 24k points (both issue-bound) and loses
    // to its packed-fp32x2 form, so it is only taken on request (idx64 bit 1 set: experiments).
    if (idx64 & 2) {
        keep_async_pool();
        const size_t total = static_cast<size_t>(B) * N;
        float4* packed = nullptr;
        const cudaError_t e = cudaMallocAsync(reinterpret_cast<void**>(&packed), total * sizeof(float4), st);
        if (e == cudaSuccess) {
            const int pg = static_cast<int>(std::min<size_t>((total + 255) / 256, 16 * static_cast<size_t>(sm_count())));
            pack_xyzn_kernel<<<pg, 256, 0, st>>>(total, xyz, packed, order);
            int rc = check_launch("pack_xyzn_kernel");
            if (rc == TGN_OK) {
                dim3 grid((S + 7) / 8, B);
                if (idx64 & 1) ball_query_stream_kernel<long long><<<grid, 256, 0, st>>>(N, S, r2, nsample, packed, new_xyz, static_cast<long long*>(group_idx), order);
                else ball_query_stream_kernel<int><<<grid, 256, 0, st>>>(N, S, r2, nsample, packed, new_xyz, static_cast<int*>(group_idx), order);
                rc = check_launch("ball_query_stream_kernel");
            }
            (void)cudaFreeAsync(packed, st);
            return rc;
        }
        (void)cudaGetLastError();     // no scratch: fall through to the shared-memory tile kernel
    }
    // Sparse balls on large clouds: uniform-grid kernel (ballquery_grid.cu); it decides per cloud and
    // leaves the dense ones to the tile kernel below.  idx64 bit 2 keeps everything on the tile kernel,
    // bit 3 sends everything through the grid (experiments / tests).
    const int* answered = nullptr;
    unsigned char* grid_ws = nullptr;
    if (!(idx64 & 4) && N <= bq_grid_max_points() && (N >= 8192 || (idx64 & 8))) {
        keep_async_pool();
        BqGridWs ws{};
        const size_t bytes = bq_grid_workspace_bytes(B, N, &ws);
        if (cudaMallocAsync(reinterpret_cast<void**>(&grid_ws), bytes, st) == cudaSuccess) {
            ws.ga = reinterpret_cast<float4*>(grid_ws + reinterpret_cast<size_t>(ws.ga));
            ws.gb = reinterpret_cast<float4*>(grid_ws + reinterpret_cast<size_t>(ws.gb));
            ws.gj = reinterpret_cast<int2*>(grid_ws + reinterpret_cast<size_t>(ws.gj));
            ws.cell_start = reinterpret_cast<int*>(grid_ws + reinterpret_cast<size_t>(ws.cell_start));
            ws.org = reinterpret_cast<float4*>(grid_ws + reinterpret_cast<size_t>(ws.org));
            ws.dim = reinterpret_cast<int4*>(grid_ws + reinterpret_cast<size_t>(ws.dim));
            ws.bnd = reinterpret_cast<float4*>(grid_ws + reinterpret_cast<size_t>(ws.bnd));
            ws.flag = reinterpret_cast<int*>(grid_ws + reinterpret_cast<size_t>(ws.flag));
            const int rc = bq_grid_launch(B, N, S, r2, nsample, xyz, new_xyz, group_idx, (idx64 & 1) != 0, (idx64 & 8) ? 1 : 0, order, ws, st);
            if (rc != TGN_OK) { (void)cudaFreeAsync(grid_ws, st); return rc; }
            answered = ws.flag;
        } else {
            (void)cudaGetLastError();     // no scratch: the tile kernel answers everything
            grid_ws = nullptr;
        }
    }
    // 16 queries per CTA when that still gives >= 2 waves, else 8 (small batches)
    const bool wide = static_cast<long long>(B) * ((S + 15) / 16) >= 2LL * sm_count();
    if (wide) {
        dim3 grid((S + 15) / 16, B);
        if (idx64 & 1) ball_query_kernel<16, long long><<<grid, 512, 0, st>>>(N, S, r2, nsample, xyz, new_xyz, static_cast<long long*>(group_idx), answered, order);
        else ball_query_kernel<16, int><<<grid, 512, 0, st>>>(N, S, r2, nsample, xyz, new_xyz, static_cast<int*>(group_idx), answered, order);
    } else {
        dim3 grid((S + 7) / 8, B);
        if (idx64 & 1) ball_query_kernel<8, long long><<<grid, 256, 0, st>>>(N, S, r2, nsample, xyz, new_xyz, static_cast<long long*>(group_idx), answered, order);
        else ball_query_kernel<8, int><<<grid, 256, 0, st>>>(N, S, r2, nsample, xyz, new_xyz, static_cast<int*>(group_idx), answered, order);
    }
    const int rc = check_launch("ball_query_kernel");
    if (grid_ws) (void)cudaFreeAsync(grid_ws, st);
    return rc;
}

int tgn_three_nn(int B, int N, int S, const float* xyz1, const float* xyz2, float* dist, int* idx, void* stream)
{
    return tgn_three_nn_ex(B, N, S, xyz1, xyz2, dist, idx, 0, stream);
}

int tgn_three_nn_ex(int B, int N, int S, const float* xyz1, const float* xyz2, float* dist, int* idx, int order, void* stream)
{
    using namespace tgn;
    if (B <= 0 || N <= 0) return TGN_OK;
    if (S < 3) { set_error("three_nn: needs at least 3 coarse points (S=%d)", S); return TGN_ERR_INVALID; }
    if (B > 65535) { set_error("three_nn: B=%d exceeds gridDim.y", B); return TGN_ERR_INVALID; }
    dim3 grid((N + 127) / 128, B);
    three_nn_kernel<128><<<grid, 128, 0, static_cast<cudaStream_t>(stream)>>>(N, S, xyz1, xyz2, dist, idx, order);
    return check_launch("three_nn_kernel");
}

int tgn_square_distance(int B, int N, int M, const float* src, const float* dst, float* out, int order, void* stream)
{
    using namespace tgn;
    if (B <= 0 || N <= 0 || M <= 0) return TGN_OK;
    if (B > 65535 || N > 65535) { set_error("square_distance: B=%d / N=%d exceed the grid limits", B, N); return TGN_ERR_INVALID; }
    dim3 grid(std::min((M + 255) / 256, 64), N, B);
    square_distance_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(N, M, src, dst, out, order);
    return check_launch("square_distance_kernel");
}

int tgn_three_interpolate(int B, int N, int S, int C, const float* points2, const float* dist, const int* idx, float* out,
                          void* stream)
{
    return tgn_three_interpolate_ex(B, N, S, C, points2, dist, idx, out, 0, stream);
}

int tgn_three_interpolate_ex(int B, int N, int S, int C, const float* points2, const float* dist, const int* idx, float* out,
                             int norm_alt, void* stream)
{
    using namespace tgn;
    if (B <= 0 || N <= 0 || C <= 0) return TGN_OK;
    if (B > 65535) { set_error("three_interpolate: B=%d exceeds gridDim.y", B); return TGN_ERR_INVALID; }
    const size_t total = static_cast<size_t>(N) * C;
    const int blocks = static_cast<int>(std::min<size_t>((total + 255) / 256, 8 * static_cast<size_t>(sm_count())));
    three_interpolate_kernel<<<dim3(blocks, B), 256, 0, static_cast<cudaStream_t>(stream)>>>(N, S, C, points2, dist, idx, out, norm_alt != 0);
    return check_launch("three_interpolate_kernel");
}

}  // extern "C"
