// fps_bucket.cu -- bucket-pruned farthest point sampling for sm_90a (bit-exact).
//
// The brute-force FPS update touches every point every iteration although, after a few
// samples, a new sample only lowers the running minimum of the points NEAR it.  This kernel
// keeps the reference's result bit for bit and skips the rest:
//
//  * prologue kernel (one CTA per cloud): the cloud is sorted by a Morton code (stable LSD radix sort;
//    clouds up to 26.6k points entirely in shared memory on 17-bit codes, larger ones through global
//    memory on 21-bit codes) so that every 64 consecutive points -- a BUCKET, two adjacent points per
//    lane of a warp -- are spatial neighbours; each bucket gets an axis-aligned bounding box (inflated
//    by an absolute slack).  Sorted points are stored lane-major as 16-byte pairs, (x0,x1,y0,y1) and
//    (z0,z1,t0,t1), so that the distance update runs on the packed fp32x2 pipe; their tie keys live
//    in an array of their own that the update loop does not read.
//  * main kernel (one CTA of 4, 8 or 16 warps per cloud, 8, 4 or 2 CTAs per SM); warp w OWNS the
//    contiguous bucket range [w*R, (w+1)*R) and caches its best candidate and the union box of the
//    range.  Per iteration, with o the new sample:
//      (a) owner warps test their range box, then their buckets: for every point p of a box,
//          |p - o|^2 >= dist^2(o, box), so if dist^2(o, box) > max_t(box) * (1 + 2e-5) the update
//          min(t, |p-o|^2) cannot change any t inside (the slack terms dominate every fp32 rounding
//          error involved; DESIGN.md "pruning is conservative") and the box is skipped;
//      (b) surviving buckets are spread over all warps, one warp per bucket, two buckets in flight: the
//          64 points are re-evaluated with the reference's exact arithmetic (FMUL dy*dy,
//          FFMA dx*dx+., FFMA dz*dz+., FMNMX; the packed forms round each half identically),
//          changed minima are written back and the bucket's cached candidate (max t, sorted position,
//          coordinates) is refreshed;
//      (c) owner warps whose range was touched refresh their range candidate; the block arg-max is
//          one CREDUX pair over the range candidates.
//    Ties are resolved by the reference's order (bitrev(j mod BS), j div BS) on ORIGINAL indices, so the
//    result does not depend on the internal order.  Candidates carry their sorted position; a reduction
//    reads the keys of the tied entries only when more than one entry holds the maximum.  The loop
//    records sorted positions in idx and maps them to original indices in one pass at the end.
//  * the bucket table lives in shared memory (52 B per bucket), the points in L2/HBM (16 B/point read per
//    visit, 4 B/point of keys apart); an iteration is three block barriers and one
//    memory round trip, hidden by the other CTAs of the SM.
#include <algorithm>
#include <climits>

#include "common.cuh"
#include "fps.cuh"
#include "tgn_b200.h"

namespace tgn {
namespace {

constexpr int kT = 512;            // sort kernel (latency-bound: more warps per cloud = shorter serial loops)
constexpr int kNW = kT / 32;
constexpr int kBP = 64;            // points per bucket: two per lane
constexpr int kBatch = 2;          // buckets a warp keeps in flight (memory-level parallelism)
constexpr int kGatherUnroll = 2;   // buckets a sort-kernel warp gathers together
constexpr int kRadixUnroll = 4;    // radix steps whose loads are issued together
constexpr int kSmemSortMaxN = 26624; // clouds up to this size are radix-sorted in shared memory (2 x 4 B per point)
constexpr int kMaxBuckets = 3600;   // 52 B of shared memory per bucket
constexpr unsigned FULL = 0xffffffffu;

struct BucketWs {
    float4* pa;       // [b][stride/2]  bucket-major, lane-major pairs (x0, x1, y0, y1); lane l holds sorted points 2l, 2l+1
    float4* pb;       // [b][stride/2]  (z0, z1, t0, t1): coordinates and running minima; pads carry t = -1
    int2* keys;       // [b][stride/2]  tie keys (key0, key1) of the same pairs; pads INT_MAX
    uint2* key_a;     // [b][stride]    radix ping (clouds too large for the shared-memory sort)
    uint2* key_b;     // [b][stride]    radix pong
    float4* box_lo;   // [b][nbmax]     inflated box minimum, w = initial max t of the bucket
    float4* box_hi;   // [b][nbmax]     inflated box maximum, w = bits of that max t
    float4* bxyz;     // [b][nbmax]     initial cached candidate (x, y, z, bits(sorted position in the cloud))
    int stride;       // points per cloud slot (multiple of 64)
    int nbmax;        // buckets per cloud slot
};


__device__ __forceinline__ int bitrev_low(int v, int bits) {
    return bits ? static_cast<int>(__brev(static_cast<unsigned>(v)) >> (32 - bits)) : 0;
}
// Total order of points under the reference's tie-break (smaller wins) and its inverse.
__device__ __forceinline__ int point_key(int j, int bs_log2) {
    return (bitrev_low(j & ((1 << bs_log2) - 1), bs_log2) << 21) | (j >> bs_log2);
}
__device__ __forceinline__ int key_to_index(int key, int bs_log2) {
    return bitrev_low(key >> 21, bs_log2) | ((key & 0x1FFFFF) << bs_log2);
}
// Skip threshold: a box whose squared distance to o exceeds this cannot change (rounded up).
__device__ __forceinline__ float skip_threshold(float max_t) { return max_t < 0.f ? -1.f : max_t * 1.00002f; }
// Squared distance from o to an axis-aligned box (0 inside).
__device__ __forceinline__ float box_dist2(float lx, float ly, float lz, float hx, float hy, float hz, float ox, float oy,
                                           float oz) {
    const float ex = fmaxf(fmaxf(lx - ox, ox - hx), 0.f);
    const float ey = fmaxf(fmaxf(ly - oy, oy - hy), 0.f);
    const float ez = fmaxf(fmaxf(lz - oz, oz - hz), 0.f);
    return ex * ex + ey * ey + ez * ez;
}
// Tie key of the point at sorted position p of this cloud (p < 0: no point, sorts last).
__device__ __forceinline__ int key_at(const int* __restrict__ key, int p) { return p < 0 ? INT_MAX : __ldg(key + p); }
// Lane holding the warp's best (v, p): larger value bits, then the smaller tie key of sorted position p.  The keys are read only
// when more than one lane holds the maximum.
__device__ __forceinline__ int warp_best_lane(int v, int p, const int* __restrict__ key, int& wv) {
    wv = __reduce_max_sync(FULL, v);
    const unsigned tied = __ballot_sync(FULL, v == wv);
    if (__popc(tied) == 1) return __ffs(tied) - 1;
    const int k = v == wv ? key_at(key, p) : INT_MAX;
    const int wk = __reduce_min_sync(FULL, k);
    return __ffs(__ballot_sync(FULL, v == wv && k == wk)) - 1;
}
// Candidate of a bucket from its 64 minima (n0, n1 of lane l = sorted points 2l, 2l+1): returns the lane holding it, its value
// bits in wmax and, in take1, whether each lane's better point is its second one.  kp = the lane's pair of tie keys, read only
// on a tie.
__device__ __forceinline__ int bucket_best(float n0, float n1, const int2* kp, int& wmax, bool& take1) {
    const int b0 = __float_as_int(n0), b1 = __float_as_int(n1);          // pads stay at -1
    take1 = b1 > b0;
    const int bl = take1 ? b1 : b0;
    wmax = __reduce_max_sync(FULL, bl);
    const unsigned tied = __ballot_sync(FULL, bl == wmax);
    const unsigned pair = __ballot_sync(FULL, bl == wmax && b0 == b1);
    if (__popc(tied) == 1 && pair == 0u) return __ffs(tied) - 1;
    int kl = INT_MAX;
    if (bl == wmax) {
        const int2 k = __ldg(kp);
        if (b0 == b1) take1 = k.y < k.x;
        kl = take1 ? k.y : k.x;
    }
    const int wk = __reduce_min_sync(FULL, kl);
    return __ffs(__ballot_sync(FULL, bl == wmax && kl == wk)) - 1;
}
// Sorted positions in idx[1, m) -> original indices (start_n + j), after the sampling loop.
__device__ __forceinline__ void positions_to_indices(int* idx, int m, int start_n, const int* __restrict__ key, int bs_log2,
                                                     int tid, int nthreads) {
    __syncthreads();
    for (int i = 1 + tid; i < m; i += nthreads) idx[i] = start_n + key_to_index(__ldg(key + idx[i]), bs_log2);
}
// Final running minima -> tmp (original order).
__device__ __forceinline__ void write_tmp(float* tmp, int start_n, int nb, const float4* pb, const int2* __restrict__ keys,
                                          int bs_log2, int tid, int nthreads) {
    __syncthreads();
    for (int q = tid; q < nb * 32; q += nthreads) {           // q = bucket * 32 + lane
        const float4 B = __ldcg(pb + q);
        const int2 k = __ldg(keys + q);
        if (k.x != INT_MAX) tmp[start_n + key_to_index(k.x, bs_log2)] = B.z;
        if (k.y != INT_MAX) tmp[start_n + key_to_index(k.y, bs_log2)] = B.w;
    }
}
__device__ __forceinline__ unsigned spread3(unsigned x) {   // 10 bits -> every third bit
    x = (x | (x << 16)) & 0x030000FFu;
    x = (x | (x << 8)) & 0x0300F00Fu;
    x = (x | (x << 4)) & 0x030C30C3u;
    x = (x | (x << 2)) & 0x09249249u;
    return x;
}
// Warp min / max of floats through the integer CREDUX path (order-preserving bit map; +-inf allowed).
__device__ __forceinline__ int float_ordered(float f) {
    const int i = __float_as_int(f);
    return i ^ ((i >> 31) & 0x7FFFFFFF);
}
__device__ __forceinline__ float ordered_float(int i) { return __int_as_float(i ^ ((i >> 31) & 0x7FFFFFFF)); }
__device__ __forceinline__ float ordered_min(float v) { return ordered_float(__reduce_min_sync(FULL, float_ordered(v))); }
__device__ __forceinline__ float ordered_max(float v) { return ordered_float(__reduce_max_sync(FULL, float_ordered(v))); }
__device__ __forceinline__ float warp_min(float v) {
#pragma unroll
    for (int o = 16; o; o >>= 1) v = fminf(v, __shfl_xor_sync(FULL, v, o));
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o; o >>= 1) v = fmaxf(v, __shfl_xor_sync(FULL, v, o));
    return v;
}

// Sort elements: (Morton code, index) pairs in global memory, or one packed word (code << 15 | index)
// when a cloud is small enough to be sorted entirely in shared memory.
__device__ __forceinline__ unsigned radix_key(uint2 e) { return e.x; }
__device__ __forceinline__ unsigned radix_key(unsigned e) { return e; }

// Lanes of the warp holding the same BITS-bit digit as the caller (what __match_any_sync returns, but
// built from BITS + 1 ballots: MATCH.ANY costs a few hundred cycles when most lanes differ).
template <int BITS>
__device__ __forceinline__ unsigned peer_mask(unsigned d, bool ok) {
    unsigned m = __ballot_sync(FULL, ok);
#pragma unroll
    for (int b = 0; b < BITS; ++b) {
        const bool bit = (d >> b) & 1u;
        const unsigned bal = __ballot_sync(FULL, bit);
        m &= bit ? bal : ~bal;
    }
    return m;
}

// One stable LSD radix pass on BITS <= 7 bits of (key >> shift).  Warp w owns a contiguous range of the
// input; ranks inside a 32-element step come from the peer masks, so the pass is deterministic.
template <typename E, int BITS>
__device__ __forceinline__ void radix_pass(const E* __restrict__ src, E* __restrict__ dst, int n, int shift,
                                           int (*hist)[128], int* dig_base)
{
    constexpr unsigned mask = (1u << BITS) - 1u;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int per_warp = ((n + kNW - 1) / kNW + 31) & ~31;
    const int lo = warp * per_warp, hi = min(n, lo + per_warp);
    for (int i = tid; i < kNW * 128; i += kT) (&hist[0][0])[i] = 0;
    __syncthreads();
    for (int base = lo; base < hi; base += 32 * kRadixUnroll) {
        unsigned code[kRadixUnroll];
#pragma unroll
        for (int u = 0; u < kRadixUnroll; ++u) {          // independent loads first (L2 latency paid once)
            const int i = base + 32 * u + lane;
            code[u] = i < hi ? radix_key(src[i]) : 0u;
        }
#pragma unroll
        for (int u = 0; u < kRadixUnroll; ++u) {
            const int i = base + 32 * u + lane;
            const bool ok = i < hi;
            const int d = static_cast<int>((code[u] >> shift) & mask);
            const unsigned m = peer_mask<BITS>(d, ok);
            if (ok && lane == __ffs(m) - 1) hist[warp][d] += __popc(m);
            __syncwarp();
        }
    }
    __syncthreads();
    // digit-major, warp-minor exclusive scan
    if (tid < 128) {
        int s = 0;
        for (int w = 0; w < kNW; ++w) s += hist[w][tid];
        dig_base[tid] = s;
    }
    __syncthreads();
    if (warp == 0) {                       // exclusive scan of 128 digit totals, 4 per lane
        int v[4], s = 0;
#pragma unroll
        for (int k = 0; k < 4; ++k) { v[k] = dig_base[lane * 4 + k]; s += v[k]; }
        int inc = s;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int t = __shfl_up_sync(FULL, inc, o);
            if (lane >= o) inc += t;
        }
        int run = inc - s;
#pragma unroll
        for (int k = 0; k < 4; ++k) { dig_base[lane * 4 + k] = run; run += v[k]; }
    }
    __syncthreads();
    if (tid < 128) {
        int run = dig_base[tid];
        for (int w = 0; w < kNW; ++w) { const int c = hist[w][tid]; hist[w][tid] = run; run += c; }
    }
    __syncthreads();
    for (int base = lo; base < hi; base += 32 * kRadixUnroll) {
        E el[kRadixUnroll];
#pragma unroll
        for (int u = 0; u < kRadixUnroll; ++u) {
            const int i = base + 32 * u + lane;
            el[u] = i < hi ? src[i] : E{};
        }
#pragma unroll
        for (int u = 0; u < kRadixUnroll; ++u) {
            const int i = base + 32 * u + lane;
            const bool ok = i < hi;
            const int d = static_cast<int>((radix_key(el[u]) >> shift) & mask);
            const unsigned m = peer_mask<BITS>(d, ok);
            const int rank = __popc(m & ((1u << lane) - 1u));
            int cur = 0;
            if (ok) cur = hist[warp][d];
            __syncwarp();
            if (ok) {
                dst[cur + rank] = el[u];
                if (lane == __ffs(m) - 1) hist[warp][d] = cur + __popc(m);
            }
            __syncwarp();
        }
    }
    __syncthreads();
}

// SMEM_ = true: clouds of at most kSmemSortMaxN points; the three radix passes ping-pong between two
// shared-memory arrays of packed words (17-bit Morton code, 15-bit point index) instead of global memory.
template <bool SMEM_>
__global__ void __launch_bounds__(kT)
fps_bucket_sort_kernel(const float* __restrict__ xyz, const int* __restrict__ offset, const float* __restrict__ tmp,
                       BucketWs ws, int bs_log2, int spad)
{
    extern __shared__ __align__(16) unsigned char dyn[];
    __shared__ float red[6][kNW];
    __shared__ float box[6];
    __shared__ int hist[kNW][128];
    __shared__ int dig_base[128];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int cloud = blockIdx.x;
    const int start_n = cloud ? offset[cloud - 1] : 0;
    const int n = offset[cloud] - start_n;
    if (n <= 0) return;
    const float* cx = xyz + 3 * static_cast<size_t>(start_n);
    float4* __restrict__ pa = ws.pa + static_cast<size_t>(cloud) * (ws.stride / 2);
    float4* __restrict__ pb = ws.pb + static_cast<size_t>(cloud) * (ws.stride / 2);
    int2* __restrict__ keys = ws.keys + static_cast<size_t>(cloud) * (ws.stride / 2);
    uint2* ka = SMEM_ ? nullptr : ws.key_a + static_cast<size_t>(cloud) * ws.stride;
    uint2* kb = SMEM_ ? nullptr : ws.key_b + static_cast<size_t>(cloud) * ws.stride;

    // ---- bounding box --------------------------------------------------------------------------------
    float mn[3] = {INFINITY, INFINITY, INFINITY}, mx[3] = {-INFINITY, -INFINITY, -INFINITY};
    for (int j = tid; j < n; j += kT) {
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            const float v = __ldg(cx + 3 * static_cast<size_t>(j) + a);
            mn[a] = fminf(mn[a], v); mx[a] = fmaxf(mx[a], v);
        }
    }
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const float lo = warp_min(mn[a]), hi = warp_max(mx[a]);
        if (lane == 0) { red[a][warp] = lo; red[3 + a][warp] = hi; }
    }
    __syncthreads();
    if (tid < 6) {
        float v = red[tid][0];
        for (int w = 1; w < kNW; ++w) v = tid < 3 ? fminf(v, red[tid][w]) : fmaxf(v, red[tid][w]);
        box[tid] = v;
    }
    __syncthreads();
    float inv[3];
    float scale = 0.f;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const float ext = box[3 + a] - box[a];
        inv[a] = ext > 0.f ? (static_cast<float>(1 << (SMEM_ ? (a == 2 ? 5 : 6) : 7)) - 0.001f) / ext : 0.f;
        scale = fmaxf(scale, fmaxf(fabsf(box[a]), fabsf(box[3 + a])));
    }
    const float slack = 4e-6f * scale;       // absolute inflation of every bucket box

    // ---- Morton keys + stable radix sort ----------------------------------------------------------------
    unsigned* sa = reinterpret_cast<unsigned*>(dyn);
    unsigned* sb = sa + spad;
    for (int j = tid; j < n; j += kT) {
        unsigned code = 0;
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            const unsigned qmax = (1u << (SMEM_ ? (a == 2 ? 5 : 6) : 7)) - 1u;
            const float v = __ldg(cx + 3 * static_cast<size_t>(j) + a);
            const unsigned q = min(qmax, static_cast<unsigned>(fmaxf((v - box[a]) * inv[a], 0.f)));
            code |= spread3(q) << a;
        }
        if (SMEM_) sa[j] = (code << 15) | static_cast<unsigned>(j);
        else ka[j] = make_uint2(code, static_cast<unsigned>(j));
    }
    __syncthreads();
    if (SMEM_) {
        radix_pass<unsigned, 6>(sa, sb, n, 15, hist, dig_base);
        radix_pass<unsigned, 6>(sb, sa, n, 21, hist, dig_base);
        radix_pass<unsigned, 5>(sa, sb, n, 27, hist, dig_base);
    } else {
        radix_pass<uint2, 7>(ka, kb, n, 0, hist, dig_base);
        radix_pass<uint2, 7>(kb, ka, n, 7, hist, dig_base);
        radix_pass<uint2, 7>(ka, kb, n, 14, hist, dig_base);
    }

    // ---- sorted points, running minima, bucket boxes and initial candidates -------------------------------
    // A warp writes one bucket (64 consecutive sorted points, two adjacent ones per lane) per step and reduces its
    // box and best candidate from the registers it just filled; kGatherUnroll buckets are in flight per warp.
    const int nb = (n + kBP - 1) / kBP;
    float4* __restrict__ blo = ws.box_lo + static_cast<size_t>(cloud) * ws.nbmax;
    float4* __restrict__ bhi = ws.box_hi + static_cast<size_t>(cloud) * ws.nbmax;
    float4* __restrict__ bxyz = ws.bxyz + static_cast<size_t>(cloud) * ws.nbmax;
    for (int bk0 = warp; bk0 < nb; bk0 += kNW * kGatherUnroll) {
        int j[kGatherUnroll][2];
        float x[kGatherUnroll][2], y[kGatherUnroll][2], z[kGatherUnroll][2], t[kGatherUnroll][2];
#pragma unroll
        for (int u = 0; u < kGatherUnroll; ++u)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int p = (bk0 + u * kNW) * kBP + 2 * lane + h;
                j[u][h] = p < n ? (SMEM_ ? static_cast<int>(sb[p] & 0x7FFFu) : static_cast<int>(kb[p].y)) : -1;
            }
#pragma unroll
        for (int u = 0; u < kGatherUnroll; ++u)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                if (j[u][h] >= 0) {
                    const float* q = cx + 3 * static_cast<size_t>(j[u][h]);
                    x[u][h] = __ldg(q); y[u][h] = __ldg(q + 1); z[u][h] = __ldg(q + 2);
                    t[u][h] = tmp ? __ldg(tmp + start_n + j[u][h]) : 1e10f;
                } else {
                    x[u][h] = y[u][h] = z[u][h] = 0.f;
                    t[u][h] = -1.0f;
                }
            }
#pragma unroll
        for (int u = 0; u < kGatherUnroll; ++u) {
            const int bk = bk0 + u * kNW;
            if (bk >= nb) break;                      // warp-uniform
            const int k0 = j[u][0] >= 0 ? point_key(j[u][0], bs_log2) : INT_MAX;
            const int k1 = j[u][1] >= 0 ? point_key(j[u][1], bs_log2) : INT_MAX;
            pa[bk * 32 + lane] = make_float4(x[u][0], x[u][1], y[u][0], y[u][1]);
            pb[bk * 32 + lane] = make_float4(z[u][0], z[u][1], t[u][0], t[u][1]);
            keys[bk * 32 + lane] = make_int2(k0, k1);
            const bool ok0 = j[u][0] >= 0, ok1 = j[u][1] >= 0;
            const float lx = ordered_min(fminf(ok0 ? x[u][0] : INFINITY, ok1 ? x[u][1] : INFINITY));
            const float ly = ordered_min(fminf(ok0 ? y[u][0] : INFINITY, ok1 ? y[u][1] : INFINITY));
            const float lz = ordered_min(fminf(ok0 ? z[u][0] : INFINITY, ok1 ? z[u][1] : INFINITY));
            const float hx = ordered_max(fmaxf(ok0 ? x[u][0] : -INFINITY, ok1 ? x[u][1] : -INFINITY));
            const float hy = ordered_max(fmaxf(ok0 ? y[u][0] : -INFINITY, ok1 ? y[u][1] : -INFINITY));
            const float hz = ordered_max(fmaxf(ok0 ? z[u][0] : -INFINITY, ok1 ? z[u][1] : -INFINITY));
            const int b0 = __float_as_int(t[u][0]), b1 = __float_as_int(t[u][1]);
            const bool take1 = b1 > b0 || (b1 == b0 && k1 < k0);
            const int bl = take1 ? b1 : b0, kl = take1 ? k1 : k0;
            const int wmax = __reduce_max_sync(FULL, bl);
            const int wkey = __reduce_min_sync(FULL, bl == wmax ? kl : INT_MAX);
            if (lane == 0) {
                blo[bk] = make_float4(lx - slack, ly - slack, lz - slack, __int_as_float(wmax));
                bhi[bk] = make_float4(hx + slack, hy + slack, hz + slack, __int_as_float(wmax));
            }
            if (bl == wmax && kl == wkey)
                bxyz[bk] = make_float4(take1 ? x[u][1] : x[u][0], take1 ? y[u][1] : y[u][0], take1 ? z[u][1] : z[u][0],
                                       __int_as_float(bk * kBP + 2 * lane + (take1 ? 1 : 0)));
        }
    }
}

// MT_ = 512: 16 warps per cloud, 2 clouds per SM (shortest iteration; batches up to 2 clouds per SM).
// MT_ = 256:  8 warps per cloud, 4 clouds per SM.
// MT_ = 128:  4 warps per cloud, 8 clouds per SM (least per-warp overhead per cloud, most clouds in flight to
//             hide the barriers and the memory round trip: the throughput shape for large batches).
// Either way <= 64 registers per thread.
template <int MT_>
__global__ void __launch_bounds__(MT_, 1024 / MT_)
fps_bucket_kernel(const float* __restrict__ xyz, const int* __restrict__ offset, const int* __restrict__ new_offset,
                  float* tmp, int* __restrict__ idx, BucketWs ws, int bs_log2)
{
    constexpr int kMT = MT_, kMNW = MT_ / 32;     // shadow the defaults
    extern __shared__ __align__(16) unsigned char dyn[];
    __shared__ int nact;
    __shared__ int4 wres[kMNW];           // per owner warp: (value bits, sorted position, bucket, -)

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int cloud = blockIdx.x;
    const int start_n = cloud ? offset[cloud - 1] : 0;
    const int n = offset[cloud] - start_n;
    const int start_m = cloud ? new_offset[cloud - 1] : 0;
    const int m = new_offset[cloud] - start_m;
    if (m <= 0 || n <= 0) return;
    if (tid == 0) idx[start_m] = start_n;                      // sampling_cuda_kernel.cu:39
    if (m == 1) return;

    const int nb = (n + kBP - 1) / kBP;
    float4* blo = reinterpret_cast<float4*>(dyn);                                   // [nbmax] box min, w = skip threshold
    float4* bhi = blo + ws.nbmax;                                                   // [nbmax] box max, w = candidate value bits
    float4* cxyz = bhi + ws.nbmax;                                                  // [nbmax] candidate x,y,z,sorted position bits
    int* alist = reinterpret_cast<int*>(cxyz + ws.nbmax);                           // [nbmax] active buckets

    const float4* __restrict__ pa = ws.pa + static_cast<size_t>(cloud) * (ws.stride / 2);
    float4* pb = ws.pb + static_cast<size_t>(cloud) * (ws.stride / 2);
    const int2* __restrict__ keys = ws.keys + static_cast<size_t>(cloud) * (ws.stride / 2);
    const int* __restrict__ key = reinterpret_cast<const int*>(keys);

    // ---- owner ranges: warp w owns buckets [r0, r1); lane l looks after r0 + l, r0 + l + 32, ... -------------
    const int per = (nb + kMNW - 1) / kMNW;
    const int r0 = min(nb, warp * per), r1 = min(nb, r0 + per);
    {
        const float4* glo = ws.box_lo + static_cast<size_t>(cloud) * ws.nbmax;
        const float4* ghi = ws.box_hi + static_cast<size_t>(cloud) * ws.nbmax;
        const float4* gx = ws.bxyz + static_cast<size_t>(cloud) * ws.nbmax;
        for (int bk = tid; bk < nb; bk += kMT) {
            float4 lo = glo[bk];
            lo.w = skip_threshold(lo.w);                     // w held the bucket's initial max t
            blo[bk] = lo; bhi[bk] = ghi[bk]; cxyz[bk] = gx[bk];
        }
        if (tid == 0) nact = 0;
    }
    __syncthreads();
    // union box of the range (registers, fixed) and the range candidate
    float ulx = INFINITY, uly = INFINITY, ulz = INFINITY, uhx = -INFINITY, uhy = -INFINITY, uhz = -INFINITY;
    for (int bk = r0 + lane; bk < r1; bk += 32) {
        const float4 lo = blo[bk], hi = bhi[bk];
        ulx = fminf(ulx, lo.x); uly = fminf(uly, lo.y); ulz = fminf(ulz, lo.z);
        uhx = fmaxf(uhx, hi.x); uhy = fmaxf(uhy, hi.y); uhz = fmaxf(uhz, hi.z);
    }
    ulx = warp_min(ulx); uly = warp_min(uly); ulz = warp_min(ulz);
    uhx = warp_max(uhx); uhy = warp_max(uhy); uhz = warp_max(uhz);

    auto refresh_range = [&]() {          // best candidate over the owned buckets -> wres[warp]
        int bv = INT_MIN, bpos = -1, bbk = r0;
        for (int bk = r0 + lane; bk < r1; bk += 32) {
            const int v = __float_as_int(bhi[bk].w), p = __float_as_int(cxyz[bk].w);
            if (v > bv || (v == bv && key_at(key, p) < key_at(key, bpos))) { bv = v; bpos = p; bbk = bk; }
        }
        int wv;
        const int wl = warp_best_lane(bv, bpos, key, wv);
        if (lane == wl) wres[warp] = make_int4(wv, bpos, bbk, 0);
        return wv;
    };
    float range_thr = skip_threshold(__int_as_float(refresh_range()));     // r0 == r1: INT_MIN -> negative -> -1

    float ox = __ldg(xyz + 3 * static_cast<size_t>(start_n)), oy = __ldg(xyz + 3 * static_cast<size_t>(start_n) + 1),
          oz = __ldg(xyz + 3 * static_cast<size_t>(start_n) + 2);
    __syncthreads();

    for (int it = 1; it < m; ++it) {
        // ---- (a) owner warps: can anything in my range change?  which buckets? ------------------------------
        bool dirty = false;
        if (r0 < r1 && !(box_dist2(ulx, uly, ulz, uhx, uhy, uhz, ox, oy, oz) > range_thr)) {
            for (int base = r0; base < r1; base += 32) {
                const int bk = base + lane;
                bool act = false;
                if (bk < r1) {
                    const float4 lo = blo[bk], hi = bhi[bk];
                    act = !(box_dist2(lo.x, lo.y, lo.z, hi.x, hi.y, hi.z, ox, oy, oz) > lo.w);
                }
                const unsigned mask = __ballot_sync(FULL, act);
                if (mask) {
                    dirty = true;
                    int pos = 0;
                    if (lane == 0) pos = atomicAdd(&nact, __popc(mask));
                    pos = __shfl_sync(FULL, pos, 0);
                    if (act) alist[pos + __popc(mask & ((1u << lane) - 1u))] = bk;
                }
            }
        }
        __syncthreads();
        const int na = nact;

        // ---- (b) exact update of the surviving buckets: one warp per bucket, kBatch buckets in flight ---------
        const uint64_t ox2 = pack2(ox, ox), oy2 = pack2(oy, oy), oz2 = pack2(oz, oz);
        for (int a0 = warp; a0 < na; a0 += kMNW * kBatch) {
            int bk[kBatch];
            float4 A[kBatch], B[kBatch];
#pragma unroll
            for (int u = 0; u < kBatch; ++u) {
                const int a = a0 + u * kMNW;
                bk[u] = a < na ? alist[a] : -1;
                if (bk[u] >= 0) {
                    A[u] = __ldg(pa + bk[u] * 32 + lane);
                    B[u] = __ldcg(pb + bk[u] * 32 + lane);
                }
            }
#pragma unroll
            for (int u = 0; u < kBatch; ++u) {
                if (bk[u] < 0) break;                         // warp-uniform
                const uint64_t dx = sub2(pack2(A[u].x, A[u].y), ox2), dy = sub2(pack2(A[u].z, A[u].w), oy2),
                               dz = sub2(pack2(B[u].x, B[u].y), oz2);
                uint64_t d = mul2(dy, dy);
                d = fma2(dx, dx, d);
                d = fma2(dz, dz, d);
                float d0, d1;
                unpack2(d, d0, d1);
                const float n0 = fminf(d0, B[u].z), n1 = fminf(d1, B[u].w);
                if (n0 < B[u].z || n1 < B[u].w) __stcg(reinterpret_cast<float2*>(pb + bk[u] * 32 + lane) + 1, make_float2(n0, n1));
                int wmax;
                bool take1;
                const int wl = bucket_best(n0, n1, keys + bk[u] * 32 + lane, wmax, take1);
                if (lane == wl) {
                    cxyz[bk[u]] = make_float4(take1 ? A[u].y : A[u].x, take1 ? A[u].w : A[u].z, take1 ? B[u].y : B[u].x,
                                              __int_as_float(bk[u] * kBP + 2 * lane + (take1 ? 1 : 0)));
                    bhi[bk[u]].w = __int_as_float(wmax);
                    blo[bk[u]].w = skip_threshold(__int_as_float(wmax));
                }
            }
        }
        __syncthreads();
        if (tid == 0) nact = 0;

        // ---- (c) touched ranges refresh their candidate; block arg-max over the range candidates ---------------
        if (dirty) range_thr = skip_threshold(__int_as_float(refresh_range()));
        __syncthreads();
        {
            int4 c = make_int4(INT_MIN, -1, 0, 0);
            if (lane < kMNW) c = wres[lane];
            int gv;
            const int src = warp_best_lane(c.x, c.y, key, gv);
            const int bstar = __shfl_sync(FULL, c.z, src);
            const float4 w = cxyz[bstar];
            ox = w.x; oy = w.y; oz = w.z;
            if (tid == 0) idx[start_m + it] = __float_as_int(w.w);
        }
    }

    positions_to_indices(idx + start_m, m, start_n, key, bs_log2, tid, kMT);
    if (tmp) write_tmp(tmp, start_n, nb, pb, keys, bs_log2, tid, kMT);
}

// ---- single-barrier main kernel ("v2") ------------------------------------------------------------------------------------
// Same tables, same exact update, same candidates -- a different schedule.  The kernel above spends an iteration on three
// block barriers (owner warps collect the active buckets | all warps process them | owners refresh | arg-max) around one
// memory round trip.  Here bucket bk belongs to warp bk mod W for good (the buckets are Morton-sorted, so the ~10 buckets a
// new sample touches are consecutive and land on ~10 different warps), and a warp does everything for its own buckets
// back to back: box tests (one bucket per lane per pass), exact update of its active buckets (two in flight), refresh of
// its best candidate -- then publishes (value, key, x, y, z) in a double-buffered slot and meets the others at ONE barrier,
// after which every warp reduces the W slots to the next sample.  The winner's coordinates travel in the slot, so nobody
// reads a bucket table entry that a faster warp may already be overwriting for the next iteration.
template <int MT_>
__global__ void __launch_bounds__(MT_, 1024 / MT_)
fps_bucket_kernel2(const float* __restrict__ xyz, const int* __restrict__ offset, const int* __restrict__ new_offset,
                   float* tmp, int* __restrict__ idx, BucketWs ws, int bs_log2)
{
    constexpr int kMT = MT_, kMNW = MT_ / 32;
    extern __shared__ __align__(16) unsigned char dyn[];
    struct Slot { int v, p; float x, y, z; int pad[3]; };     // value bits, sorted position, coordinates
    __shared__ Slot slot[2][kMNW];

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int cloud = blockIdx.x;
    const int start_n = cloud ? offset[cloud - 1] : 0;
    const int n = offset[cloud] - start_n;
    const int start_m = cloud ? new_offset[cloud - 1] : 0;
    const int m = new_offset[cloud] - start_m;
    if (m <= 0 || n <= 0) return;
    if (tid == 0) idx[start_m] = start_n;                      // sampling_cuda_kernel.cu:39
    if (m == 1) return;

    const int nb = (n + kBP - 1) / kBP;
    float4* blo = reinterpret_cast<float4*>(dyn);                                   // [nbmax] box min, w = skip threshold
    float4* bhi = blo + ws.nbmax;                                                   // [nbmax] box max, w = candidate value bits
    float4* cxyz = bhi + ws.nbmax;                                                  // [nbmax] candidate x,y,z,sorted position bits

    const float4* __restrict__ pa = ws.pa + static_cast<size_t>(cloud) * (ws.stride / 2);
    float4* pb = ws.pb + static_cast<size_t>(cloud) * (ws.stride / 2);
    const int2* __restrict__ keys = ws.keys + static_cast<size_t>(cloud) * (ws.stride / 2);
    const int* __restrict__ key = reinterpret_cast<const int*>(keys);
    {
        const float4* glo = ws.box_lo + static_cast<size_t>(cloud) * ws.nbmax;
        const float4* ghi = ws.box_hi + static_cast<size_t>(cloud) * ws.nbmax;
        const float4* gx = ws.bxyz + static_cast<size_t>(cloud) * ws.nbmax;
        for (int bk = tid; bk < nb; bk += kMT) {
            float4 lo = glo[bk];
            lo.w = skip_threshold(lo.w);                     // w held the bucket's initial max t
            blo[bk] = lo; bhi[bk] = ghi[bk]; cxyz[bk] = gx[bk];
        }
    }
    __syncthreads();

    // best candidate over this warp's buckets (warp, warp + W, ...) -> registers of every lane
    int my_v = INT_MIN, my_p = -1;
    float my_x = 0.f, my_y = 0.f, my_z = 0.f;
    auto refresh_own = [&]() {
        int bv = INT_MIN, bpos = -1, bbk = -1;
        for (int bk = warp + kMNW * lane; bk < nb; bk += kMNW * 32) {
            const int v = __float_as_int(bhi[bk].w), p = __float_as_int(cxyz[bk].w);
            if (v > bv || (v == bv && key_at(key, p) < key_at(key, bpos))) { bv = v; bpos = p; bbk = bk; }
        }
        const int src = warp_best_lane(bv, bpos, key, my_v);
        my_p = __shfl_sync(FULL, bpos, src);
        const int wb = __shfl_sync(FULL, bbk, src);
        float4 w = make_float4(0.f, 0.f, 0.f, 0.f);
        if (wb >= 0) w = cxyz[wb];
        my_x = w.x; my_y = w.y; my_z = w.z;
    };
    refresh_own();

    float ox = __ldg(xyz + 3 * static_cast<size_t>(start_n)), oy = __ldg(xyz + 3 * static_cast<size_t>(start_n) + 1),
          oz = __ldg(xyz + 3 * static_cast<size_t>(start_n) + 2);

    for (int it = 1; it < m; ++it) {
        const uint64_t ox2 = pack2(ox, ox), oy2 = pack2(oy, oy), oz2 = pack2(oz, oz);
        bool dirty = false;
        // ---- own buckets: test 32 per pass, update the active ones (kBatch in flight) ---------------------------------
        for (int base = warp; base < nb; base += kMNW * 32) {
            const int bk_l = base + kMNW * lane;
            bool act = false;
            if (bk_l < nb) {
                const float4 lo = blo[bk_l], hi = bhi[bk_l];
                act = !(box_dist2(lo.x, lo.y, lo.z, hi.x, hi.y, hi.z, ox, oy, oz) > lo.w);
            }
            unsigned mask = __ballot_sync(FULL, act);
            dirty |= mask != 0u;
            while (mask) {
                int bk[kBatch];
                float4 A[kBatch], B[kBatch];
#pragma unroll
                for (int u = 0; u < kBatch; ++u) {
                    if (mask) {
                        const int l = __ffs(mask) - 1;
                        mask &= mask - 1;
                        bk[u] = base + kMNW * l;
                        A[u] = __ldg(pa + bk[u] * 32 + lane);
                        B[u] = __ldcg(pb + bk[u] * 32 + lane);
                    } else {
                        bk[u] = -1;
                    }
                }
#pragma unroll
                for (int u = 0; u < kBatch; ++u) {
                    if (bk[u] < 0) break;                         // warp-uniform
                    const uint64_t dx = sub2(pack2(A[u].x, A[u].y), ox2), dy = sub2(pack2(A[u].z, A[u].w), oy2),
                                   dz = sub2(pack2(B[u].x, B[u].y), oz2);
                    uint64_t d = mul2(dy, dy);
                    d = fma2(dx, dx, d);
                    d = fma2(dz, dz, d);
                    float d0, d1;
                    unpack2(d, d0, d1);
                    const float n0 = fminf(d0, B[u].z), n1 = fminf(d1, B[u].w);
                    if (n0 < B[u].z || n1 < B[u].w) __stcg(reinterpret_cast<float2*>(pb + bk[u] * 32 + lane) + 1, make_float2(n0, n1));
                    int wmax;
                    bool take1;
                    const int wl = bucket_best(n0, n1, keys + bk[u] * 32 + lane, wmax, take1);
                    if (lane == wl) {
                        cxyz[bk[u]] = make_float4(take1 ? A[u].y : A[u].x, take1 ? A[u].w : A[u].z, take1 ? B[u].y : B[u].x,
                                                  __int_as_float(bk[u] * kBP + 2 * lane + (take1 ? 1 : 0)));
                        bhi[bk[u]].w = __int_as_float(wmax);
                        blo[bk[u]].w = skip_threshold(__int_as_float(wmax));
                    }
                }
            }
        }
        // ---- this warp's candidate (only the warp itself writes its buckets' entries) ------------------------------------
        if (dirty) {
            __syncwarp();
            refresh_own();
        }
        Slot* sl = slot[it & 1];
        if (lane == 0) { sl[warp].v = my_v; sl[warp].p = my_p; sl[warp].x = my_x; sl[warp].y = my_y; sl[warp].z = my_z; }
        __syncthreads();
        {
            int cv = INT_MIN, cp = -1;
            if (lane < kMNW) { cv = sl[lane].v; cp = sl[lane].p; }
            int gv;
            const int src = warp_best_lane(cv, cp, key, gv);
            ox = sl[src].x; oy = sl[src].y; oz = sl[src].z;
            if (tid == 0) idx[start_m + it] = sl[src].p;
        }
    }

    positions_to_indices(idx + start_m, m, start_n, key, bs_log2, tid, kMT);
    if (tmp) write_tmp(tmp, start_n, nb, pb, keys, bs_log2, tid, kMT);
}

// ---- register-resident bucket tables ("v3") --------------------------------------------------------------------------------
// At small batches (one cloud per SM or fewer) an iteration is a DEPENDENT CHAIN: a profile shows
// ~190 warp instructions per warp per iteration, low issue utilisation, most samples waiting at the barrier for
// the warp that had a bucket to update.  v3 keeps the single barrier of v2 and shortens the chain: the table entries of a
// warp's OWN buckets (box, skip threshold, candidate value / key / coordinates: 12 registers per bucket, BPL buckets per lane)
// never leave registers -- box tests need no shared-memory loads, an update hands the new candidate to the owner lane with
// three shuffles, the warp's candidate is two CREDUX over registers and the winning lane publishes its slot directly.
template <int MT_, int BPL>
__global__ void __launch_bounds__(MT_, (MT_ == 512 && BPL >= 3) ? 1 : (1024 / MT_ > 2 ? 2 : 1024 / MT_))     // raw-mesh shapes: one CTA per SM, 128 registers
fps_bucket_kernel3(const float* __restrict__ xyz, const int* __restrict__ offset, const int* __restrict__ new_offset,
                   float* tmp, int* __restrict__ idx, BucketWs ws, int bs_log2)
{
    constexpr int kMT = MT_, kMNW = MT_ / 32;
    struct Slot { int v, p; float x, y, z; int pad[3]; };     // value bits, sorted position, coordinates
    __shared__ Slot slot[2][kMNW];

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int cloud = blockIdx.x;
    const int start_n = cloud ? offset[cloud - 1] : 0;
    const int n = offset[cloud] - start_n;
    const int start_m = cloud ? new_offset[cloud - 1] : 0;
    const int m = new_offset[cloud] - start_m;
    if (m <= 0 || n <= 0) return;
    if (tid == 0) idx[start_m] = start_n;                      // sampling_cuda_kernel.cu:39
    if (m == 1) return;

    const int nb = (n + kBP - 1) / kBP;
    const float4* __restrict__ pa = ws.pa + static_cast<size_t>(cloud) * (ws.stride / 2);
    float4* pb = ws.pb + static_cast<size_t>(cloud) * (ws.stride / 2);
    const int2* __restrict__ keys = ws.keys + static_cast<size_t>(cloud) * (ws.stride / 2);
    const int* __restrict__ key = reinterpret_cast<const int*>(keys);

    // own buckets: bucket (warp + W * (lane + 32 j)), j < BPL; ck = sorted position of the candidate
    float lx[BPL], ly[BPL], lz[BPL], hx[BPL], hy[BPL], hz[BPL], thr[BPL], cx[BPL], cy[BPL], cz[BPL];
    int cv[BPL], ck[BPL];
    {
        const float4* glo = ws.box_lo + static_cast<size_t>(cloud) * ws.nbmax;
        const float4* ghi = ws.box_hi + static_cast<size_t>(cloud) * ws.nbmax;
        const float4* gx = ws.bxyz + static_cast<size_t>(cloud) * ws.nbmax;
#pragma unroll
        for (int j = 0; j < BPL; ++j) {
            const int bk = warp + kMNW * (lane + 32 * j);
            if (bk < nb) {
                const float4 lo = glo[bk], hi = ghi[bk], c = gx[bk];
                lx[j] = lo.x; ly[j] = lo.y; lz[j] = lo.z; thr[j] = skip_threshold(lo.w);
                hx[j] = hi.x; hy[j] = hi.y; hz[j] = hi.z; cv[j] = __float_as_int(hi.w);
                cx[j] = c.x; cy[j] = c.y; cz[j] = c.z; ck[j] = __float_as_int(c.w);
            } else {
                lx[j] = ly[j] = lz[j] = INFINITY; hx[j] = hy[j] = hz[j] = -INFINITY; thr[j] = -1.f;     // never active
                cv[j] = INT_MIN; ck[j] = -1; cx[j] = cy[j] = cz[j] = 0.f;
            }
        }
    }
    float ox = __ldg(xyz + 3 * static_cast<size_t>(start_n)), oy = __ldg(xyz + 3 * static_cast<size_t>(start_n) + 1),
          oz = __ldg(xyz + 3 * static_cast<size_t>(start_n) + 2);

    for (int it = 1; it < m; ++it) {
        const uint64_t ox2 = pack2(ox, ox), oy2 = pack2(oy, oy), oz2 = pack2(oz, oz);
#pragma unroll
        for (int j = 0; j < BPL; ++j) {
            const bool act = !(box_dist2(lx[j], ly[j], lz[j], hx[j], hy[j], hz[j], ox, oy, oz) > thr[j]);
            unsigned mask = __ballot_sync(FULL, act);
            while (mask) {
                int ol[kBatch];                               // owner lanes of the buckets in flight
                float4 A[kBatch], B[kBatch];
#pragma unroll
                for (int u = 0; u < kBatch; ++u) {
                    if (mask) {
                        ol[u] = __ffs(mask) - 1;
                        mask &= mask - 1;
                        const int bk = warp + kMNW * (ol[u] + 32 * j);
                        A[u] = __ldg(pa + bk * 32 + lane);
                        B[u] = __ldcg(pb + bk * 32 + lane);
                    } else {
                        ol[u] = -1;
                    }
                }
#pragma unroll
                for (int u = 0; u < kBatch; ++u) {
                    if (ol[u] < 0) break;                         // warp-uniform
                    const int bk = warp + kMNW * (ol[u] + 32 * j);
                    const uint64_t dx = sub2(pack2(A[u].x, A[u].y), ox2), dy = sub2(pack2(A[u].z, A[u].w), oy2),
                                   dz = sub2(pack2(B[u].x, B[u].y), oz2);
                    uint64_t d = mul2(dy, dy);
                    d = fma2(dx, dx, d);
                    d = fma2(dz, dz, d);
                    float d0, d1;
                    unpack2(d, d0, d1);
                    const float n0 = fminf(d0, B[u].z), n1 = fminf(d1, B[u].w);
                    if (n0 < B[u].z || n1 < B[u].w) __stcg(reinterpret_cast<float2*>(pb + bk * 32 + lane) + 1, make_float2(n0, n1));
                    int wmax;
                    bool take1;
                    const int wl = bucket_best(n0, n1, keys + bk * 32 + lane, wmax, take1);      // the lane holding the candidate point
                    const float nx = __shfl_sync(FULL, take1 ? A[u].y : A[u].x, wl), ny = __shfl_sync(FULL, take1 ? A[u].w : A[u].z, wl),
                                nz = __shfl_sync(FULL, take1 ? B[u].y : B[u].x, wl);
                    const int np = __shfl_sync(FULL, bk * kBP + 2 * lane + (take1 ? 1 : 0), wl);
                    if (lane == ol[u]) { cv[j] = wmax; ck[j] = np; thr[j] = skip_threshold(__int_as_float(wmax)); cx[j] = nx; cy[j] = ny; cz[j] = nz; }
                }
            }
        }
        // ---- this warp's candidate: registers only -------------------------------------------------------------------------
        int bv = cv[0], bpos = ck[0];
        float bx = cx[0], by = cy[0], bz = cz[0];
#pragma unroll
        for (int j = 1; j < BPL; ++j)
            if (cv[j] > bv || (cv[j] == bv && key_at(key, ck[j]) < key_at(key, bpos))) { bv = cv[j]; bpos = ck[j]; bx = cx[j]; by = cy[j]; bz = cz[j]; }
        int wv;
        const int wl = warp_best_lane(bv, bpos, key, wv);
        Slot* sl = slot[it & 1];
        if (lane == wl) { sl[warp].v = wv; sl[warp].p = bpos; sl[warp].x = bx; sl[warp].y = by; sl[warp].z = bz; }
        __syncthreads();
        {
            int sv = INT_MIN, sp = -1;
            if (lane < kMNW) { sv = sl[lane].v; sp = sl[lane].p; }
            int gv;
            const int src = warp_best_lane(sv, sp, key, gv);
            ox = sl[src].x; oy = sl[src].y; oz = sl[src].z;
            if (tid == 0) idx[start_m + it] = sl[src].p;
        }
    }

    positions_to_indices(idx + start_m, m, start_n, key, bs_log2, tid, kMT);
    if (tmp) write_tmp(tmp, start_n, nb, pb, keys, bs_log2, tid, kMT);
}

template <int MT_, int BPL>
int launch_main3(int b, const float* xyz, const int* offset, const int* new_offset, float* tmp, int* idx, const BucketWs& ws,
                 int bs_log2, cudaStream_t stream)
{
    fps_bucket_kernel3<MT_, BPL><<<b, MT_, 0, stream>>>(xyz, offset, new_offset, tmp, idx, ws, bs_log2);
    return check_launch("fps_bucket_kernel3");
}

template <int MT_>
int launch_main2(int b, size_t smem, const float* xyz, const int* offset, const int* new_offset, float* tmp, int* idx,
                 const BucketWs& ws, int bs_log2, cudaStream_t stream)
{
    const int rc_attr = ensure_dynamic_smem(reinterpret_cast<const void*>(fps_bucket_kernel2<MT_>), smem);
    if (rc_attr != TGN_OK) return rc_attr;
    fps_bucket_kernel2<MT_><<<b, MT_, smem, stream>>>(xyz, offset, new_offset, tmp, idx, ws, bs_log2);
    return check_launch("fps_bucket_kernel2");
}

template <int MT_>
int launch_main(int b, size_t smem, const float* xyz, const int* offset, const int* new_offset, float* tmp, int* idx,
                const BucketWs& ws, int bs_log2, cudaStream_t stream)
{
    const int rc_attr = ensure_dynamic_smem(reinterpret_cast<const void*>(fps_bucket_kernel<MT_>), smem);
    if (rc_attr != TGN_OK) return rc_attr;
    fps_bucket_kernel<MT_><<<b, MT_, smem, stream>>>(xyz, offset, new_offset, tmp, idx, ws, bs_log2);
    return check_launch("fps_bucket_kernel");
}

}  // namespace

// Largest cloud the bucket kernel takes (the bucket table must fit in shared memory).
int fps_bucket_max_points() { return kMaxBuckets * kBP; }

int fps_bucket_launch(int b, int n_max, const float* xyz, const int* offset, const int* new_offset, float* tmp, int* idx,
                      int bs_log2, int shape, cudaStream_t stream)
{
    BucketWs ws{};
    ws.stride = (n_max + kBP - 1) / kBP * kBP;
    ws.nbmax = ws.stride / kBP;
    // The main kernel's shape is decided before anything is allocated or launched: a refused shape launches nothing.
    const size_t smem = static_cast<size_t>(ws.nbmax) * (sizeof(float4) * 3 + sizeof(int));
    // Warps per cloud by batch size: the more clouds per SM are available, the narrower the CTA (fewer
    // redundant per-warp steps and cheaper barriers per cloud, more clouds in flight to hide latency).
    const int sms = sm_count();
    auto fits = [&](int per_sm) { return static_cast<size_t>(per_sm) * (smem + 1024) <= 220 * 1024; };
    // Auto (shape 0), 24k-point clouds -> 1024 samples: up to 4 clouds per SM the single-barrier kernel with register-resident
    // tables at 16 warps per cloud; beyond that the batch is DRAM-bound and the three-barrier kernel at 4 warps per cloud,
    // 8 clouds per SM, is used.
    // Raw meshes (one cloud of 1e5..2e5 vertices -> 24 000, gen_utils.py:135-140): the same kernel with 4-8 buckets per lane
    // while every cloud can have an SM to itself.
    if (shape == 0 && ((b <= 4 * sms && ws.nbmax <= 2 * 512) || (b <= sms && ws.nbmax <= 8 * 512))) shape = 200 + 16;
    const bool v2 = shape >= 100 && shape < 200;          // 100 + W: the single-barrier schedule (fps_bucket_kernel2)
    const bool v3 = shape >= 200;                         // 200 + W: the same with register-resident bucket tables (fps_bucket_kernel3)
    int warps = shape % 100;
    if (warps == 0) warps = (b > 4 * sms && fits(8)) ? 4 : (b > 2 * sms && fits(4)) ? 8 : 16;
    if (v3 && warps != 32 && warps != 16 && warps != 8 && warps != 4) {
        set_error("furthestsampling: bucket kernel v3 has no shape of %d warps per cloud", warps);
        return TGN_ERR_INVALID;
    }
    if (v2 && warps != 32 && warps != 16 && warps != 8 && warps != 4 && warps != 2) {
        set_error("furthestsampling: bucket kernel v2 has no shape of %d warps per cloud", warps);
        return TGN_ERR_INVALID;
    }
    if (!v2 && !v3 && warps != 16 && warps != 8 && warps != 4 && warps != 2 && warps != 1) {
        set_error("furthestsampling: bucket kernel has no shape of %d warps per cloud", warps);
        return TGN_ERR_INVALID;
    }

    const bool smem_sort = n_max <= kSmemSortMaxN;
    const size_t pts = static_cast<size_t>(b) * ws.stride;
    const size_t nbt = static_cast<size_t>(b) * ws.nbmax;
    // one stream-ordered allocation, carved
    size_t off = 0;
    auto take = [&off](size_t bytes) { const size_t o = off; off = (off + bytes + 255) & ~static_cast<size_t>(255); return o; };
    const size_t o_pa = take(pts / 2 * sizeof(float4)), o_pb = take(pts / 2 * sizeof(float4)), o_k = take(pts / 2 * sizeof(int2)),
                 o_ka = take(smem_sort ? 0 : pts * sizeof(uint2)), o_kb = take(smem_sort ? 0 : pts * sizeof(uint2)),
                 o_lo = take(nbt * sizeof(float4)), o_hi = take(nbt * sizeof(float4)), o_bx = take(nbt * sizeof(float4));
    keep_async_pool();
    unsigned char* base = nullptr;
    cudaError_t e = cudaMallocAsync(reinterpret_cast<void**>(&base), off, stream);
    if (e != cudaSuccess) { set_error("furthestsampling: workspace of %zu bytes: %s", off, cudaGetErrorString(e)); (void)cudaGetLastError(); return TGN_ERR_CUDA; }
    ws.pa = reinterpret_cast<float4*>(base + o_pa);
    ws.pb = reinterpret_cast<float4*>(base + o_pb);
    ws.keys = reinterpret_cast<int2*>(base + o_k);
    ws.key_a = reinterpret_cast<uint2*>(base + o_ka);
    ws.key_b = reinterpret_cast<uint2*>(base + o_kb);
    ws.box_lo = reinterpret_cast<float4*>(base + o_lo);
    ws.box_hi = reinterpret_cast<float4*>(base + o_hi);
    ws.bxyz = reinterpret_cast<float4*>(base + o_bx);

    if (n_max <= kSmemSortMaxN) {
        const int spad = (n_max + 31) & ~31;
        const size_t sort_smem = 2 * sizeof(unsigned) * static_cast<size_t>(spad);
        const int rc_attr = ensure_dynamic_smem(reinterpret_cast<const void*>(fps_bucket_sort_kernel<true>), 2 * sizeof(unsigned) * kSmemSortMaxN);
        if (rc_attr != TGN_OK) return rc_attr;
        fps_bucket_sort_kernel<true><<<b, kT, sort_smem, stream>>>(xyz, offset, tmp, ws, bs_log2, spad);
    } else {
        fps_bucket_sort_kernel<false><<<b, kT, 0, stream>>>(xyz, offset, tmp, ws, bs_log2, 0);
    }
    int rc = check_launch("fps_bucket_sort_kernel");
    if (rc == TGN_OK) {
        // every (kernel, warps) pair below was admitted above
        if (v3) {
            const int bpl = (ws.nbmax + warps * 32 - 1) / (warps * 32);          // buckets per lane
            rc = -1;
            if (warps == 32 && bpl <= 1) rc = launch_main3<1024, 1>(b, xyz, offset, new_offset, tmp, idx, ws, bs_log2, stream);
            else if (warps == 16 && bpl <= 1) rc = launch_main3<512, 1>(b, xyz, offset, new_offset, tmp, idx, ws, bs_log2, stream);
            else if (warps == 16 && bpl <= 2) rc = launch_main3<512, 2>(b, xyz, offset, new_offset, tmp, idx, ws, bs_log2, stream);
            else if (warps == 16 && bpl <= 4) rc = launch_main3<512, 4>(b, xyz, offset, new_offset, tmp, idx, ws, bs_log2, stream);     // <= 131 072 points
            else if (warps == 16 && bpl <= 6) rc = launch_main3<512, 6>(b, xyz, offset, new_offset, tmp, idx, ws, bs_log2, stream);     // <= 196 608
            else if (warps == 16 && bpl <= 8) rc = launch_main3<512, 8>(b, xyz, offset, new_offset, tmp, idx, ws, bs_log2, stream);     // <= kMaxBuckets
            else if (warps == 8 && bpl <= 1) rc = launch_main3<256, 1>(b, xyz, offset, new_offset, tmp, idx, ws, bs_log2, stream);
            else if (warps == 8 && bpl <= 2) rc = launch_main3<256, 2>(b, xyz, offset, new_offset, tmp, idx, ws, bs_log2, stream);
            else if (warps == 8 && bpl <= 4) rc = launch_main3<256, 4>(b, xyz, offset, new_offset, tmp, idx, ws, bs_log2, stream);
            else if (warps == 4 && bpl <= 2) rc = launch_main3<128, 2>(b, xyz, offset, new_offset, tmp, idx, ws, bs_log2, stream);
            else if (warps == 4 && bpl <= 3) rc = launch_main3<128, 3>(b, xyz, offset, new_offset, tmp, idx, ws, bs_log2, stream);
            else if (warps == 4 && bpl <= 4) rc = launch_main3<128, 4>(b, xyz, offset, new_offset, tmp, idx, ws, bs_log2, stream);
            // more buckets per lane than the registers of this CTA width hold: the same single-barrier schedule with the
            // tables in shared memory (fps_bucket_kernel2, bitwise the same samples)
            if (rc == -1) {
                switch (warps) {
                    case 32: rc = launch_main2<1024>(b, smem, xyz, offset, new_offset, tmp, idx, ws, bs_log2, stream); break;
                    case 16: rc = launch_main2<512>(b, smem, xyz, offset, new_offset, tmp, idx, ws, bs_log2, stream); break;
                    case 8: rc = launch_main2<256>(b, smem, xyz, offset, new_offset, tmp, idx, ws, bs_log2, stream); break;
                    case 4: rc = launch_main2<128>(b, smem, xyz, offset, new_offset, tmp, idx, ws, bs_log2, stream); break;
                    default: set_error("furthestsampling: bucket kernel v3 has no shape of %d warps x %d buckets per lane", warps, bpl); rc = TGN_ERR_INVALID;
                }
            }
        } else if (v2) {
            switch (warps) {
                case 16: rc = launch_main2<512>(b, smem, xyz, offset, new_offset, tmp, idx, ws, bs_log2, stream); break;
                case 8: rc = launch_main2<256>(b, smem, xyz, offset, new_offset, tmp, idx, ws, bs_log2, stream); break;
                case 4: rc = launch_main2<128>(b, smem, xyz, offset, new_offset, tmp, idx, ws, bs_log2, stream); break;
                case 2: rc = launch_main2<64>(b, smem, xyz, offset, new_offset, tmp, idx, ws, bs_log2, stream); break;
                case 32: rc = launch_main2<1024>(b, smem, xyz, offset, new_offset, tmp, idx, ws, bs_log2, stream); break;
                default: set_error("furthestsampling: bucket kernel v2 has no shape of %d warps per cloud", warps); rc = TGN_ERR_INVALID;
            }
        } else
        switch (warps) {
            case 16: rc = launch_main<512>(b, smem, xyz, offset, new_offset, tmp, idx, ws, bs_log2, stream); break;
            case 8: rc = launch_main<256>(b, smem, xyz, offset, new_offset, tmp, idx, ws, bs_log2, stream); break;
            case 4: rc = launch_main<128>(b, smem, xyz, offset, new_offset, tmp, idx, ws, bs_log2, stream); break;
            case 2: rc = launch_main<64>(b, smem, xyz, offset, new_offset, tmp, idx, ws, bs_log2, stream); break;
            case 1: rc = launch_main<32>(b, smem, xyz, offset, new_offset, tmp, idx, ws, bs_log2, stream); break;
            default: set_error("furthestsampling: bucket kernel has no shape of %d warps per cloud", warps); rc = TGN_ERR_INVALID;
        }
    }
    (void)cudaFreeAsync(base, stream);
    return rc;
}

}  // namespace tgn
