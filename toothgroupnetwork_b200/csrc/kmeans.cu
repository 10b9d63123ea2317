// kmeans.cu -- scikit-learn 1.9's KMeans(init="k-means++", n_init=1, algorithm="lloyd").fit on float32 (n,3) points, one whole
// fit per CTA in one launch (DESIGN §3.13).  Every rounding is the one single-threaded scikit-learn makes on x86-64 with its
// bundled OpenBLAS (SkylakeX kernels): explicit __f*_rn / __d*_rn / __fmaf_rn, so nvcc contracts nothing.
//
// Seeding (_kmeans_plusplus):  squared distances through float64 ((-2 * dot) + |c|^2) + |x|^2 rounded to float32 and clamped
// at 0; potentials as cblas_sdot / cblas_sgemv order their sums; candidates by searchsorted into the float32 running sum.
// Lloyd (_kmeans_single_lloyd):  labels by float32 ||c||^2 + (-2) * fma-chain(x . c), first minimum; each cluster's members
// compacted in index order, so that its sum is the same float32 chain scikit-learn adds; averages by the float32 reciprocal of
// the double 1 / count; strict convergence first, then sum(shift^2) <= tol (numpy's pairwise order).  A cluster that empties
// is relocated by scikit-learn's argpartition step, which is not restated: the fit stops and sets its relocation flag.
#include "common.cuh"
#include "tgn_b200.h"

#include <algorithm>
#include <cmath>

namespace tgn {
namespace {

constexpr int kKMax = 64;          // k <= 64, so n_local_trials = 2 + int(log k) <= 6
constexpr int kTMax = 6;
constexpr int kThreads = 512;
constexpr int kWarps = kThreads / 32;
constexpr int kNb = 4096;          // sgemv_t's row block (NBMAX)
constexpr int kSmemFloats = 48 * 1024;   // closest distances copied to shared memory for the running sum when n <= this

struct KmArgs {
    int k, T, max_iter, smem_floats;
    const int* offsets;            // (B+1) point offsets of the fits
    const float* X;                // (N,3) centred points
    const int* first;              // (B) first seed
    const double* uniforms;        // (B, k-1, T)
    const float* tol;              // (B)
    float* rows;                   // (T+1) float32 rows per point: the closest distances and the candidates' rows
    int* order;                    // per point: members of each cluster, in index order
    float* lanes;                  // per fit: (T, blocks, 8) sgemv lane sums
    int* labels;
    long long* init;
    float* centers;
    int* n_iter;
    float* inertia;
    int* relocated;
};

__device__ __forceinline__ double norm64(const float* p)
{
    const double a = p[0], b = p[1], c = p[2];
    return __dadd_rn(__dadd_rn(__dmul_rn(a, a), __dmul_rn(b, b)), __dmul_rn(c, c));
}

// _euclidean_distances_upcast for one (centre, point) pair
__device__ __forceinline__ float sqdist_up(const float* c, double cc, const float* p)
{
    const double dot = __dadd_rn(__dadd_rn(__dmul_rn((double)c[0], (double)p[0]), __dmul_rn((double)c[1], (double)p[1])),
                                 __dmul_rn((double)c[2], (double)p[2]));
    const float d = __double2float_rn(__dadd_rn(__dadd_rn(__dmul_rn(-2.0, dot), cc), norm64(p)));
    return d > 0.f ? d : 0.f;          // np.maximum(d, 0); a sum of the form ((-2 dot) + |c|^2) + |x|^2 never rounds to -0
}

// cblas_sdot(x, ones) of sdot_k_SKYLAKEX: 64 lanes over the 64-blocks, folded to 32, one more 32-block, then the fold; the tail
// past the last 32-block in float64.  Called by all threads; thread 0 returns the result.
__device__ float sdot_ones(const float* x, int n, float* red)
{
    const int n1 = n & ~31, n64 = n1 & ~63;
    const int t = threadIdx.x;
    if (t < 64) {
        float acc = 0.f;
        for (int i = t; i < n64; i += 64) acc = __fadd_rn(acc, x[i]);
        red[t] = acc;
    }
    __syncthreads();
    float out = 0.f;
    if (t == 0) {
        float kpart = 0.f;
        if (n1) {
            float a[4][8];
#pragma unroll
            for (int q = 0; q < 4; ++q)
#pragma unroll
                for (int l = 0; l < 8; ++l) {
                    a[q][l] = __fadd_rn(red[q * 16 + l], red[q * 16 + 8 + l]);
                    if (n1 > n64) a[q][l] = __fadd_rn(a[q][l], x[n64 + q * 8 + l]);
                }
            float s[8], h[4];
#pragma unroll
            for (int l = 0; l < 8; ++l) s[l] = __fadd_rn(__fadd_rn(__fadd_rn(a[0][l], a[1][l]), a[2][l]), a[3][l]);
#pragma unroll
            for (int l = 0; l < 4; ++l) h[l] = __fadd_rn(s[l], s[l + 4]);
            kpart = __fadd_rn(__fadd_rn(h[0], h[1]), __fadd_rn(h[2], h[3]));
        }
        double tail = 0.0;
        for (int i = n1; i < n; ++i) tail = __dadd_rn(tail, (double)x[i]);
        out = __double2float_rn(__dadd_rn(tail, (double)kpart));
    }
    __syncthreads();
    return out;
}

// cblas_sgemv(rows (T,n), ones) of sgemv_t_SKYLAKEX for T >= 2: pot[t] for every t, in shared memory.  Row blocks of 4096 (the
// last cut to a multiple of 4) whose sums are added to y in float32, the n % 4 last rows added as ((a0 + a1) + a2).  Within a
// block, the columns of the 4x4 and 4x1 kernels run 8 lanes (the 4x1 kernel's two 4-lane accumulators fold the same way) and the
// 4x2 kernel's 4 lanes; a lane's chain starts with row lane of an n % 8 == 4 block, then takes every 8th (4th) row.
__device__ void sgemv_ones(const float* rows, int n, int T, float* lanes, float* pot)
{
    const int m3 = n & 3;
    const int body = n - m3;
    const int nblocks = (body + kNb - 1) / kNb;
    const int items = T * nblocks * 8;
    for (int it = threadIdx.x; it < items; it += blockDim.x) {
        const int l = it & 7, b = (it >> 3) % nblocks, t = (it >> 3) / nblocks;
        const int W = (t < (T & ~3) || t >= (T & ~1)) ? 8 : 4;
        float acc = 0.f;
        if (l < W) {
            const float* r = rows + (size_t)t * n + (size_t)b * kNb;
            const int NB = min(kNb, body - b * kNb);
            int i = 0;
            if (NB & 4) {
                if (l < 4) acc = __fadd_rn(acc, r[l]);
                i = 4;
            }
#pragma unroll 8
            for (int j = i + l; j < NB; j += W) acc = __fadd_rn(acc, r[j]);
        }
        lanes[it] = acc;
    }
    __syncthreads();
    if (threadIdx.x < T) {
        const int t = threadIdx.x;
        const int W = (t < (T & ~3) || t >= (T & ~1)) ? 8 : 4;
        float y = 0.f;
        for (int b = 0; b < nblocks; ++b) {
            const float* a = lanes + (t * nblocks + b) * 8;
            float h[4];
#pragma unroll
            for (int l = 0; l < 4; ++l) h[l] = W == 8 ? __fadd_rn(a[l], a[l + 4]) : a[l];
            y = __fadd_rn(y, __fadd_rn(__fadd_rn(h[0], h[1]), __fadd_rn(h[2], h[3])));
        }
        if (m3) {
            const float* r = rows + (size_t)t * n + body;
            float s = r[0];
            for (int q = 1; q < m3; ++q) s = __fadd_rn(s, r[q]);
            y = __fadd_rn(y, s);
        }
        pot[t] = y;
    }
    __syncthreads();
}

// searchsorted(cumsum(x), v[t]) for the T values, clipped to n - 1 (thread 0 alone): the first index whose float32 running sum is
// >= v[t] in float64.  The sum is one float32 chain.  Every summand is >= 0, so the sum never decreases: the walk adds a whole
// 8-block, compares only the block's last sum with the smallest open value, and rescans a block only when that sum reaches it.
// (double)cum >= v is cum >= v rounded up to float32, so the hot loop stays in float32.
__device__ __forceinline__ void search_running_sum(const float* x, int n, int T, const double* v, int* cand)
{
    int left = T;
    auto close = [&](float sum, int at) {                  // resolve every open value the running sum at index `at` reaches
        for (int t = 0; t < T; ++t)
            if (cand[t] < 0 && sum >= __double2float_ru(v[t])) { cand[t] = at; --left; }
    };
    auto open_min = [&]() {
        float m = INFINITY;
        for (int t = 0; t < T; ++t) if (cand[t] < 0) m = fminf(m, __double2float_ru(v[t]));
        return m;
    };
    float vmin = open_min();
    float cum = 0.f;
    const int n8 = n & ~7;
    float cur[8], nxt[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) cur[q] = q < n8 ? x[q] : 0.f;
    int i = 0;
    for (; i < n8 && left; i += 8) {
#pragma unroll
        for (int q = 0; q < 8; ++q) nxt[q] = i + 8 + q < n8 ? x[i + 8 + q] : 0.f;
        float s = cum;
#pragma unroll
        for (int q = 0; q < 8; ++q) s = __fadd_rn(s, cur[q]);
        if (s >= vmin) {                                    // rare: rescan this block element by element
            float r = cum;
            for (int q = 0; q < 8; ++q) {
                r = __fadd_rn(r, x[i + q]);
                close(r, i + q);
            }
            vmin = open_min();
        }
        cum = s;
#pragma unroll
        for (int q = 0; q < 8; ++q) cur[q] = nxt[q];
    }
    for (; i < n && left; ++i) {
        cum = __fadd_rn(cum, x[i]);
        close(cum, i);
    }
    for (int t = 0; t < T; ++t) if (cand[t] < 0) cand[t] = n - 1;
}

// labels by _update_chunk_dense; returns (to every thread) whether any label changed.  Counts per cluster into cnt.
__device__ bool assign(const float* X, int n, int k, const float* cen, const float* cn, int* labels, int* cnt)
{
    bool changed = false;
    for (int i0 = 0; i0 < n; i0 += blockDim.x) {                     // whole warps in every round, for match_any below
        const int i = i0 + threadIdx.x;
        int lab = -1;
        if (i < n) {
            const float x0 = X[3 * i], x1 = X[3 * i + 1], x2 = X[3 * i + 2];
            float best = 0.f;
            for (int j = 0; j < k; ++j) {
                float acc = __fmul_rn(x0, cen[3 * j]);
                acc = __fmaf_rn(x1, cen[3 * j + 1], acc);
                acc = __fmaf_rn(x2, cen[3 * j + 2], acc);
                const float d = __fadd_rn(cn[j], __fmul_rn(-2.f, acc));
                if (j == 0 || d < best) { best = d; lab = j; }
            }
            changed |= labels[i] != lab;
            labels[i] = lab;
        }
        if (cnt) {                                                     // one shared-memory atomic per label per warp
            const unsigned same = __match_any_sync(0xffffffffu, lab);
            if (lab >= 0 && (same & ((1u << (threadIdx.x & 31)) - 1u)) == 0) atomicAdd(&cnt[lab], __popc(same));
        }
    }
    return __syncthreads_or(changed) != 0;
}

__device__ void centre_norms(const float* cen, int k, float* cn)
{
    for (int j = threadIdx.x; j < k; j += blockDim.x) {
        const float* c = cen + 3 * j;
        cn[j] = __fadd_rn(__fadd_rn(__fmul_rn(c[0], c[0]), __fmul_rn(c[1], c[1])), __fmul_rn(c[2], c[2]));
    }
    __syncthreads();
}

__global__ void __launch_bounds__(kThreads, 1) kmeans_kernel(KmArgs a)
{
    __shared__ float cen[kKMax * 3], nw[kKMax * 3], cn[kKMax], shift[kKMax];
    __shared__ int cnt[kKMax], base[kKMax], wcnt[kWarps][kKMax];
    __shared__ float red[64], pot[kTMax];
    __shared__ int cand[kTMax];
    __shared__ int s_best, s_stop;
    __shared__ float s_pot;
    __shared__ double s_v[kTMax], s_cc[kTMax];
    extern __shared__ float dyn[];

    const int f = blockIdx.x;
    const int o = a.offsets[f], n = a.offsets[f + 1] - o;
    const int k = a.k, T = a.T, tid = threadIdx.x;
    const float* X = a.X + 3 * (size_t)o;
    float* rows = a.rows + (size_t)(T + 1) * o;                     // row r of this fit at rows + r * n
    int* order = a.order + o;
    int* labels = a.labels + o;
    float* lanes = a.lanes + (size_t)(o / kNb + f) * kTMax * 8;
    const double* u = a.uniforms + (size_t)f * (k - 1) * T;

    // ---- k-means++ seeding: the closest distances live in row T, candidate t's row in row t
    float* closest = rows + (size_t)T * n;
    const int first = a.first[f];
    if (tid == 0) a.init[(size_t)f * k] = first;
    {
        const double cc = norm64(X + 3 * first);
        for (int i = tid; i < n; i += blockDim.x) closest[i] = sqdist_up(X + 3 * first, cc, X + 3 * i);
    }
    __syncthreads();
    const float p0 = sdot_ones(closest, n, red);
    if (tid == 0) s_pot = p0;
    __syncthreads();
    const bool in_smem = n <= a.smem_floats;                         // the running sum reads shared memory when the row fits
    if (in_smem)
        for (int i = tid; i < n; i += blockDim.x) dyn[i] = closest[i];
    __syncthreads();
    for (int c = 1; c < k; ++c) {
        if (tid == 0) {
            for (int t = 0; t < T; ++t) { s_v[t] = __dmul_rn(u[(size_t)(c - 1) * T + t], (double)s_pot); cand[t] = -1; }
            if (in_smem) search_running_sum(dyn, n, T, s_v, cand);
            else search_running_sum(closest, n, T, s_v, cand);
        }
        __syncthreads();
        if (tid < T) s_cc[tid] = norm64(X + 3 * cand[tid]);
        __syncthreads();
        for (int i = tid; i < n; i += blockDim.x) {                    // np.minimum(closest, d(candidate, x)), each point read once
            const float* p = X + 3 * i;
            const double xx = norm64(p), p0 = p[0], p1 = p[1], p2 = p[2];
            const float cl = closest[i];
            for (int t = 0; t < T; ++t) {
                const float* cp = X + 3 * cand[t];
                const double dot = __dadd_rn(__dadd_rn(__dmul_rn((double)cp[0], p0), __dmul_rn((double)cp[1], p1)), __dmul_rn((double)cp[2], p2));
                float d = __double2float_rn(__dadd_rn(__dadd_rn(__dmul_rn(-2.0, dot), s_cc[t]), xx));
                d = d > 0.f ? d : 0.f;
                rows[(size_t)t * n + i] = fminf(cl, d);
            }
        }
        __syncthreads();
        sgemv_ones(rows, n, T, lanes, pot);
        if (tid == 0) {
            int best = 0;
            for (int t = 1; t < T; ++t) if (pot[t] < pot[best]) best = t;
            s_pot = pot[best];
            s_best = best;
            a.init[(size_t)f * k + c] = cand[best];
        }
        __syncthreads();
        const float* br = rows + (size_t)s_best * n;
        for (int i = tid; i < n; i += blockDim.x) {
            const float v = br[i];
            closest[i] = v;
            if (in_smem) dyn[i] = v;
        }
        __syncthreads();
    }
    for (int j = tid; j < k; j += blockDim.x) {
        const int id = (int)a.init[(size_t)f * k + j];
        cen[3 * j] = X[3 * id]; cen[3 * j + 1] = X[3 * id + 1]; cen[3 * j + 2] = X[3 * id + 2];
    }
    for (int i = tid; i < n; i += blockDim.x) labels[i] = -1;
    __syncthreads();

    // ---- Lloyd
    const float tol = a.tol[f];
    bool strict = false;
    int relocated = 0, it = 0;
    for (it = 0; it < a.max_iter; ++it) {
        centre_norms(cen, k, cn);
        for (int j = tid; j < k; j += blockDim.x) { cnt[j] = 0; base[j] = 0; }
        __syncthreads();
        const bool changed = assign(X, n, k, cen, cn, labels, cnt);
        if (tid == 0) {
            s_stop = 0;
            for (int j = 0; j < k; ++j) if (cnt[j] == 0) s_stop = 1;
            int s = 0;
            for (int j = 0; j < k; ++j) { base[j] = s; s += cnt[j]; }
        }
        __syncthreads();
        if (s_stop) { relocated = 1; break; }
        // stable compaction by label: tiles of blockDim points, ranks within a warp by match_any, warps in order
        const int warp = tid >> 5, lane = tid & 31;
        for (int t0 = 0; t0 < n; t0 += blockDim.x) {
            const int i = t0 + tid;
            for (int j = lane; j < k; j += 32) wcnt[warp][j] = 0;
            __syncwarp();
            const int lab = i < n ? labels[i] : kKMax + 1;
            const unsigned same = __match_any_sync(0xffffffffu, lab);
            const int rank = __popc(same & ((1u << lane) - 1u));
            if (i < n && rank == 0) wcnt[warp][lab] = __popc(same);
            __syncthreads();
            for (int j = tid; j < k; j += blockDim.x) {            // exclusive prefix over the warps, per label
                int s = base[j];
                for (int w = 0; w < kWarps; ++w) { const int c = wcnt[w][j]; wcnt[w][j] = s; s += c; }
                base[j] = s;
            }
            __syncthreads();
            if (i < n) order[wcnt[warp][lab] + rank] = i;
            __syncthreads();
        }
        // cluster sums: one float32 chain per (cluster, feature) over the members in index order
        for (int j = tid; j < k; j += blockDim.x) {
            const int e = base[j], m0 = e - cnt[j];
            float s0 = 0.f, s1 = 0.f, s2 = 0.f;
            for (int m = m0; m < e; m += 8) {                          // loads batched ahead of the three chains
                float v0[8], v1[8], v2[8];
#pragma unroll
                for (int q = 0; q < 8; ++q) {
                    const int id = m + q < e ? order[m + q] : -1;
                    v0[q] = id >= 0 ? X[3 * id] : 0.f;
                    v1[q] = id >= 0 ? X[3 * id + 1] : 0.f;
                    v2[q] = id >= 0 ? X[3 * id + 2] : 0.f;
                }
#pragma unroll
                for (int q = 0; q < 8; ++q) {
                    if (m + q < e) { s0 = __fadd_rn(s0, v0[q]); s1 = __fadd_rn(s1, v1[q]); s2 = __fadd_rn(s2, v2[q]); }
                }
            }
            const float s[3] = {s0, s1, s2};
            const float alpha = __double2float_rn(__ddiv_rn(1.0, (double)(float)cnt[j]));
            float ss = 0.f;
#pragma unroll
            for (int d = 0; d < 3; ++d) {
                nw[3 * j + d] = __fmul_rn(__fadd_rn(0.f, s[d]), alpha);
                const float df = __fsub_rn(nw[3 * j + d], cen[3 * j + d]);
                ss = __fadd_rn(ss, __fmul_rn(df, df));
            }
            shift[j] = __fsqrt_rn(ss);
        }
        __syncthreads();
        for (int j = tid; j < 3 * k; j += blockDim.x) cen[j] = nw[j];
        if (tid == 0) {
            s_stop = 0;
            if (!changed) s_stop = 2;
            else {
                // numpy's pairwise float32 sum of shift**2
                float tot;
                if (k < 8) {
                    tot = 0.f;
                    for (int j = 0; j < k; ++j) tot = __fadd_rn(tot, __fmul_rn(shift[j], shift[j]));
                } else {
                    float r[8];
#pragma unroll
                    for (int l = 0; l < 8; ++l) r[l] = __fmul_rn(shift[l], shift[l]);
                    const int m8 = k - k % 8;
                    for (int j = 8; j < m8; j += 8)
#pragma unroll
                        for (int l = 0; l < 8; ++l) r[l] = __fadd_rn(r[l], __fmul_rn(shift[j + l], shift[j + l]));
                    tot = __fadd_rn(__fadd_rn(__fadd_rn(r[0], r[1]), __fadd_rn(r[2], r[3])), __fadd_rn(__fadd_rn(r[4], r[5]), __fadd_rn(r[6], r[7])));
                    for (int j = m8; j < k; ++j) tot = __fadd_rn(tot, __fmul_rn(shift[j], shift[j]));
                }
                if (tot <= tol) s_stop = 1;
            }
        }
        __syncthreads();
        if (s_stop) { strict = s_stop == 2; break; }
    }
    if (it == a.max_iter) it = a.max_iter - 1;
    if (!strict && !relocated) {
        centre_norms(cen, k, cn);
        assign(X, n, k, cen, cn, labels, nullptr);
    }
    // inertia: float32 chain over the points in index order
    float* sq = rows;
    for (int i = tid; i < n; i += blockDim.x) {
        const float* x = X + 3 * i;
        const float* c = cen + 3 * labels[i];
        const float d0 = __fsub_rn(x[0], c[0]), d1 = __fsub_rn(x[1], c[1]), d2 = __fsub_rn(x[2], c[2]);
        sq[i] = __fadd_rn(__fadd_rn(__fadd_rn(0.f, __fmul_rn(d0, d0)), __fmul_rn(d1, d1)), __fmul_rn(d2, d2));
    }
    __syncthreads();
    if (tid == 0) {
        float in = 0.f;
        for (int i = 0; i < n; i += 8) {
            float x[8];
#pragma unroll
            for (int q = 0; q < 8; ++q) x[q] = i + q < n ? sq[i + q] : 0.f;
#pragma unroll
            for (int q = 0; q < 8; ++q) if (i + q < n) in = __fadd_rn(in, x[q]);
        }
        a.inertia[f] = in;
        a.n_iter[f] = it + 1;
        a.relocated[f] = relocated;
    }
    for (int j = tid; j < 3 * k; j += blockDim.x) a.centers[(size_t)f * 3 * k + j] = cen[j];
}

size_t km_layout(long long n_total, int B, void* base, float** rows, int** order, float** lanes)
{
    auto up = [](size_t v) { return (v + 255) & ~size_t(255); };
    const size_t r = up(sizeof(float) * (kTMax + 1) * (size_t)n_total);
    const size_t o = up(sizeof(int) * (size_t)n_total);
    const size_t l = up(sizeof(float) * kTMax * 8 * (size_t)(n_total / kNb + B));
    if (base) {
        unsigned char* p = static_cast<unsigned char*>(base);
        *rows = reinterpret_cast<float*>(p);
        *order = reinterpret_cast<int*>(p + r);
        *lanes = reinterpret_cast<float*>(p + r + o);
    }
    return r + o + l;
}

}  // namespace
}  // namespace tgn

extern "C" {

size_t tgn_kmeans_bytes(long long n_total, int B) { return tgn::km_layout(std::max(n_total, 1LL), std::max(B, 1), nullptr, nullptr, nullptr, nullptr); }

int tgn_kmeans(int B, long long n_total, int k, int max_iter, const int* offsets, const float* X, const int* first, const double* uniforms,
               const float* tol, void* workspace, int* labels, long long* init, float* centers, int* n_iter, float* inertia,
               int* relocated, void* stream)
{
    using namespace tgn;
    if (B < 0 || n_total < 0 || k < 1 || k > kKMax || max_iter < 1) {
        set_error("kmeans: bad arguments B=%d k=%d max_iter=%d (1 <= k <= %d)", B, k, max_iter, kKMax);
        return TGN_ERR_INVALID;
    }
    if (B == 0) return TGN_OK;
    if (!offsets || !X || !first || !tol || !workspace || !labels || !init || !centers || !n_iter || !inertia || !relocated || (k > 1 && !uniforms)) {
        set_error("kmeans: null argument");
        return TGN_ERR_INVALID;
    }
    KmArgs a;
    a.k = k;
    a.T = 2 + (int)std::log((double)k);
    a.max_iter = max_iter;
    a.offsets = offsets; a.X = X; a.first = first; a.uniforms = uniforms; a.tol = tol;
    km_layout(n_total, B, workspace, &a.rows, &a.order, &a.lanes);
    a.labels = labels; a.init = init; a.centers = centers; a.n_iter = n_iter; a.inertia = inertia; a.relocated = relocated;
    a.smem_floats = (int)std::min<long long>(n_total, kSmemFloats);
    const size_t smem = sizeof(float) * (size_t)a.smem_floats;
    // opt in to the largest size once: without it, static + dynamic shared memory is capped at 48 KB
    if (ensure_dynamic_smem(reinterpret_cast<const void*>(kmeans_kernel), sizeof(float) * kSmemFloats) != TGN_OK) return TGN_ERR_CUDA;
    kmeans_kernel<<<B, kThreads, smem, static_cast<cudaStream_t>(stream)>>>(a);
    return check_launch("kmeans");
}

}  // extern "C"
