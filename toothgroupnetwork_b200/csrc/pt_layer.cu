// pt_layer.cu -- fused forward of blocks.PointTransformerLayer (models/modules/cbl_point_transformer/blocks.py:14-44),
// SURVEY.md 8(f)-3.
//
// The reference builds, per layer, two grouped (n, K, c) tensors with two identical kNN searches, and runs ~30 torch kernels
// over them: three BatchNorms on (n, c, K)-shaped views (cudnn::bn_fw_tr_1C11, the largest
// share of the kernel time of a tgnet_fps step), four small Linears, a softmax over K and the share-planes aggregation.
// Its inference runs those BatchNorms on BATCH statistics (no .eval(), SURVEY 3c), so one fused kernel is not valid; this file
// is the multi-pass form.  For query i and neighbour j (nbr = idx[i, j]) everything is a function of a handful of gathers:
//
//      rel  = p[nbr] - p[i]                                   (queryandgroup, use_xyz: pointops.py:94-99)
//      t    = W_p0 rel + b_p0                        (3)      -> BatchNorm_p statistics          [pass 0]
//      pr   = W_p1 relu(bn_p(t)) + b_p1              (c)
//      w0   = (x_k[nbr] - x_q[i]) + pr               (c)      -> BatchNorm_a statistics          [pass 1]
//      w1   = W_a relu(bn_a(w0)) + b_a               (c/8)    -> BatchNorm_b statistics          [pass 2]
//      w2   = W_b relu(bn_b(w1)) + b_b               (c/8)
//      out[i, ch] = sum_j (x_v[nbr, ch] + pr[ch]) * softmax_j(w2)[j, ch mod c/8]                 [pass 3]
//
// Every pass recomputes the chain up to its stage from the gathers (the arithmetic is tiny: 24 000 x 36 rows x ~250 MACs at
// c = 32) instead of materialising (n, K, c) tensors; statistics are fp64 sums accumulated with two atomics per channel per
// CTA, turned into scale / shift in the next pass's prologue.  With running statistics (eval mode) only pass 3 runs.
// One warp per query; lane l owns channels l, l + 32, ... (CPL = c / 32 of them); the c -> c/8 product is per-lane partial
// sums + a butterfly, so every lane ends up with all c/8 values; logits of the K neighbours wait in shared memory for the
// softmax.  fp32 FMA arithmetic throughout.  Shapes: c in {16, 32, 64, 128, 256, 512}, share_planes = 8, K <= 64.
//
// c = 16 (the boundary network's first level) runs two queries per warp, one per half-warp (W = 16 lanes per query): lane l owns
// channel l & 15 of query 2 w + (l >> 4), the c -> c/8 butterfly stays inside the half (xor 8, 4, 2, 1), and each half has its
// own logits.  One warp per query would leave 16 of 32 lanes idle in an fp32-issue-bound kernel.  The grid-stride loop steps over
// query PAIRS so that both halves run the same trip count: a half without a query (odd n, the end of the stride) computes on a
// clamped index and keeps nothing, because it still has to take part in every full-mask shuffle and __syncwarp.  The CTA-per-query
// schedule (tgn_pt_layer_set_cta_threshold) is for wide channels at deep levels and does not apply to c = 16.
#include <algorithm>

#include "common.cuh"
#include "tgn_b200.h"

namespace tgn {
namespace {

constexpr int kWarps = 8;
constexpr unsigned FULL = 0xffffffffu;

// BatchNorm as (x - mean) * scale + beta with the mean carried as hi + lo floats: folding the mean into a shift
// (x * scale + (beta - mean * scale)) costs |mean| / std ulps on the normalised value -- the 3-channel BatchNorm_p sees
// |mean| / std ~ 50 (a bias in front of centimetre-sized offsets) -- and this form has no such term at all.
struct BnAffine { float mean_hi, mean_lo, scale, beta; };

__device__ __forceinline__ BnAffine scale_shift(int mode, int ch, int cn, const double* stats, double cnt, const float* gamma,
                                                const float* beta, float eps, const float* rmean, const float* rvar)
{
    double mean, var;
    if (mode == 1) {
        mean = stats[ch] / cnt;
        var = fmax(stats[cn + ch] / cnt - mean * mean, 0.0);
    } else {
        mean = static_cast<double>(rmean[ch]);
        var = static_cast<double>(rvar[ch]);
    }
    BnAffine a;
    a.mean_hi = static_cast<float>(mean);
    a.mean_lo = static_cast<float>(mean - static_cast<double>(a.mean_hi));
    a.scale = static_cast<float>(static_cast<double>(gamma ? gamma[ch] : 1.f) / sqrt(var + static_cast<double>(eps)));
    a.beta = beta ? beta[ch] : 0.f;
    return a;
}

__device__ __forceinline__ float bn_relu(float x, const BnAffine& a)
{
    return fmaxf(fmaf((x - a.mean_hi) - a.mean_lo, a.scale, a.beta), 0.f);
}

// CTAQ = false: one warp per query (shallow levels: tens of thousands of queries).
// CTAQ = true : one CTA per query, its warps take the neighbours round-robin and meet in shared memory for the softmax and the
//               output sum (deep levels: a few hundred queries of 128-512 channels, where a single warp walking K neighbours
//               times c/8 x c products is pure latency).
// W = 16: two queries per warp, one per half-warp (c = 16 only).
// SUMS (pass 3 only): also accumulate fp64 Σ / Σ² per channel of `out` into out_stats, for the BatchNorm that follows the layer
// in PointTransformerBlock (bn2).  Each element goes into its fp64 sums directly, as in pass 1, so that a channel whose |mean| is
// far above its std keeps its variance.  The per-lane sums live in shared memory (a row per query slot of a warp, or a slot per
// channel in the CTA schedule), not in registers: at c = 512 pass 3 already holds 255 registers.
template <int CPL, int PASS, bool CTAQ, int W = 32, bool SUMS = false>
__global__ void __launch_bounds__(kWarps * 32) pt_layer_kernel(const tgn_pt_layer_t L, double* out_stats)
{
    static_assert(W == 32 || (W == 16 && CPL == 1 && !CTAQ), "half-warp queries: c = 16, warp schedule only");
    static_assert(!SUMS || PASS == 3, "output sums: pass 3 only");
    constexpr int C = W * CPL, CS = C / 8;                     // channels, channels / share_planes (= 8)
    constexpr int QPW = 32 / W;                                // queries per warp
    extern __shared__ __align__(16) unsigned char dyn[];
    BnAffine* ss_a = reinterpret_cast<BnAffine*>(dyn);         // [C]   BatchNorm_a mean / scale / beta
    BnAffine* ss_b = ss_a + C;                                 // [CS]  BatchNorm_b
    BnAffine* ss_p = ss_b + CS;                                // [4]   BatchNorm_p (3 used)
    float* logits_all = reinterpret_cast<float*>(ss_p + 4);    // [kWarps * QPW][K][CS]; CTAQ: [K][CS] then [kWarps][C] output partials
    __shared__ double red[kWarps][8];

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int sl = lane & (W - 1), half = lane / W;            // lane within the query's lanes, the query's slot in the warp
    const double cnt = static_cast<double>(L.n) * L.K;
    if (PASS >= 1) for (int a = tid; a < 3; a += kWarps * 32)
        ss_p[a] = scale_shift(L.bn_mode[0], a, 3, L.stats_p, cnt, L.p_gamma, L.p_beta, L.p_eps, L.p_rmean, L.p_rvar);
    if (PASS >= 2) for (int ch = tid; ch < C; ch += kWarps * 32)
        ss_a[ch] = scale_shift(L.bn_mode[1], ch, C, L.stats_a, cnt, L.a_gamma, L.a_beta, L.a_eps, L.a_rmean, L.a_rvar);
    if (PASS >= 3) for (int m = tid; m < CS; m += kWarps * 32)
        ss_b[m] = scale_shift(L.bn_mode[2], m, CS, L.stats_b, cnt, L.b_gamma, L.b_beta, L.b_eps, L.b_rmean, L.b_rvar);
    // SUMS: [slots][2][C] doubles after the logits / partials; slots = kWarps * QPW (warp schedule) or 1 (CTA schedule)
    constexpr int kSlots = CTAQ ? 1 : kWarps * QPW;
    double* osum = nullptr;
    if constexpr (SUMS) {
        osum = reinterpret_cast<double*>(logits_all + (CTAQ ? static_cast<size_t>(L.K) * CS + kWarps * C
                                                            : static_cast<size_t>(kWarps) * QPW * L.K * CS));
        for (int e = tid; e < kSlots * 2 * C; e += kWarps * 32) osum[e] = 0.0;
    }
    __syncthreads();
    float* logits = CTAQ ? logits_all : logits_all + static_cast<size_t>(warp * QPW + half) * L.K * CS;
    float* out_part = logits_all + static_cast<size_t>(L.K) * CS;           // CTAQ only
    const int j0 = CTAQ ? warp : 0, jstep = CTAQ ? kWarps : 1;

    // small parameters of linear_p into registers
    float w0m[9], b0v[3];
#pragma unroll
    for (int a = 0; a < 9; ++a) w0m[a] = __ldg(L.p_w0 + a);
#pragma unroll
    for (int a = 0; a < 3; ++a) b0v[a] = __ldg(L.p_b0 + a);
    float w1m[CPL][3], b1v[CPL];
    if (PASS >= 1) {
#pragma unroll
        for (int q = 0; q < CPL; ++q) {
            const int ch = W * q + sl;
#pragma unroll
            for (int a = 0; a < 3; ++a) w1m[q][a] = __ldg(L.p_w1 + 3 * ch + a);
            b1v[q] = __ldg(L.p_b1 + ch);
        }
    }
    double acc1[PASS == 1 ? CPL : 1], acc2[PASS == 1 ? CPL : 1];         // pass 1: per-lane channel sums
    double sp1[3] = {0.0, 0.0, 0.0}, sp2[3] = {0.0, 0.0, 0.0};           // pass 0
    double sb1[PASS == 2 ? (CS + W - 1) / W : 1], sb2[PASS == 2 ? (CS + W - 1) / W : 1];
    if (PASS == 1) {
#pragma unroll
        for (int q = 0; q < CPL; ++q) { acc1[q] = 0.0; acc2[q] = 0.0; }
    }
    if (PASS == 2) {
#pragma unroll
        for (int q = 0; q < (CS + W - 1) / W; ++q) { sb1[q] = 0.0; sb2[q] = 0.0; }
    }

    // the loop runs over warp-uniform first queries i0, so that both halves of a W = 16 warp take the same trip count
    for (int i0 = CTAQ ? blockIdx.x : (blockIdx.x * kWarps + warp) * QPW; i0 < L.n; i0 += CTAQ ? gridDim.x : gridDim.x * kWarps * QPW) {
        const bool valid = W == 32 || i0 + half < L.n;         // false: an idle half-warp, computing on the last query, keeping nothing
        const int i = W == 32 ? i0 : (valid ? i0 + half : L.n - 1);
        const float pix = __ldg(L.p + 3 * static_cast<size_t>(i)), piy = __ldg(L.p + 3 * static_cast<size_t>(i) + 1),
                    piz = __ldg(L.p + 3 * static_cast<size_t>(i) + 2);
        float xq[CPL];
        if (PASS >= 1) {
#pragma unroll
            for (int q = 0; q < CPL; ++q) xq[q] = __ldg(L.xq + static_cast<size_t>(i) * C + W * q + sl);
        }
        float out[PASS == 3 ? CPL : 1];

        for (int phase = 0; phase < (PASS == 3 ? 2 : 1); ++phase) {
            if (PASS == 3 && phase == 1) {
                // softmax over the K neighbours, one column m per lane (strided), in place (nn.Softmax(dim=1), blocks.py:40)
                if (CTAQ) __syncthreads(); else __syncwarp();
                for (int m = CTAQ ? tid : sl; m < CS; m += CTAQ ? kWarps * 32 : W) {
                    float mx = -INFINITY;
                    for (int j = 0; j < L.K; ++j) mx = fmaxf(mx, logits[j * CS + m]);
                    float sum = 0.f;
                    for (int j = 0; j < L.K; ++j) { const float e = expf(logits[j * CS + m] - mx); logits[j * CS + m] = e; sum += e; }
                    for (int j = 0; j < L.K; ++j) logits[j * CS + m] = logits[j * CS + m] / sum;
                }
                if (CTAQ) __syncthreads(); else __syncwarp();
#pragma unroll
                for (int q = 0; q < CPL; ++q) out[q] = 0.f;
            }
            for (int j = j0; j < L.K; j += jstep) {
                const int nbr = __ldg(L.idx + static_cast<size_t>(i) * L.K + j);
                const float rx = __ldg(L.p + 3 * static_cast<size_t>(nbr)) - pix, ry = __ldg(L.p + 3 * static_cast<size_t>(nbr) + 1) - piy,
                            rz = __ldg(L.p + 3 * static_cast<size_t>(nbr) + 2) - piz;
                float t[3];
#pragma unroll
                for (int a = 0; a < 3; ++a) t[a] = fmaf(w0m[3 * a + 2], rz, fmaf(w0m[3 * a + 1], ry, fmaf(w0m[3 * a], rx, b0v[a])));
                if (PASS == 0) {
                    if (sl == 0 && valid) {
#pragma unroll
                        for (int a = 0; a < 3; ++a) { sp1[a] += t[a]; sp2[a] += static_cast<double>(t[a]) * t[a]; }
                    }
                    continue;
                }
                float tn[3];
#pragma unroll
                for (int a = 0; a < 3; ++a) tn[a] = bn_relu(t[a], ss_p[a]);
                float pr[CPL];
#pragma unroll
                for (int q = 0; q < CPL; ++q) pr[q] = fmaf(w1m[q][2], tn[2], fmaf(w1m[q][1], tn[1], fmaf(w1m[q][0], tn[0], b1v[q])));
                if (PASS == 3 && phase == 1) {
#pragma unroll
                    for (int q = 0; q < CPL; ++q) {
                        const int ch = W * q + sl;
                        const float v = __ldg(L.xv + static_cast<size_t>(nbr) * C + ch) + pr[q];
                        out[q] = fmaf(v, logits[j * CS + (ch % CS)], out[q]);
                    }
                    continue;
                }
                float w0[CPL];
#pragma unroll
                for (int q = 0; q < CPL; ++q) w0[q] = (__ldg(L.xk + static_cast<size_t>(nbr) * C + W * q + sl) - xq[q]) + pr[q];
                if (PASS == 1) {
                    // fp64 per element, as passes 0 and 2: fp32 partial sums of w0^2 lose the variance of a channel whose |mean| >> std
                    if (valid) {
#pragma unroll
                        for (int q = 0; q < CPL; ++q) { acc1[q] += w0[q]; acc2[q] = fma(static_cast<double>(w0[q]), static_cast<double>(w0[q]), acc2[q]); }
                    }
                    continue;
                }
                // c -> c/8: per-lane partial sums over this lane's channels, butterfly, every lane holds all CS values
                float u[CPL];
#pragma unroll
                for (int q = 0; q < CPL; ++q) u[q] = bn_relu(w0[q], ss_a[W * q + sl]);
                float w1[CS];
#pragma unroll
                for (int m = 0; m < CS; ++m) {
                    float part = 0.f;
#pragma unroll
                    for (int q = 0; q < CPL; ++q) part = fmaf(__ldg(L.a_w + static_cast<size_t>(m) * C + W * q + sl), u[q], part);
#pragma unroll
                    for (int o = W / 2; o; o >>= 1) part += __shfl_xor_sync(FULL, part, o);
                    w1[m] = part + __ldg(L.a_b + m);
                }
                if (PASS == 2) {
#pragma unroll
                    for (int m = 0; m < CS; ++m)
                        if (sl == (m & (W - 1)) && valid) { sb1[m / W] += w1[m]; sb2[m / W] += static_cast<double>(w1[m]) * w1[m]; }
                    continue;
                }
                // PASS 3, phase 0: second small product, logits to shared memory
                float v1[CS];
#pragma unroll
                for (int m = 0; m < CS; ++m) v1[m] = bn_relu(w1[m], ss_b[m]);
                for (int mo = sl; mo < CS; mo += W) {
                    float s = __ldg(L.b_b + mo);
#pragma unroll
                    for (int m = 0; m < CS; ++m) s = fmaf(__ldg(L.b_w + static_cast<size_t>(mo) * CS + m), v1[m], s);
                    logits[j * CS + mo] = s;
                }
            }
        }
        if (PASS == 3 && !CTAQ) {
            if (valid) {
#pragma unroll
                for (int q = 0; q < CPL; ++q) L.out[static_cast<size_t>(i) * C + W * q + sl] = out[q];
                if constexpr (SUMS) {
                    double* os = osum + static_cast<size_t>(warp * QPW + half) * 2 * C;
#pragma unroll
                    for (int q = 0; q < CPL; ++q) {
                        const double v = out[q];
                        os[W * q + sl] += v;
                        os[C + W * q + sl] = fma(v, v, os[C + W * q + sl]);
                    }
                }
            }
            __syncwarp();                                          // the next query's logits overwrite the weights read above
        }
        if (PASS == 3 && CTAQ) {
#pragma unroll
            for (int q = 0; q < CPL; ++q) out_part[warp * C + 32 * q + lane] = out[q];
            __syncthreads();
            for (int ch = tid; ch < C; ch += kWarps * 32) {
                float sum = 0.f;
#pragma unroll
                for (int w = 0; w < kWarps; ++w) sum += out_part[w * C + ch];
                L.out[static_cast<size_t>(i) * C + ch] = sum;
                if constexpr (SUMS) {                                  // channel ch belongs to this thread for every query
                    const double v = sum;
                    osum[ch] += v;
                    osum[C + ch] = fma(v, v, osum[C + ch]);
                }
            }
            __syncthreads();                                       // logits / partials are reused by the next query
        }
    }
    if (PASS == 1 || PASS == 2) __syncthreads();                   // the statistics below reuse the logits area
    if constexpr (W == 16) {
        // lanes l and l + 16 hold sums of the same channels (of two queries): fold the upper half into the lower before the CTA sum
#pragma unroll
        for (int a = 0; a < 3; ++a) { sp1[a] += __shfl_xor_sync(FULL, sp1[a], 16); sp2[a] += __shfl_xor_sync(FULL, sp2[a], 16); }
        if (PASS == 1) {
#pragma unroll
            for (int q = 0; q < CPL; ++q) { acc1[q] += __shfl_xor_sync(FULL, acc1[q], 16); acc2[q] += __shfl_xor_sync(FULL, acc2[q], 16); }
        }
        if (PASS == 2) {
#pragma unroll
            for (int q = 0; q < (CS + W - 1) / W; ++q) { sb1[q] += __shfl_xor_sync(FULL, sb1[q], 16); sb2[q] += __shfl_xor_sync(FULL, sb2[q], 16); }
        }
    }

    // ---- statistics: CTA reduction, two fp64 atomics per channel per CTA --------------------------------------------------
    if (PASS == 0) {
        if (lane == 0) {
#pragma unroll
            for (int a = 0; a < 3; ++a) { red[warp][a] = sp1[a]; red[warp][3 + a] = sp2[a]; }
        }
        __syncthreads();
        if (tid < 6) {
            double s = 0.0;
            for (int w = 0; w < kWarps; ++w) s += red[w][tid];
            atomicAdd(L.stats_p + tid, s);
        }
    }
    if (PASS == 1) {
        double* sh = reinterpret_cast<double*>(logits_all);      // [kWarps][2][C] doubles (the logits area is idle in this pass)
#pragma unroll
        for (int q = 0; q < CPL; ++q) {
            if (lane < W) {
                sh[(warp * 2) * C + W * q + lane] = acc1[q];
                sh[(warp * 2 + 1) * C + W * q + lane] = acc2[q];
            }
        }
        __syncthreads();
        for (int e = tid; e < 2 * C; e += kWarps * 32) {
            const int which = e / C, ch = e - which * C;
            double s = 0.0;
            for (int w = 0; w < kWarps; ++w) s += sh[(w * 2 + which) * C + ch];
            atomicAdd(L.stats_a + which * C + ch, s);
        }
    }
    if (PASS == 2) {
        double* sh = reinterpret_cast<double*>(logits_all);      // [kWarps][2][CS]
#pragma unroll
        for (int m = 0; m < CS; ++m)
            if (lane == (m & (W - 1))) { sh[(warp * 2) * CS + m] = sb1[m / W]; sh[(warp * 2 + 1) * CS + m] = sb2[m / W]; }
        __syncthreads();
        for (int e = tid; e < 2 * CS; e += kWarps * 32) {
            const int which = e / CS, m = e - which * CS;
            double s = 0.0;
            for (int w = 0; w < kWarps; ++w) s += sh[(w * 2 + which) * CS + m];
            atomicAdd(L.stats_b + which * CS + m, s);
        }
    }
    if constexpr (SUMS) {
        __syncthreads();
        for (int e = tid; e < 2 * C; e += kWarps * 32) {
            double s = 0.0;
            for (int w = 0; w < kSlots; ++w) s += osum[w * 2 * C + e];
            atomicAdd(out_stats + e, s);
        }
    }
}

// torch's training-mode side effect on the three BatchNorms: running = (1 - m) running + m batch (variance unbiased)
__global__ void pt_update_running_kernel(const tgn_pt_layer_t L)
{
    const double cnt = static_cast<double>(L.n) * L.K;
    const int c = L.c, cs = L.c / 8;
    for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < 3 + c + cs; e += gridDim.x * blockDim.x) {
        const double* st; float *rm, *rv; float mom; int ch, cn, mode;
        if (e < 3) { st = L.stats_p; rm = L.p_rmean; rv = L.p_rvar; mom = L.p_momentum; ch = e; cn = 3; mode = L.bn_mode[0]; }
        else if (e < 3 + c) { st = L.stats_a; rm = L.a_rmean; rv = L.a_rvar; mom = L.a_momentum; ch = e - 3; cn = c; mode = L.bn_mode[1]; }
        else { st = L.stats_b; rm = L.b_rmean; rv = L.b_rvar; mom = L.b_momentum; ch = e - 3 - c; cn = cs; mode = L.bn_mode[2]; }
        if (mode != 1 || !rm || !rv) continue;
        const double mean = st[ch] / cnt;
        const double var = fmax(st[cn + ch] / cnt - mean * mean, 0.0);
        const double unbiased = cnt > 1.0 ? var * cnt / (cnt - 1.0) : var;
        rm[ch] = (1.f - mom) * rm[ch] + mom * static_cast<float>(mean);
        rv[ch] = (1.f - mom) * rv[ch] + mom * static_cast<float>(unbiased);
    }
}

template <int CPL, int PASS, bool CTAQ, int W = 32, bool SUMS = false>
int launch_pass_as(const tgn_pt_layer_t& L, cudaStream_t st, double* out_stats = nullptr)
{
    constexpr int C = W * CPL, CS = C / 8, QPW = 32 / W;
    const size_t head = (C + CS + 4) * sizeof(BnAffine);
    size_t smem = head + static_cast<size_t>(kWarps) * QPW * L.K * CS * sizeof(float);
    smem = std::max(smem, head + static_cast<size_t>(kWarps) * 2 * C * sizeof(double));
    smem = std::max(smem, head + (static_cast<size_t>(L.K) * CS + static_cast<size_t>(kWarps) * C) * sizeof(float));
    if (SUMS) {
        const size_t work = CTAQ ? static_cast<size_t>(L.K) * CS + static_cast<size_t>(kWarps) * C : static_cast<size_t>(kWarps) * QPW * L.K * CS;
        smem = std::max(smem, head + work * sizeof(float) + static_cast<size_t>(CTAQ ? 1 : kWarps * QPW) * 2 * C * sizeof(double));
    }
    const int rc = ensure_dynamic_smem(reinterpret_cast<const void*>(pt_layer_kernel<CPL, PASS, CTAQ, W, SUMS>), smem);
    if (rc != TGN_OK) return rc;
    const int per_cta = CTAQ ? 1 : kWarps * QPW;
    const int grid = std::max(1, std::min((L.n + per_cta - 1) / per_cta, (CTAQ ? 8 : 4) * sm_count()));
    pt_layer_kernel<CPL, PASS, CTAQ, W, SUMS><<<grid, kWarps * 32, smem, st>>>(L, out_stats);
    return check_launch("pt_layer_kernel");
}

// queries below this count get a CTA each (0 = never, INT_MAX = always: tgn_pt_layer_set_cta_threshold, for measurements)
int g_cta_threshold = 1024;

// c = 16 (W = 16) always runs two queries per warp: the threshold does not apply to it
template <int CPL, int PASS, int W, bool SUMS = false>
int launch_pass(const tgn_pt_layer_t& L, cudaStream_t st, double* out_stats = nullptr)
{
    if constexpr (W == 16) return launch_pass_as<CPL, PASS, false, 16, SUMS>(L, st, out_stats);
    else return L.n < g_cta_threshold ? launch_pass_as<CPL, PASS, true, 32, SUMS>(L, st, out_stats)
                                      : launch_pass_as<CPL, PASS, false, 32, SUMS>(L, st, out_stats);
}

// out_stats != NULL: the output pass also accumulates Σ / Σ² of out (tgn_pt_layer_forward_sums)
template <int CPL, int W = 32>
int run_layer(const tgn_pt_layer_t& L, cudaStream_t st, double* out_stats = nullptr)
{
    int rc = TGN_OK;
    if (L.bn_mode[0] == 1 && (rc = launch_pass<CPL, 0, W>(L, st)) != TGN_OK) return rc;
    if (L.bn_mode[1] == 1 && (rc = launch_pass<CPL, 1, W>(L, st)) != TGN_OK) return rc;
    if (L.bn_mode[2] == 1 && (rc = launch_pass<CPL, 2, W>(L, st)) != TGN_OK) return rc;
    rc = out_stats ? launch_pass<CPL, 3, W, true>(L, st, out_stats) : launch_pass<CPL, 3, W>(L, st);
    if (rc != TGN_OK) return rc;
    if (L.update_running) {
        pt_update_running_kernel<<<(3 + L.c + L.c / 8 + 127) / 128, 128, 0, st>>>(L);
        rc = check_launch("pt_update_running_kernel");
    }
    return rc;
}

int validate(const tgn_pt_layer_t& L, const char* who)
{
    if (L.K < 1 || L.K > 64 || !(L.c == 16 || L.c == 32 || L.c == 64 || L.c == 128 || L.c == 256 || L.c == 512)) {
        set_error("%s: unsupported shape c=%d K=%d", who, L.c, L.K);
        return TGN_ERR_INVALID;
    }
    if (!L.p || !L.xq || !L.xk || !L.xv || !L.idx || !L.out || !L.p_w0 || !L.p_b0 || !L.p_w1 || !L.p_b1 || !L.a_w || !L.a_b || !L.b_w || !L.b_b ||
        !L.stats_p || !L.stats_a || !L.stats_b) { set_error("%s: null argument", who); return TGN_ERR_INVALID; }
    return TGN_OK;
}

int dispatch(const tgn_pt_layer_t& L, cudaStream_t st, double* out_stats)
{
    switch (L.c) {
        case 16: return run_layer<1, 16>(L, st, out_stats);
        case 32: return run_layer<1>(L, st, out_stats);
        case 64: return run_layer<2>(L, st, out_stats);
        case 128: return run_layer<4>(L, st, out_stats);
        case 256: return run_layer<8>(L, st, out_stats);
        default: return run_layer<16>(L, st, out_stats);
    }
}

}  // namespace
}  // namespace tgn

extern "C" {

int tgn_pt_layer_struct_size(void) { return static_cast<int>(sizeof(tgn_pt_layer_t)); }

int tgn_pt_layer_set_cta_threshold(int n_queries)
{
    const int old = tgn::g_cta_threshold;
    tgn::g_cta_threshold = n_queries;
    return old;
}

int tgn_pt_layer_cta_threshold(void) { return tgn::g_cta_threshold; }

int tgn_pt_layer_forward(const tgn_pt_layer_t* layer, void* stream)
{
    using namespace tgn;
    if (!layer) { set_error("pt_layer_forward: null descriptor"); return TGN_ERR_INVALID; }
    const tgn_pt_layer_t& L = *layer;
    if (L.n <= 0) return TGN_OK;
    const int rc = validate(L, "pt_layer_forward");
    return rc != TGN_OK ? rc : dispatch(L, static_cast<cudaStream_t>(stream), nullptr);
}

int tgn_pt_layer_sums_struct_size(void) { return static_cast<int>(sizeof(tgn_pt_layer_sums_t)); }

int tgn_pt_layer_forward_sums(const tgn_pt_layer_sums_t* p, void* stream)
{
    using namespace tgn;
    if (!p) { set_error("pt_layer_forward_sums: null descriptor"); return TGN_ERR_INVALID; }
    const tgn_pt_layer_t& L = p->layer;
    if (L.n <= 0) return TGN_OK;
    int rc = validate(L, "pt_layer_forward_sums");
    if (rc != TGN_OK) return rc;
    if (!p->out_stats) { set_error("pt_layer_forward_sums: null out_stats"); return TGN_ERR_INVALID; }
    return dispatch(L, static_cast<cudaStream_t>(stream), p->out_stats);
}

}  // extern "C"
