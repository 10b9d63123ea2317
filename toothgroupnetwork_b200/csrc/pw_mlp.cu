// pw_mlp.cu -- 1x1-convolution chains with BATCH-STATISTICS BatchNorm on warpgroup MMAs (any width).
//
// Every reference call site of a set-abstraction / feature-propagation MLP runs BatchNorm in training mode,
// inference included (SURVEY.md 3c: the inference pipelines never call .eval()), i.e. layer l+1 cannot start
// before the mean / variance of layer l over ALL rows are known (pointnet2_utils.py:232-237, 289-294, 346-352).
// The single-kernel engines (sa_mlp_tc*.cu) therefore only serve folded, eval-mode BatchNorm.  This file is the
// general form: one launch per layer,
//
//      Y_l^T[c, r] = sum_k W_l[c, k] * act(X_l)[r, k] + bias_l[c]           (raw pre-activation, channel-major)
//
//   * act() of layer l is BN_{l-1} + ReLU applied WHILE BUILDING THE OPERAND: the scale/shift of every input
//     channel is derived in the kernel prologue from the fp64 sum / sum-of-squares the previous launch
//     accumulated (train mode) or from the running statistics (eval mode); CTA (0,0) also performs the
//     running-mean / running-var momentum update torch's BatchNorm would have done;
//   * layer 0 of a set abstraction builds its operand straight from the neighbourhood gather
//     ([feats | xyz - centre] or [xyz - centre | feats]); layer 0 of a feature propagation reads up to two strided
//     segments (skip features channel-first, interpolated features point-major): no grouped tensor, no concat;
//     layer 0 of a DGCNN EdgeConv builds [x_j - x_i | x_i] from the neighbour index and the strided features (mode 2);
//   * the activation after BatchNorm is ReLU, or LeakyReLU (DGCNN) written as torch writes it: v > 0 ? v : v * slope;
//   * the GEMM runs TRANSPOSED (weights = M side, rows = N side); after the K loop the accumulators are staged
//     channel-major in shared memory, so that in the epilogue a thread owns one output channel: the per-channel
//     sum / sum^2 (fp64 atomics, two per channel per CTA), and for the last set-abstraction layer the
//     per-neighbourhood max AND min over the K rows (BN's scale may be negative, so both are kept), are
//     loops inside one thread; the last SA layer never writes its (rows x C) pre-activation at all;
//   * arithmetic: batch-statistics BatchNorm amplifies rounding differences (a channel whose variance is small is
//     scaled up by 1/sqrt(var)), so this engine is fp32-GRADE: both operands are split into THREE bf16 parts
//     (x = x1 + x2 + x3 exactly: 3 x 8 = 24 significand bits) and six bf16 MMAs per K-step accumulate every
//     product term down to 2^-16 of the leading one (x1w1, x1w2, x2w1, x2w2, x1w3, x3w1) into fp32
//     accumulators; what is dropped (x2w3, x3w2, x3w3) is ~2^-23 per product, the size of an fp32 rounding.
//     `precision` 2 keeps two parts and three MMAs (~2^-16 per product, ~1e-5 end to end) for callers that do
//     not need more (eval-mode BatchNorm);
//   * weights are pre-split once per parameter version into the canonical K-major no-swizzle layout, one
//     contiguous 24 KB block per (128-channel tile, 32-wide K chunk), and fetched by the TMA engine with ONE
//     cp.async.bulk per pipeline stage completing on the stage's mbarrier; the activation side of the stage is
//     produced by the 256 threads of the CTA (one row each).
//
// Pipeline per CTA (tile = 128 output channels x 256 rows): two warpgroups, warpgroup j owns output channels
// 64j..64j+63 of the tile (one m64n256 accumulator, 128 registers per thread).  Two stages of {weights 24 KB |
// activations 48 KB}: while the MMAs of K chunk k run asynchronously, the same threads build the operand of chunk k+1.
#include <cuda_bf16.h>

#include <algorithm>
#include <cmath>

#include "common.cuh"
#include "pw_bn.cuh"
#include "tc_common.cuh"
#include "tgn_b200.h"

namespace tgn {
namespace {

using namespace tc;

constexpr int kMT = 128;                 // output channels per tile (M of the MMAs: two 64-channel warpgroup slices)
constexpr int kNT = 256;                 // rows per tile (N of the MMA)
constexpr int kKC = 32;                  // K per pipeline stage (two K=16 MMA steps)
constexpr int kThreads = kNT;            // one producer thread per row; two consumer warpgroups
constexpr int kParts = 3;                                // bf16 parts per operand
constexpr uint32_t kWPart = kMT * kKC * 2;               // bytes of one part of a packed weight block (8 KB)
constexpr uint32_t kWBlock = kWPart * kParts;            // 24 KB
constexpr uint32_t kXPart = kNT * kKC * 2;               // bytes of one part of the activation side of a stage (16 KB)
constexpr uint32_t kStageBytes = kWBlock + kParts * kXPart;   // 72 KB
constexpr int kStages = 2;
constexpr int kYStride = kNT + 1;                        // floats per channel of the staged accumulator tile: odd, so the 32
                                                         // channels a warp reads at one column fall in 32 different banks
static_assert(kMT * kYStride * 4 <= kStages * kStageBytes, "the staged accumulator tile reuses the stage buffers");

struct PwArgs {
    tgn_pw_layer_t L;
    int nkc;                 // K chunks
    uint32_t off_affine;     // float4[cin] (mean_hi, mean_lo, scale, beta) when in_affine != 0
    uint32_t off_bars;
    uint32_t smem_total;
    int n_groups;            // rows / group when extrema are produced
};

__device__ __forceinline__ uint32_t pack_bf16(float a, float b) {
    uint32_t r;
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(b), "f"(a));
    return r;
}
// (a, b) -> three packed bf16 pairs with a = a1 + a2 + a3 exactly (each subtraction is exact in fp32)
__device__ __forceinline__ void split_bf16_pair3(float a, float b, uint32_t& p1, uint32_t& p2, uint32_t& p3) {
    p1 = pack_bf16(a, b);
    const float ra = __fsub_rn(a, __uint_as_float(p1 << 16)), rb = __fsub_rn(b, __uint_as_float(p1 & 0xFFFF0000u));
    p2 = pack_bf16(ra, rb);
    p3 = pack_bf16(__fsub_rn(ra, __uint_as_float(p2 << 16)), __fsub_rn(rb, __uint_as_float(p2 & 0xFFFF0000u)));
}
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}
// ordered by the sign BIT, not by v >= 0: -0.0 compares >= 0 but its bits are INT_MIN as a signed int, so it belongs on the
// unsigned side with the other negative values (where it is the largest)
__device__ __forceinline__ void atomic_max_float(float* addr, float v) {
    if (__float_as_int(v) >= 0) atomicMax(reinterpret_cast<int*>(addr), __float_as_int(v));
    else atomicMin(reinterpret_cast<unsigned int*>(addr), __float_as_uint(v));
}
__device__ __forceinline__ void atomic_min_float(float* addr, float v) {
    if (__float_as_int(v) >= 0) atomicMin(reinterpret_cast<int*>(addr), __float_as_int(v));
    else atomicMax(reinterpret_cast<unsigned int*>(addr), __float_as_uint(v));
}

__global__ void __launch_bounds__(kThreads, 1) pw_layer_kernel(const PwArgs a)
{
    extern __shared__ __align__(1024) uint8_t smem[];
    const tgn_pw_layer_t& L = a.L;
    const uint32_t sbase = smem_u32(smem);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int r0 = blockIdx.x * kNT;               // first row of the tile
    const int m0 = blockIdx.y * kMT;               // first output channel of the tile
    const uint32_t bar_full = sbase + a.off_bars;                      // kStages x 8: weights of the stage have landed
    float4* affine = reinterpret_cast<float4*>(smem + a.off_affine);

    if (tid == 0) {
        for (int s = 0; s < kStages; ++s) mbar_init(bar_full + 8 * s, 1);
        mbar_fence_init();
    }
    // ---- input BatchNorm (of the previous layer) -> per-channel scale / shift ------------------------------
    if (L.in_affine) {
        const double cnt = static_cast<double>(L.rows);
        for (int c = tid; c < L.cin; c += kThreads) {
            affine[c] = bn_scale_shift(L.in_affine, c, L.cin, L.in_stats, cnt, L.in_gamma, L.in_beta, L.in_eps, L.in_running_mean,
                                       L.in_running_var);
        }
    }
    __syncthreads();
    if (L.in_affine == 1 && L.in_update_running && blockIdx.x == 0 && blockIdx.y == 0) {
        for (int c = tid; c < L.cin; c += kThreads)
            bn_update_running(c, L.cin, L.in_stats, static_cast<double>(L.rows), L.in_momentum, L.in_running_mean, L.in_running_var);
    }
    float acc[kNT / 2];              // D^T[m0 + 64 wg + .., r0 + ..] of this thread's warpgroup wg
#pragma unroll
    for (int i = 0; i < kNT / 2; ++i) acc[i] = 0.f;
    {
        // =========================== producers: one row each; MMAs: one 64-channel slice per warpgroup ==========
        const int r = r0 + tid;
        const bool valid = r < L.rows;
        // source addressing of this row
        const float* seg0 = nullptr; const float* seg1 = nullptr;   // mode 0
        const float* pf = nullptr;                                    // mode 1: gathered feature row; mode 2: neighbour's features
        const float* pe = nullptr;                                    // mode 2: the centre point's features
        float rel0 = 0.f, rel1 = 0.f, rel2 = 0.f;
        bool row_ok = valid;
        if (L.mode == 0) {
            if (valid) {
                const int b = r / L.rows_per_batch, n = r - b * L.rows_per_batch;
                seg0 = L.seg_ptr[0] + b * L.seg_batch_stride[0] + n * L.seg_row_stride[0];
                if (L.seg_channels[1] > 0) seg1 = L.seg_ptr[1] + b * L.seg_batch_stride[1] + n * L.seg_row_stride[1];
            }
        } else if (L.mode == 2) {
            if (valid) {
                const int pt = r / L.K;                                   // b*N + n
                const int b = pt / L.N, n = pt - b * L.N;
                const int m = __ldg(L.gidx + r);
                if (m >= 0 && m < L.N) {
                    const float* xb = L.edge_x + b * L.edge_stride[0];
                    pe = xb + n * L.edge_stride[2];
                    pf = xb + m * L.edge_stride[2];
                } else {
                    row_ok = false;
                }
            }
        } else if (valid) {
            const int grp = r / L.K;                                  // (b*S + s)
            const int b = grp / L.S;
            const int j = __ldg(L.gidx + r);
            if (j >= 0 && j < L.N) {
                const float* px = L.xyz + 3 * (static_cast<size_t>(b) * L.N + j);
                const float* pc = L.new_xyz + 3 * static_cast<size_t>(grp);
                rel0 = __fsub_rn(__ldg(px), __ldg(pc));
                rel1 = __fsub_rn(__ldg(px + 1), __ldg(pc + 1));
                rel2 = __fsub_rn(__ldg(px + 2), __ldg(pc + 2));
                pf = L.feats ? L.feats + (static_cast<size_t>(b) * L.N + j) * L.D : nullptr;
            } else {
                row_ok = false;                                       // empty ball (index N): zero row, as the fused engines do
            }
        }
        const int c0seg = L.seg_channels[0];
        const long long cs0 = L.seg_chan_stride[0], cs1 = L.seg_chan_stride[1];
        const int feat_lo = L.xyz_first ? 3 : 0;                      // channel of feats[0]
        const int rel_lo = L.xyz_first ? 0 : L.D;                     // channel of rel0
        const int wg = warp >> 2;
        for (int kc = 0; kc < a.nkc; ++kc) {
            // stage s was last read by the MMAs of chunk kc - 2, which both warpgroups have waited for (end of the
            // previous iteration)
            const int s = kc % kStages;
            const uint32_t stage = sbase + s * kStageBytes;
            if (tid == 0) {
                mbar_arrive_expect_tx(bar_full + 8 * s, kWBlock);
                bulk_g2s(stage, static_cast<const uint8_t*>(L.w_packed) + (static_cast<size_t>(blockIdx.y) * a.nkc + kc) * kWBlock, kWBlock,
                         bar_full + 8 * s);
            }
            const int k0 = kc * kKC;
            float x[kKC];
            if (!row_ok) {
#pragma unroll
                for (int i = 0; i < kKC; ++i) x[i] = 0.f;
            } else if (L.mode == 0) {
#pragma unroll
                for (int i = 0; i < kKC; ++i) {
                    const int k = k0 + i;
                    float v = 0.f;
                    if (k < c0seg) v = __ldg(seg0 + k * cs0);
                    else if (k < L.cin) v = __ldg(seg1 + (k - c0seg) * cs1);
                    x[i] = v;
                }
            } else if (L.mode == 2) {
                // channel order of cat((feature - x, x), dim=3).permute(0, 3, 1, 2) (dgcnn.py:39)
#pragma unroll
                for (int i = 0; i < kKC; ++i) {
                    const int k = k0 + i;
                    float v = 0.f;
                    if (k < L.edge_C) v = __fsub_rn(__ldg(pf + k * L.edge_stride[1]), __ldg(pe + k * L.edge_stride[1]));
                    else if (k < L.cin) v = __ldg(pe + (k - L.edge_C) * L.edge_stride[1]);
                    x[i] = v;
                }
            } else {
#pragma unroll
                for (int i = 0; i < kKC; ++i) {
                    const int k = k0 + i;
                    const int kf = k - feat_lo;
                    float v = 0.f;
                    if (kf >= 0 && kf < L.D) v = __ldg(pf + kf);
                    else if (k == rel_lo) v = rel0;
                    else if (k == rel_lo + 1) v = rel1;
                    else if (k == rel_lo + 2) v = rel2;
                    x[i] = v;
                }
            }
            if (L.in_affine && row_ok) {
#pragma unroll
                for (int i = 0; i < kKC; ++i) {
                    const int k = k0 + i;
                    if (k < L.cin) {
                        const float v = bn_apply(x[i], affine[k]);
                        x[i] = L.in_act == 1 ? leaky_relu(v, L.in_act_slope) : fmaxf(v, 0.f);
                    }
                }
            }
            const uint32_t x1 = stage + kWBlock + tid * 16;
#pragma unroll
            for (int j = 0; j < kKC / 8; ++j) {
                uint32_t p1[4], p2[4], p3[4];
#pragma unroll
                for (int u = 0; u < 4; ++u) split_bf16_pair3(x[8 * j + 2 * u], x[8 * j + 2 * u + 1], p1[u], p2[u], p3[u]);
                st_shared_v4(x1 + j * (kNT * 16), p1[0], p1[1], p1[2], p1[3]);
                st_shared_v4(x1 + kXPart + j * (kNT * 16), p2[0], p2[1], p2[2], p2[3]);
                st_shared_v4(x1 + 2 * kXPart + j * (kNT * 16), p3[0], p3[1], p3[2], p3[3]);
            }
            proxy_fence_async();
            __syncthreads();                                  // the activation side of the stage is complete
            mbar_wait(bar_full + 8 * s, (kc / kStages) & 1);  // ... and its weights have landed
            fence_regs(acc);
            wgmma_fence();
            const uint32_t w0 = stage + wg * 64 * 16, x0 = stage + kWBlock;
#pragma unroll
            for (int ks = 0; ks < kKC / 16; ++ks) {
                uint64_t dw[kParts], dx[kParts];
#pragma unroll
                for (int i = 0; i < kParts; ++i) {
                    dw[i] = make_smem_desc(w0 + i * kWPart + ks * 2 * (kMT * 16), kMT * 16);
                    dx[i] = make_smem_desc(x0 + i * kXPart + ks * 2 * (kNT * 16), kNT * 16);
                }
                wgmma_bf16<kNT>(acc, dw[0], dx[0], kc > 0 || ks > 0);
                wgmma_bf16<kNT>(acc, dw[0], dx[1], true);
                wgmma_bf16<kNT>(acc, dw[1], dx[0], true);
                if (L.precision != 2) {
                    wgmma_bf16<kNT>(acc, dw[1], dx[1], true);
                    wgmma_bf16<kNT>(acc, dw[0], dx[2], true);
                    wgmma_bf16<kNT>(acc, dw[2], dx[0], true);
                }
            }
            wgmma_commit();
            wgmma_wait<1>();                                  // the MMAs of chunk kc - 1 are complete in this warpgroup,
            fence_regs(acc);
            __syncthreads();                                  // ... and in the other one: stage (kc + 1) % 2 is free
        }
        wgmma_wait<0>();
        fence_regs(acc);
        __syncthreads();                                      // every MMA is complete: the stage buffers are free
        // accumulators -> channel-major tile in the (now idle) stage buffers
        float* ytile = reinterpret_cast<float*>(smem);
        const int ch = 64 * wg + 16 * (warp & 3) + (lane >> 2);
#pragma unroll
        for (int i = 0; i < kNT / 8; ++i) {
            const int col = 8 * i + 2 * (lane & 3);
            ytile[ch * kYStride + col] = acc[4 * i];
            ytile[ch * kYStride + col + 1] = acc[4 * i + 1];
            ytile[(ch + 8) * kYStride + col] = acc[4 * i + 2];
            ytile[(ch + 8) * kYStride + col + 1] = acc[4 * i + 3];
        }
        __syncthreads();

        // =========================== epilogue: thread = output channel ======================================
        const int q = warp & 3, half = warp >> 2;
        const int c = m0 + 32 * q + lane;
        const bool c_ok = c < L.cout;
        const float bias = (c_ok && L.bias) ? __ldg(L.bias + c) : 0.f;
        const float* trow = ytile + (32 * q + lane) * kYStride + half * (kNT / 2);
        double s1 = 0.0, s2 = 0.0;
        const int G = L.group;
        float gmax = -INFINITY, gmin = INFINITY;
        const int col_lo = r0 + half * (kNT / 2);
        const bool vec_ok = (L.rows & 3) == 0;
        for (int cb = 0; cb < kNT / 2; cb += 32) {
            const int rb = col_lo + cb;                       // global row of the block's first column
            if (rb >= L.rows) break;                          // warp-uniform
            uint32_t v[32];
#pragma unroll
            for (int i = 0; i < 32; ++i) v[i] = __float_as_uint(trow[cb + i]);
            const int nvalid = min(32, L.rows - rb);
            // the block's fp32 partial sums are taken about its first value p (row rb is always valid) and re-expanded in fp64:
            // sum (y - p)^2 keeps the variance of a channel whose |mean| >> std, which sum y^2 in fp32 would round away
            float p = 0.f, f1 = 0.f, f2 = 0.f;
#pragma unroll
            for (int i = 0; i < 32; ++i) {
                float y = __uint_as_float(v[i]) + bias;
                if (L.cloud_bias && c_ok && i < nvalid) y += __ldg(L.cloud_bias + static_cast<size_t>((rb + i) / L.rows_per_batch) * L.cout + c);
                v[i] = __float_as_uint(y);
                if (i == 0) p = y;
                if (i < nvalid) { const float d = __fsub_rn(y, p); f1 += d; f2 = fmaf(d, d, f2); }
            }
            const double pd = static_cast<double>(p), np = static_cast<double>(nvalid) * pd;
            s1 += np + static_cast<double>(f1);
            s2 += fma(pd, np + 2.0 * static_cast<double>(f1), static_cast<double>(f2));
            if (L.y && c_ok) {
                float* dst = L.y + static_cast<size_t>(c) * L.rows + rb;
                if (vec_ok && nvalid == 32) {
#pragma unroll
                    for (int i = 0; i < 32; i += 4)
                        *reinterpret_cast<float4*>(dst + i) = make_float4(__uint_as_float(v[i]), __uint_as_float(v[i + 1]),
                                                                          __uint_as_float(v[i + 2]), __uint_as_float(v[i + 3]));
                } else {
#pragma unroll
                    for (int i = 0; i < 32; ++i)
                        if (i < nvalid) dst[i] = __uint_as_float(v[i]);
                }
            }
            if (L.ymax) {
                // extrema over groups of G consecutive rows (rows is a multiple of G)
#pragma unroll
                for (int i = 0; i < 32; ++i) {
                    if (i < nvalid) {
                        const float y = __uint_as_float(v[i]);
                        gmax = fmaxf(gmax, y);
                        gmin = fminf(gmin, y);
                        const int rr = rb + i;
                        const bool group_end = ((rr + 1) % G) == 0;
                        const bool range_end = (cb + i == kNT / 2 - 1) || (rr == L.rows - 1);
                        if (group_end || range_end) {
                            if (c_ok) {
                                const size_t o = static_cast<size_t>(c) * a.n_groups + rr / G;
                                if (L.extrema_atomic) { atomic_max_float(L.ymax + o, gmax); atomic_min_float(L.ymin + o, gmin); }
                                else { L.ymax[o] = gmax; L.ymin[o] = gmin; }
                            }
                            gmax = -INFINITY; gmin = INFINITY;
                        }
                    }
                }
            }
        }
        if (L.stats && c_ok) {
            atomicAdd(L.stats + c, s1);
            atomicAdd(L.stats + L.cout + c, s2);
        }
    }
}

// W (cout, cin) fp32 row-major -> packed blocks [(mt, kc)] of three parts, each [4 chunks][128 rows][8 bf16]
__global__ void pw_pack_weights_kernel(int cout, int cin, int nkc, const float* __restrict__ w, uint8_t* __restrict__ packed)
{
    const int mt = blockIdx.y, kc = blockIdx.x;
    uint8_t* blk = packed + (static_cast<size_t>(mt) * nkc + kc) * kWBlock;
    for (int e = threadIdx.x; e < kMT * kKC; e += blockDim.x) {
        const int row = e / kKC, kk = e - row * kKC;
        const int c = mt * kMT + row, k = kc * kKC + kk;
        const float v = (c < cout && k < cin) ? __ldg(w + static_cast<size_t>(c) * cin + k) : 0.f;
        const __nv_bfloat16 w1 = __float2bfloat16_rn(v);
        const float r1 = __fsub_rn(v, __bfloat162float(w1));
        const __nv_bfloat16 w2 = __float2bfloat16_rn(r1);
        const __nv_bfloat16 w3 = __float2bfloat16_rn(__fsub_rn(r1, __bfloat162float(w2)));
        const uint32_t off = static_cast<uint32_t>(kk >> 3) * (kMT * 16) + row * 16 + (kk & 7) * 2;
        *reinterpret_cast<__nv_bfloat16*>(blk + off) = w1;
        *reinterpret_cast<__nv_bfloat16*>(blk + kWPart + off) = w2;
        *reinterpret_cast<__nv_bfloat16*>(blk + 2 * kWPart + off) = w3;
    }
}

// out[b, c_off + c, n] = act(scale_c * v + shift_c), v = Y[c, b*rpb + n] or the max / min pick by sign(scale): BatchNorm and
// the activation are both monotone, so the extreme that maps to the largest output is the max when scale >= 0, else the min
__global__ void pw_apply_kernel(const tgn_pw_apply_t p)
{
    __shared__ float4 ss;
    const int c = blockIdx.y;
    if (threadIdx.x == 0) {
        ss = p.affine ? bn_scale_shift(p.affine, c, p.channels, p.stats, static_cast<double>(p.stat_rows), p.gamma, p.beta, p.eps,
                                       p.running_mean, p.running_var)
                      : make_float4(0.f, 0.f, 1.f, 0.f);
        if (p.affine == 1 && p.update_running && blockIdx.x == 0)
            bn_update_running(c, p.channels, p.stats, static_cast<double>(p.stat_rows), p.momentum, p.running_mean, p.running_var);
    }
    __syncthreads();
    const float4 aff = ss;
    const float* src = (p.ymin && aff.z < 0.f) ? p.ymin : p.src;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < p.rows; i += gridDim.x * blockDim.x) {
        const int b = i / p.rows_per_batch, n = i - b * p.rows_per_batch;
        float v = bn_apply(src[static_cast<size_t>(c) * p.rows + i], aff);
        if (p.act == 1) v = leaky_relu(v, p.act_slope);
        else if (p.relu) v = fmaxf(v, 0.f);
        p.out[(static_cast<size_t>(b) * p.out_channels + p.out_c_offset + c) * p.rows_per_batch + n] = v;
    }
}

// out[b, c] = sum_k w[c, k] * g[b, k], accumulated in fp64 in index order and rounded once: one warp per output
__global__ void pw_cloud_bias_kernel(int B, int cout, int cin, const float* __restrict__ w, long long w_row_stride,
                                     const float* __restrict__ g, long long g_batch_stride, float* __restrict__ out)
{
    const int o = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (o >= B * cout) return;
    const int b = o / cout, c = o - b * cout;
    const float* wr = w + c * w_row_stride;
    const float* gr = g + b * g_batch_stride;
    double acc = 0.0;
    for (int k = lane; k < cin; k += 32) acc = fma(static_cast<double>(__ldg(wr + k)), static_cast<double>(__ldg(gr + k)), acc);
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, d);
    if (lane == 0) out[o] = static_cast<float>(acc);
}

__global__ void pw_fill_kernel(float* p, size_t n, float v)
{
    for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n; i += static_cast<size_t>(gridDim.x) * blockDim.x) p[i] = v;
}

}  // namespace
}  // namespace tgn

extern "C" {

int tgn_pw_struct_size(int which) { return which == 0 ? static_cast<int>(sizeof(tgn_pw_layer_t)) : static_cast<int>(sizeof(tgn_pw_apply_t)); }

size_t tgn_pw_packed_bytes(int cout, int cin)
{
    using namespace tgn;
    const size_t mt = (static_cast<size_t>(cout) + kMT - 1) / kMT, nkc = (static_cast<size_t>(cin) + kKC - 1) / kKC;
    return mt * nkc * kWBlock;
}

int tgn_pw_pack_weights(int cout, int cin, const float* w, void* packed, void* stream)
{
    using namespace tgn;
    if (cout < 1 || cin < 1 || !w || !packed) { set_error("pw_pack_weights: bad arguments"); return TGN_ERR_INVALID; }
    const int nkc = (cin + kKC - 1) / kKC;
    dim3 grid(nkc, (cout + kMT - 1) / kMT);
    pw_pack_weights_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(cout, cin, nkc, w, static_cast<uint8_t*>(packed));
    return check_launch("pw_pack_weights_kernel");
}

int tgn_pw_layer_forward(const tgn_pw_layer_t* layer, void* stream)
{
    using namespace tgn;
    if (!layer) { set_error("pw_layer_forward: null descriptor"); return TGN_ERR_INVALID; }
    PwArgs a{};
    a.L = *layer;
    const tgn_pw_layer_t& L = a.L;
    if (L.rows < 1 || L.cin < 1 || L.cout < 1 || !L.w_packed) { set_error("pw_layer_forward: bad shape"); return TGN_ERR_INVALID; }
    if (L.mode == 0) {
        if (!L.seg_ptr[0] || L.seg_channels[0] + L.seg_channels[1] != L.cin || L.rows_per_batch < 1 ||
            (L.seg_channels[1] > 0 && !L.seg_ptr[1])) { set_error("pw_layer_forward: bad segments"); return TGN_ERR_INVALID; }
    } else if (L.mode == 1) {
        if (!L.xyz || !L.new_xyz || !L.gidx || L.K < 1 || L.S < 1 || L.cin != L.D + 3 || (L.D > 0 && !L.feats)) {
            set_error("pw_layer_forward: bad gather arguments"); return TGN_ERR_INVALID;
        }
    } else if (L.mode == 2) {
        if (!L.edge_x || !L.gidx || L.K < 1 || L.N < 1 || L.edge_C < 1 || L.cin != 2 * L.edge_C ||
            L.rows % (static_cast<long long>(L.N) * L.K) != 0) {
            set_error("pw_layer_forward: bad edge-feature arguments (need edge_x, gidx, K, N >= 1, cin = 2 * edge_C, rows %% (N * K) == 0)");
            return TGN_ERR_INVALID;
        }
    } else { set_error("pw_layer_forward: unknown mode %d", L.mode); return TGN_ERR_INVALID; }
    if (L.cloud_bias && L.rows_per_batch < 1) { set_error("pw_layer_forward: cloud_bias needs rows_per_batch"); return TGN_ERR_INVALID; }
    if (L.in_affine == 1 && !L.in_stats) { set_error("pw_layer_forward: in_affine=1 needs in_stats"); return TGN_ERR_INVALID; }
    if (L.in_affine == 2 && (!L.in_running_mean || !L.in_running_var)) { set_error("pw_layer_forward: in_affine=2 needs running statistics"); return TGN_ERR_INVALID; }
    if (L.ymax) {
        if (!L.ymin || L.group < 1 || L.rows % L.group != 0) { set_error("pw_layer_forward: bad extrema arguments"); return TGN_ERR_INVALID; }
        a.n_groups = L.rows / L.group;
        if (!L.extrema_atomic && (kNT / 2) % L.group != 0) { set_error("pw_layer_forward: group %d needs the atomic extrema path", L.group); return TGN_ERR_INVALID; }
    }
    a.nkc = (L.cin + kKC - 1) / kKC;
    const uint32_t affine_bytes = L.in_affine ? static_cast<uint32_t>(L.cin) * 16 : 0;
    a.off_affine = kStages * kStageBytes;
    a.off_bars = (a.off_affine + affine_bytes + 15) / 16 * 16;
    a.smem_total = a.off_bars + 8 * kStages;
    if (a.smem_total > 227 * 1024) { set_error("pw_layer_forward: cin %d too wide", L.cin); return TGN_ERR_INVALID; }
    const int rc_attr = ensure_dynamic_smem(reinterpret_cast<const void*>(pw_layer_kernel), 227 * 1024);
    if (rc_attr != TGN_OK) return rc_attr;
    dim3 grid((L.rows + kNT - 1) / kNT, (L.cout + kMT - 1) / kMT);
    pw_layer_kernel<<<grid, kThreads, a.smem_total, static_cast<cudaStream_t>(stream)>>>(a);
    return check_launch("pw_layer_kernel");
}

int tgn_pw_apply(const tgn_pw_apply_t* p, void* stream)
{
    using namespace tgn;
    if (!p || !p->src || !p->out || p->rows < 1 || p->channels < 1 || p->rows_per_batch < 1) { set_error("pw_apply: bad arguments"); return TGN_ERR_INVALID; }
    if (p->affine == 1 && !p->stats) { set_error("pw_apply: affine=1 needs stats"); return TGN_ERR_INVALID; }
    const int bx = std::max(1, std::min((p->rows + 255) / 256, std::max(1, 4 * sm_count() / p->channels)));
    dim3 grid(bx, p->channels);
    pw_apply_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(*p);
    return check_launch("pw_apply_kernel");
}

int tgn_pw_cloud_bias(int B, int cout, int cin, const float* w, long long w_row_stride, const float* g, long long g_batch_stride,
                      float* out, void* stream)
{
    using namespace tgn;
    if (B < 1 || cout < 1 || cin < 1 || !w || !g || !out || w_row_stride < cin || g_batch_stride < 0) {
        set_error("pw_cloud_bias: bad arguments"); return TGN_ERR_INVALID;
    }
    const int outputs = B * cout;
    pw_cloud_bias_kernel<<<(outputs + 7) / 8, 256, 0, static_cast<cudaStream_t>(stream)>>>(B, cout, cin, w, w_row_stride, g, g_batch_stride, out);
    return check_launch("pw_cloud_bias_kernel");
}

int tgn_pw_fill(float* ptr, long long n, float value, void* stream)
{
    using namespace tgn;
    if (n <= 0) return TGN_OK;
    const int blocks = static_cast<int>(std::min<long long>((n + 255) / 256, 8LL * sm_count()));
    pw_fill_kernel<<<blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(ptr, static_cast<size_t>(n), value);
    return check_launch("pw_fill_kernel");
}

}  // extern "C"
