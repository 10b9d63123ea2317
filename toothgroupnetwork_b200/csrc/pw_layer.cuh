// pw_layer.cuh -- the layer kernel of the 1x1-convolution chain (pw_mlp.cu), templated on its tile and its accumulation.
//
//   pw_layer_kernel<256, 0>  tile = 128 output channels x 256 rows; each consumer warpgroup's 64 channels x 256 rows are one m64n256
//                            wgmma accumulator that takes the whole K of the layer (pw_mlp.cu);
//   pw_layer_kernel<128, P>  tile = 128 output channels x 128 rows, PROMOTED accumulation (pw_mlp_promoted.cu): every P K-steps of
//                            16 the m64n128 accumulator is added into an fp32 register total with a round-to-nearest FADD, and the
//                            next K-step's first MMA starts a fresh accumulator (scale-d = 0).
//
// Why: the tensor cores truncate when they accumulate, so each MMA can leave up to about one ulp of the running sum behind, always
// towards zero.  Over 6 MMAs per K-step and K up to ~1 200 that bias grows with K.  Batch-statistics BatchNorm subtracts the batch
// mean and with it most of the common bias; BatchNorm on running statistics does not, so a layer whose outputs carry large
// per-cloud offsets shows the bias after the running-mean subtraction (DESIGN §3.12).  The promoted total bounds the truncated
// part to one chunk of 6 P MMAs; what crosses the chunks is rounded to nearest.
//
// Both forms share the producers (one row per thread at 256 rows; two threads per row at 128 rows, each building 16 of the stage's
// 32 K values), the two-stage cp.async.bulk weight pipeline and the epilogue (staged channel-major, pivoted per-channel sums,
// cloud_bias, max / min over groups).
#pragma once
#include <cuda_bf16.h>

#include <cmath>

#include "common.cuh"
#include "pw_bn.cuh"
#include "tc_common.cuh"
#include "tgn_b200.h"

namespace tgn {
namespace pw {

using namespace tc;

constexpr int kMT = 128;                 // output channels per tile (M of the MMAs: two 64-channel warpgroup slices)
constexpr int kKC = 32;                  // K per pipeline stage (two K=16 MMA steps)
constexpr int kThreads = 256;            // two consumer warpgroups; producers: one or two threads per row
constexpr int kParts = 3;                                // bf16 parts per operand
constexpr uint32_t kWPart = kMT * kKC * 2;               // bytes of one part of a packed weight block (8 KB)
constexpr uint32_t kWBlock = kWPart * kParts;            // 24 KB
constexpr int kStages = 2;

// NT = rows per tile (N of the MMA)
template <int NT>
struct Tile {
    static constexpr uint32_t kXPart = NT * kKC * 2;                    // bytes of one part of the activation side of a stage
    static constexpr uint32_t kStageBytes = kWBlock + kParts * kXPart;  // 72 KB at NT = 256, 48 KB at NT = 128
    static constexpr int kYStride = NT + 1;              // floats per channel of the staged accumulator tile: odd, so the 32
                                                         // channels a warp reads at one column fall in 32 different banks
    static constexpr int kSplit = kThreads / NT;         // producer threads per row
    static constexpr int kKT = kKC / kSplit;             // K values of a stage one producer thread builds
    static_assert(kMT * kYStride * 4 <= kStages * kStageBytes, "the staged accumulator tile reuses the stage buffers");
    static_assert(kKT % 8 == 0, "a producer thread stores whole 8-value K chunks");
};

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

// NT rows per tile; P = 0: one accumulator over the whole K; P > 0: promoted every P K-steps of 16
template <int NT, int P>
__global__ void __launch_bounds__(kThreads, 1) pw_layer_kernel(const PwArgs a)
{
    using T = Tile<NT>;
    constexpr int kNT = NT, kYStride = T::kYStride, kKT = T::kKT;
    constexpr uint32_t kXPart = T::kXPart, kStageBytes = T::kStageBytes;
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
    float acc[kNT / 2];              // D^T[m0 + 64 wg + .., r0 + ..] of this thread's warpgroup wg (of the current chunk when P > 0)
#pragma unroll
    for (int i = 0; i < kNT / 2; ++i) acc[i] = 0.f;
    float tot[P > 0 ? kNT / 2 : 1];  // P > 0: the round-to-nearest sum of the completed chunks
#pragma unroll
    for (int i = 0; i < (P > 0 ? kNT / 2 : 1); ++i) tot[i] = 0.f;
    {
        // =========================== producers: one row each (two at NT = 128); MMAs: one 64-channel slice per warpgroup ======
        const int prow = T::kSplit == 1 ? tid : tid % kNT;            // this thread's row of the tile
        const int kq = T::kSplit == 1 ? 0 : tid / kNT;                // ... and its part of the stage's K
        const int r = r0 + prow;
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
            const int k0 = kc * kKC + kq * kKT;
            float x[kKT];
            if (!row_ok) {
#pragma unroll
                for (int i = 0; i < kKT; ++i) x[i] = 0.f;
            } else if (L.mode == 0) {
#pragma unroll
                for (int i = 0; i < kKT; ++i) {
                    const int k = k0 + i;
                    float v = 0.f;
                    if (k < c0seg) v = __ldg(seg0 + k * cs0);
                    else if (k < L.cin) v = __ldg(seg1 + (k - c0seg) * cs1);
                    x[i] = v;
                }
            } else if (L.mode == 2) {
                // channel order of cat((feature - x, x), dim=3).permute(0, 3, 1, 2) (dgcnn.py:39)
#pragma unroll
                for (int i = 0; i < kKT; ++i) {
                    const int k = k0 + i;
                    float v = 0.f;
                    if (k < L.edge_C) v = __fsub_rn(__ldg(pf + k * L.edge_stride[1]), __ldg(pe + k * L.edge_stride[1]));
                    else if (k < L.cin) v = __ldg(pe + (k - L.edge_C) * L.edge_stride[1]);
                    x[i] = v;
                }
            } else {
#pragma unroll
                for (int i = 0; i < kKT; ++i) {
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
                for (int i = 0; i < kKT; ++i) {
                    const int k = k0 + i;
                    if (k < L.cin) {
                        const float v = bn_apply(x[i], affine[k]);
                        x[i] = L.in_act == 1 ? leaky_relu(v, L.in_act_slope) : fmaxf(v, 0.f);
                    }
                }
            }
            const uint32_t x1 = stage + kWBlock + prow * 16 + kq * (kKT / 8) * (kNT * 16);
#pragma unroll
            for (int j = 0; j < kKT / 8; ++j) {
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
                bool fresh;                                   // this K-step's first MMA starts the accumulator (scale-d = 0)
                if constexpr (P == 0) {
                    fresh = kc == 0 && ks == 0;
                } else {
                    const int step = kc * (kKC / 16) + ks;
                    fresh = step % P == 0;
                    if (fresh && step > 0) {
                        // promotion: the chunk that ends here is complete in this warpgroup; add it into the total, rounded to nearest
                        if (ks > 0) wgmma_commit();
                        wgmma_wait<0>();
                        fence_regs(acc);
#pragma unroll
                        for (int i = 0; i < kNT / 2; ++i) tot[i] = __fadd_rn(tot[i], acc[i]);
                        fence_regs(acc);
                        wgmma_fence();
                    }
                }
                uint64_t dw[kParts], dx[kParts];
#pragma unroll
                for (int i = 0; i < kParts; ++i) {
                    dw[i] = make_smem_desc(w0 + i * kWPart + ks * 2 * (kMT * 16), kMT * 16);
                    dx[i] = make_smem_desc(x0 + i * kXPart + ks * 2 * (kNT * 16), kNT * 16);
                }
                wgmma_bf16<kNT>(acc, dw[0], dx[0], !fresh);
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
        if constexpr (P > 0) {
#pragma unroll
            for (int i = 0; i < kNT / 2; ++i) acc[i] = __fadd_rn(tot[i], acc[i]);      // the last chunk
        }
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

// Shared-memory layout, the half-tile extrema check and the launch of pw_layer_kernel<NT, P>; `a` holds a validated descriptor
template <int NT, int P>
int pw_layer_launch(PwArgs& a, cudaStream_t stream, const char* name)
{
    const tgn_pw_layer_t& L = a.L;
    if (L.ymax && !L.extrema_atomic && (NT / 2) % L.group != 0) {
        set_error("pw_layer_forward: group %d needs the atomic extrema path at %d-row tiles", L.group, NT);
        return TGN_ERR_INVALID;
    }
    a.nkc = (L.cin + kKC - 1) / kKC;
    const uint32_t affine_bytes = L.in_affine ? static_cast<uint32_t>(L.cin) * 16 : 0;
    a.off_affine = kStages * Tile<NT>::kStageBytes;
    a.off_bars = (a.off_affine + affine_bytes + 15) / 16 * 16;
    a.smem_total = a.off_bars + 8 * kStages;
    if (a.smem_total > 227 * 1024) { set_error("pw_layer_forward: cin %d too wide", L.cin); return TGN_ERR_INVALID; }
    const int rc_attr = ensure_dynamic_smem(reinterpret_cast<const void*>(pw_layer_kernel<NT, P>), 227 * 1024);
    if (rc_attr != TGN_OK) return rc_attr;
    dim3 grid((L.rows + NT - 1) / NT, (L.cout + kMT - 1) / kMT);
    pw_layer_kernel<NT, P><<<grid, kThreads, a.smem_total, stream>>>(a);
    return check_launch(name);
}

// pw_mlp_promoted.cu: pw_layer_kernel<128, kPromoteSteps>
constexpr int kPromoteNT = 128;
int pw_layer_launch_promoted(PwArgs& a, cudaStream_t stream);

}  // namespace pw
}  // namespace tgn
