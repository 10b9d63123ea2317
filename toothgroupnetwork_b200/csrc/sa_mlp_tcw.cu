// sa_mlp_tcw.cu -- warpgroup-MMA engine of the fused set-abstraction body for WIDE hidden layers (up to 128).
//
// The 3xTF32 engine in sa_mlp_tc.cu keeps every inter-layer operand as two tf32 tiles; at 128 channels
// that is 128 KB per 128-row tile and nothing fits.  The reference's real pointnet_pp SA1
// (PointNetSetAbstractionMsg(1024,[.025,.05],[32,64],6,[[128,128],[128,128]]), pointnet_pp.py:13) is
// exactly that shape, 15x the FLOPs of the BASELINE form.  This engine keeps the same structure (tile
// groups of 128 threads = one warpgroup, two 64-row wgmma slices per layer, accumulators in registers, last layer
// transposed so that the max over the K neighbours stays inside one quad of threads) with two changes:
//   * layer 0 (the raw [xyz_rel | feats] row, <= 16 channels) stays 3xTF32;
//   * every later layer splits its operands into TWO BF16 parts, x = x1 + x2 with x1 = bf16(x) and
//     x2 = bf16(x - x1) (16 mantissa bits kept), and issues three bf16 MMAs per K-step of 16
//     (x1*w1 + x2*w1 + x1*w2) into the fp32 accumulator: ~2^-17 relative error per product -- 60x
//     tighter than the TF32 the reference's own convolutions run in by default (SURVEY.md 7.1), inside
//     the 1e-4 bar (measured ~1e-5 end to end), at half the operand bytes and half the MMA count of 3xTF32;
//   * biases are added in the epilogue in fp32 (exact), not through an extra MMA.
// Two tile groups per CTA at 128 channels (operand tile 64 KB each, 80 KB of weights), four when the layers
// are narrow enough; persistent over tiles.  On narrow shapes the 3xTF32 engine is more accurate, so the dispatcher
// prefers it when it fits.
#include <cuda_bf16.h>

#include <algorithm>

#include "common.cuh"
#include "sa_mlp.cuh"
#include "tc_common.cuh"
#include "tgn_b200.h"

namespace tgn {
namespace {

using namespace tc;

constexpr int kRows = 128;
constexpr int kMaxGroups = 4;          // tile groups per CTA: 4 when the operand tiles are small enough, else 2
constexpr uint32_t kChunk = kRows * 16;               // bytes of one 16-byte K-chunk of all 128 rows (LBO of a 128-row operand)

struct WLayout {
    int kpad[kSaMaxLayers];          // K of layer l (layer 0: multiple of 8, 16 at most; later: multiple of 16)
    int npad[kSaMaxLayers];          // N of layer l, multiple of 16
    uint32_t w_hi[kSaMaxLayers], w_lo[kSaMaxLayers];   // byte offsets of the weight operands
    uint32_t act[kMaxGroups];        // per group operand buffer: [hi | lo], lo at act_lo_off
    int groups;
    uint32_t act_lo_off;
    uint32_t total;
    int tiles_per_cloud, gpt;
    uint32_t tpc_magic;
};

// (a, b) -> packed bf16 pair, a in the LOW half (the lower K index), round to nearest even
__device__ __forceinline__ uint32_t pack_bf16(float a, float b) {
    uint32_t r;
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(b), "f"(a));
    return r;
}
// x = x1 + x2 (two bf16 parts each) for a pair of values: hi word, lo word
__device__ __forceinline__ void split_bf16_pair(float a, float b, uint32_t& hi, uint32_t& lo) {
    hi = pack_bf16(a, b);
    const float a1 = __uint_as_float(hi << 16), b1 = __uint_as_float(hi & 0xFFFF0000u);
    lo = pack_bf16(__fsub_rn(a, a1), __fsub_rn(b, b1));
}
// One inner layer on one 64-row slice (rows 64h..64h+63) of a group's tile -- layer 0: 3xTF32 from the tf32 hi / lo
// operands at x_hi / a0_lo, K = 8 per MMA; later layers: three bf16 terms from x_hi / x_lo, K = 16 per MMA -- then + bias,
// ReLU, bf16 hi/lo split and 4-byte stores of the fragment pairs into the next layer's operand (the slice only
// overwrites its own rows, which no other slice reads).
template <int NP>
__device__ __forceinline__ void inner_layer(int h, bool first, int kp, uint32_t x_hi, uint32_t x_lo, uint32_t a0_lo, uint32_t w_hi,
                                            uint32_t w_lo, const float* __restrict__ bias, int cout, int g)
{
    const int lane = threadIdx.x & 31, w = (threadIdx.x >> 5) & 3;
    const uint32_t lbo_w = NP * 16, row_off = h * 64 * 16;
    uint64_t d_xh = make_smem_desc(x_hi + row_off, kChunk), d_xl = make_smem_desc((first ? a0_lo : x_lo) + row_off, kChunk);
    uint64_t d_wh = make_smem_desc(w_hi, lbo_w), d_wl = make_smem_desc(w_lo, lbo_w);
    float acc[NP / 2];
#pragma unroll
    for (int i = 0; i < NP / 2; ++i) acc[i] = 0.f;
    fence_regs(acc);
    wgmma_fence();
    if (first) {
        for (int ks = 0; ks < kp / 8; ++ks) {
            wgmma_tf32<NP>(acc, d_xh, d_wh, ks > 0);
            wgmma_tf32<NP>(acc, d_xl, d_wh, true);
            wgmma_tf32<NP>(acc, d_xh, d_wl, true);
            d_xh += desc_step(2 * kChunk); d_xl += desc_step(2 * kChunk); d_wh += desc_step(2 * lbo_w); d_wl += desc_step(2 * lbo_w);
        }
    } else {
        for (int ks = 0; ks < kp / 16; ++ks) {
            wgmma_bf16<NP>(acc, d_xh, d_wh, ks > 0);
            wgmma_bf16<NP>(acc, d_xl, d_wh, true);
            wgmma_bf16<NP>(acc, d_xh, d_wl, true);
            d_xh += desc_step(2 * kChunk); d_xl += desc_step(2 * kChunk); d_wh += desc_step(2 * lbo_w); d_wl += desc_step(2 * lbo_w);
        }
    }
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(acc);
    group_sync(g);                   // every warp's MMAs have read the operand before any row of it is overwritten
    const int row = h * 64 + w * 16 + (lane >> 2);
#pragma unroll
    for (int i = 0; i < NP / 8; ++i) {
        const int c = 8 * i + 2 * (lane & 3);
        const float b0 = c < cout ? __ldg(bias + c) : 0.f, b1 = c + 1 < cout ? __ldg(bias + c + 1) : 0.f;
        const uint32_t off = static_cast<uint32_t>(c >> 3) * kChunk + (c & 7) * 2;
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            uint32_t hi, lo;
            split_bf16_pair(fmaxf(acc[4 * i + 2 * e] + b0, 0.f), fmaxf(acc[4 * i + 2 * e + 1] + b1, 0.f), hi, lo);
            const uint32_t o = off + (row + 8 * e) * 16;
            st_shared_b32(x_hi + o, hi);
            st_shared_b32(x_lo + o, lo);
        }
    }
}

template <int kGroups>
__global__ void __launch_bounds__(kRows * kGroups, 1)
sa_mlp_tcw_kernel(const SaParams p, const WLayout lay)
{
    constexpr int kThreads = kRows * kGroups;
    extern __shared__ __align__(1024) uint8_t smem[];
    const uint32_t sbase = smem_u32(smem);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int g = tid / kRows;
    const int r = tid - g * kRows;

    // ---- weights, once per CTA -----------------------------------------------------------------------
    // layer 0: tf32 hi/lo B operand [np x 16] (LBO = np*16); inner layers: bf16 hi/lo B operand [np x kp]
    // (LBO = np*16); last layer: bf16 hi/lo A operand [128 x kp] (LBO = 128*16), zero rows beyond cout.
    for (int l = 0; l < p.L; ++l) {
        const int cin = p.ch[l], cout = p.ch[l + 1], kp = lay.kpad[l];
        const int rows_w = l == p.L - 1 ? kRows : lay.npad[l];
        for (int e = tid; e < rows_w * kp; e += kThreads) {
            const int n = e / kp, k = e - n * kp;
            const float w = (n < cout && k < cin) ? __ldg(p.W[l] + static_cast<size_t>(n) * cin + k) : 0.f;
            if (l == 0) {
                uint32_t hi, lo;
                split_tf32(w, hi, lo);
                const uint32_t off = static_cast<uint32_t>(k >> 2) * (rows_w * 16) + n * 16 + (k & 3) * 4;
                *reinterpret_cast<uint32_t*>(smem + lay.w_hi[l] + off) = hi;
                *reinterpret_cast<uint32_t*>(smem + lay.w_lo[l] + off) = lo;
            } else {
                const __nv_bfloat16 w1 = __float2bfloat16_rn(w);
                const __nv_bfloat16 w2 = __float2bfloat16_rn(w - __bfloat162float(w1));
                const uint32_t off = static_cast<uint32_t>(k >> 3) * (rows_w * 16) + n * 16 + (k & 7) * 2;
                *reinterpret_cast<__nv_bfloat16*>(smem + lay.w_hi[l] + off) = w1;
                *reinterpret_cast<__nv_bfloat16*>(smem + lay.w_lo[l] + off) = w2;
            }
        }
    }
    proxy_fence_async();
    __syncthreads();
    const uint32_t x_hi = sbase + lay.act[g], x_lo = x_hi + lay.act_lo_off;
    const uint32_t a0_lo = x_hi + 4 * kChunk;       // layer 0: four tf32 chunks of hi, then four of lo

    const int cout_last = p.ch[p.L];
    const int total_tiles = lay.tiles_per_cloud * p.B;
    const int tile_step = gridDim.x * kGroups;
    const int r_div_k = r / p.K;
    auto cloud_of = [&](int t) -> int {
        int q = static_cast<int>(__umulhi(static_cast<unsigned>(t), lay.tpc_magic));
        if (t - q * lay.tiles_per_cloud >= lay.tiles_per_cloud) ++q;
        return q;
    };
    auto load_index = [&](int t) -> int {
        if (t >= total_tiles) return -1;
        const int tb = cloud_of(t);
        const int ts0 = (t - tb * lay.tiles_per_cloud) * lay.gpt;
        if (r >= min(lay.gpt, p.S - ts0) * p.K) return -1;
        return __ldg(p.gidx + (static_cast<size_t>(tb) * p.S + ts0) * p.K + r);
    };
    auto load_row16 = [&](int t, int j, float (&out)[16]) {
#pragma unroll
        for (int c = 0; c < 16; ++c) out[c] = 0.f;
        if (t < total_tiles && j >= 0 && j < p.N) {
            const int tb = cloud_of(t);
            const int ts = (t - tb * lay.tiles_per_cloud) * lay.gpt + r_div_k;
            const float* px = p.xyz + 3 * (static_cast<size_t>(tb) * p.N + j);
            const float* pc = p.new_xyz + 3 * (static_cast<size_t>(tb) * p.S + ts);
            const float* pf = p.feats ? p.feats + (static_cast<size_t>(tb) * p.N + j) * p.D : px;
            const float rel0 = __fsub_rn(__ldg(px), __ldg(pc)), rel1 = __fsub_rn(__ldg(px + 1), __ldg(pc + 1)),
                        rel2 = __fsub_rn(__ldg(px + 2), __ldg(pc + 2));
            if (p.xyz_first) {
                out[0] = rel0; out[1] = rel1; out[2] = rel2;
#pragma unroll
                for (int i = 0; i < 13; ++i)
                    if (i < p.D) out[3 + i] = __ldg(pf + i);
            } else {
#pragma unroll
                for (int c = 0; c < 16; ++c) {
                    if (c < p.D) out[c] = __ldg(pf + c);
                    else if (c == p.D) out[c] = rel0;
                    else if (c == p.D + 1) out[c] = rel1;
                    else if (c == p.D + 2) out[c] = rel2;
                }
            }
        }
    };
    float row[16];
    int j_next;
    {
        const int t0 = blockIdx.x * kGroups + g;
        load_row16(t0, load_index(t0), row);
        j_next = load_index(t0 + tile_step);
    }

    for (int tile = blockIdx.x * kGroups + g; tile < total_tiles; tile += tile_step) {
        const int b = cloud_of(tile);
        const int s0 = (tile - b * lay.tiles_per_cloud) * lay.gpt;
        const int groups = min(lay.gpt, p.S - s0);
        const int rows = groups * p.K;

        // ---- layer-0 operand (tf32 hi/lo) from the row prefetched one tile ago ---------------------------------
#pragma unroll
        for (int kc = 0; kc < 4; ++kc) {
            uint32_t hi[4], lo[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) split_tf32(row[4 * kc + i], hi[i], lo[i]);
            const uint32_t off = kc * kChunk + r * 16;
            st_shared_v4(x_hi + off, hi[0], hi[1], hi[2], hi[3]);
            st_shared_v4(a0_lo + off, lo[0], lo[1], lo[2], lo[3]);
        }
        load_row16(tile + tile_step, j_next, row);
        j_next = load_index(tile + 2 * tile_step);

        for (int l = 0; l < p.L; ++l) {
            const int kp = lay.kpad[l], np = lay.npad[l];
            proxy_fence_async();
            group_sync(g);
            if (l < p.L - 1) {
                const uint32_t wh = sbase + lay.w_hi[l], wl = sbase + lay.w_lo[l];
                for (int h = 0; h < 2 && 64 * h < rows; ++h) {          // tile-uniform
                    switch (np) {
                        case 16: inner_layer<16>(h, l == 0, kp, x_hi, x_lo, a0_lo, wh, wl, p.bias[l], p.ch[l + 1], g); break;
                        case 32: inner_layer<32>(h, l == 0, kp, x_hi, x_lo, a0_lo, wh, wl, p.bias[l], p.ch[l + 1], g); break;
                        case 48: inner_layer<48>(h, l == 0, kp, x_hi, x_lo, a0_lo, wh, wl, p.bias[l], p.ch[l + 1], g); break;
                        case 64: inner_layer<64>(h, l == 0, kp, x_hi, x_lo, a0_lo, wh, wl, p.bias[l], p.ch[l + 1], g); break;
                        case 80: inner_layer<80>(h, l == 0, kp, x_hi, x_lo, a0_lo, wh, wl, p.bias[l], p.ch[l + 1], g); break;
                        case 96: inner_layer<96>(h, l == 0, kp, x_hi, x_lo, a0_lo, wh, wl, p.bias[l], p.ch[l + 1], g); break;
                        case 112: inner_layer<112>(h, l == 0, kp, x_hi, x_lo, a0_lo, wh, wl, p.bias[l], p.ch[l + 1], g); break;
                        default: inner_layer<128>(h, l == 0, kp, x_hi, x_lo, a0_lo, wh, wl, p.bias[l], p.ch[l + 1], g); break;
                    }
                }
            } else {
                // D^T[channel, row] += W[channel, k] * X[row, k], three bf16 terms, one 64-channel slice at a time
                float* ob = p.out + (static_cast<size_t>(b) * p.out_c_total + p.out_c_offset) * p.S;
                for (int hc = 0; 64 * hc < cout_last; ++hc) {
                    uint64_t d_wh = make_smem_desc(sbase + lay.w_hi[l] + hc * 64 * 16, kChunk);
                    uint64_t d_wl = make_smem_desc(sbase + lay.w_lo[l] + hc * 64 * 16, kChunk);
                    uint64_t d_xh = make_smem_desc(x_hi, kChunk), d_xl = make_smem_desc(x_lo, kChunk);
                    float acc[64];
#pragma unroll
                    for (int i = 0; i < 64; ++i) acc[i] = 0.f;
                    fence_regs(acc);
                    wgmma_fence();
                    for (int ks = 0; ks < kp / 16; ++ks) {
                        wgmma_bf16<128>(acc, d_wh, d_xh, ks > 0);
                        wgmma_bf16<128>(acc, d_wh, d_xl, true);
                        wgmma_bf16<128>(acc, d_wl, d_xh, true);
                        d_xh += desc_step(2 * kChunk); d_xl += desc_step(2 * kChunk); d_wh += desc_step(2 * kChunk); d_wl += desc_step(2 * kChunk);
                    }
                    wgmma_commit();
                    wgmma_wait<0>();
                    fence_regs(acc);
                    store_neighbourhood_max(acc, 64 * hc + 16 * (warp & 3) + (lane >> 2), cout_last, p.bias[l], ob, p.S, s0, p.K, groups);
                }
                group_sync(g);             // the next tile's first-layer stores overwrite the operand these MMAs read
            }
        }
    }
}

bool make_wlayout_groups(const SaParams& p, WLayout& lay, int kGroups)
{
    lay.groups = kGroups;
    if (p.L < 2 || p.L > kSaMaxLayers) return false;                       // one layer: the other engines
    if (!(p.K == 16 || p.K == 32 || p.K == 64 || p.K == 128)) return false;
    if (p.ch[0] > 16) return false;                                        // the gathered row is built in 16 registers
    uint32_t off = 0;
    auto take = [&off](uint32_t bytes, uint32_t align) {
        off = (off + align - 1) / align * align;
        const uint32_t o = off;
        off += bytes;
        return o;
    };
    int kmax = 0;
    for (int l = 0; l < p.L; ++l) {
        lay.npad[l] = (p.ch[l + 1] + 15) / 16 * 16;
        lay.kpad[l] = l == 0 ? 16 : lay.npad[l - 1];
        if (lay.npad[l] > 128) return false;
        if (l > 0) kmax = std::max(kmax, lay.kpad[l]);
    }
    // operand buffer of a group: bf16 hi then lo, kmax/8 chunks each; layer 0 needs 8 tf32 chunks in the same space
    const uint32_t half = std::max<uint32_t>(static_cast<uint32_t>(kmax / 8) * kChunk, 4 * kChunk);
    lay.act_lo_off = half;
    for (int g = 0; g < kGroups; ++g) lay.act[g] = take(2 * half, 1024);
    for (int l = 0; l < p.L; ++l) {
        const int rows_w = l == p.L - 1 ? kRows : lay.npad[l];
        const uint32_t wb = static_cast<uint32_t>(rows_w) * lay.kpad[l] * (l == 0 ? 4 : 2);
        lay.w_hi[l] = take(wb, 128);
        lay.w_lo[l] = take(wb, 128);
    }
    lay.total = off;
    lay.gpt = kRows / p.K;
    lay.tiles_per_cloud = (p.S + lay.gpt - 1) / lay.gpt;
    lay.tpc_magic = static_cast<uint32_t>(std::min<unsigned long long>((1ull << 32) / static_cast<unsigned long long>(lay.tiles_per_cloud), 0xFFFFFFFFull));
    return lay.total <= 224 * 1024;
}

// four tile groups when they fit (narrow layers), else two
bool make_wlayout(const SaParams& p, WLayout& lay)
{
    return make_wlayout_groups(p, lay, 4) || make_wlayout_groups(p, lay, 2);
}

template <int kGroups>
int launch_tcw(const SaParams& p, const WLayout& lay, cudaStream_t st)
{
    const int rc_attr = ensure_dynamic_smem(reinterpret_cast<const void*>(sa_mlp_tcw_kernel<kGroups>), lay.total);
    if (rc_attr != TGN_OK) return rc_attr;
    const long long tiles = static_cast<long long>(lay.tiles_per_cloud) * p.B;
    const int grid = static_cast<int>(std::min<long long>((tiles + kGroups - 1) / kGroups, sm_count()));
    sa_mlp_tcw_kernel<kGroups><<<grid, kRows * kGroups, lay.total, st>>>(p, lay);
    return check_launch("sa_mlp_tcw_kernel");
}

}  // namespace

bool sa_mlp_tcw_supported(const SaParams& p)
{
    WLayout lay{};
    return make_wlayout(p, lay);
}

int sa_mlp_tcw_launch(SaParams p, cudaStream_t st)
{
    WLayout lay{};
    if (!make_wlayout(p, lay)) { set_error("sa_group_mlp_max: shape not supported by the wide tensor-core engine"); return TGN_ERR_INVALID; }
    return lay.groups == 4 ? launch_tcw<4>(p, lay, st) : launch_tcw<2>(p, lay, st);
}

}  // namespace tgn
