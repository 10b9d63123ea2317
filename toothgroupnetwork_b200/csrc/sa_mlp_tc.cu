// sa_mlp_tc.cu -- warpgroup-MMA (wgmma) tensor-core engine of the fused set-abstraction body.
//
// Same contract as the fp32 engine in sa_mlp.cu, but the per-layer contraction
//      D[128 rows, N] = A[128 rows, K] * W[N, K]^T
// runs on the tensor cores with the accumulator in registers:
//   * a CTA is up to 4 independent TILE GROUPS of 128 threads (one warpgroup each); a group owns one 128-row tile
//     (128/K neighbourhoods) at a time.  Thread r of the group gathers row r's [xyz_rel | feats] row into the
//     first layer's operand; each layer then runs as two 64-row wgmma slices, and after each slice the threads
//     add the bias, apply ReLU and write the next layer's operand from their accumulator fragments -- the grouped
//     tensor and the inter-layer activations never leave the SM.  The groups share the weights but nothing else
//     (own operand buffers, named barriers instead of __syncthreads), so while one group waits for its gather or
//     its MMAs the others fill the issue slots and the tensor pipe;
//   * operands live in shared memory in the canonical K-major, no-swizzle layout (8x16-byte core matrices;
//     element (r,k) at (k/4)*LBO + r*16 + (k%4)*4 with SBO = 128 B);
//   * fp32 fidelity: inputs are split a = a_hi + a_lo with a_hi the tf32 truncation, and each K-step issues
//     three tf32 MMAs (hi*hi + lo*hi + hi*lo) into the same accumulator ("3xTF32"), so the result carries
//     ~2^-21 relative error instead of tf32's 2^-10 -- the reference's own default for these 1x1 convolutions is
//     plain TF32 (SURVEY.md 7.1);
//   * the LAST layer runs transposed, D^T[channel, row] = W[channel, K] * X[row, K]^T: the weights (zero-padded
//     to 128 channels) are the A operand and the activation tile is the B operand (N = 128 rows), so a thread's
//     accumulator fragment holds two channels across all rows of the tile; the max over the K rows of a
//     neighbourhood is a chain of max inside the thread plus two shuffles across its quad.
// Weights are split and laid out once per CTA; CTAs are persistent over tiles.
#include <algorithm>

#include "common.cuh"
#include "sa_mlp.cuh"
#include "tc_common.cuh"
#include "tgn_b200.h"

namespace tgn {
namespace {

using namespace tc;

constexpr int kRows = 128;                            // rows of a tile = threads of a tile group
constexpr int kMaxGroups = 4;                         // tile groups per CTA: 4 (one CTA owns the SM) or 2 (two CTAs per SM, or one
                                                      // beside another kernel's CTAs: 32K registers each)
constexpr uint32_t kChunkStrideA = kRows * 16;        // LBO of the A operand: one 16-byte K-chunk of all rows

struct TcLayout {
    int kpad[kSaMaxLayers];          // K of layer l, multiple of 8
    int npad[kSaMaxLayers];          // N of layer l, multiple of 16
    uint32_t w_hi[kSaMaxLayers], w_lo[kSaMaxLayers];   // byte offsets in dynamic smem
    uint32_t a_hi[kMaxGroups], a_lo[kMaxGroups];   // per group activation operands (A of the inner layers, B of the last)
    int groups;                      // tile groups per CTA
    uint32_t total;
    int tiles_per_cloud, gpt;
    uint32_t tpc_magic;              // floor(2^32 / tiles_per_cloud): t / tiles_per_cloud by IMAD.HI + one fix-up
};

// One inner layer on one 64-row slice (rows 64h..64h+63) of a group's tile: 3xTF32 MMAs, then + bias, ReLU, tf32 hi/lo
// split and 8-byte stores of the fragment pairs into the next layer's K-major operand (the same buffers: the slice
// only overwrites its own rows, which no other slice reads).
template <int NP>
__device__ __forceinline__ void inner_layer(int h, int kp, uint32_t a_hi, uint32_t a_lo, uint32_t w_hi, uint32_t w_lo,
                                            const float* __restrict__ bias, int cout, int g)
{
    const int lane = threadIdx.x & 31, w = (threadIdx.x >> 5) & 3;
    const uint32_t lbo_w = NP * 16;
    uint64_t d_xhi = make_smem_desc(a_hi + h * 64 * 16, kChunkStrideA), d_xlo = make_smem_desc(a_lo + h * 64 * 16, kChunkStrideA);
    uint64_t d_whi = make_smem_desc(w_hi, lbo_w), d_wlo = make_smem_desc(w_lo, lbo_w);
    float acc[NP / 2];
#pragma unroll
    for (int i = 0; i < NP / 2; ++i) acc[i] = 0.f;
    fence_regs(acc);
    wgmma_fence();
    for (int ks = 0; ks < kp / 8; ++ks) {
        wgmma_tf32<NP>(acc, d_xhi, d_whi, ks > 0);
        wgmma_tf32<NP>(acc, d_xlo, d_whi, true);
        wgmma_tf32<NP>(acc, d_xhi, d_wlo, true);
        d_xhi += desc_step(2 * kChunkStrideA); d_xlo += desc_step(2 * kChunkStrideA);
        d_whi += desc_step(2 * lbo_w); d_wlo += desc_step(2 * lbo_w);
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
        const uint32_t off = static_cast<uint32_t>(c >> 2) * kChunkStrideA + (c & 3) * 4;
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            uint32_t hi0, lo0, hi1, lo1;
            split_tf32(fmaxf(acc[4 * i + 2 * e] + b0, 0.f), hi0, lo0);
            split_tf32(fmaxf(acc[4 * i + 2 * e + 1] + b1, 0.f), hi1, lo1);
            const uint32_t o = off + (row + 8 * e) * 16;
            st_shared_v2(a_hi + o, hi0, hi1);
            st_shared_v2(a_lo + o, lo0, lo1);
        }
    }
}

template <int kGroups>
__global__ void __launch_bounds__(kRows * kGroups, 4 / kGroups)
sa_mlp_tc_kernel(const SaParams p, const TcLayout lay)
{
    constexpr int kThreads = kRows * kGroups;
    extern __shared__ __align__(1024) uint8_t smem[];
    const uint32_t sbase = smem_u32(smem);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int g = tid / kRows;                 // tile group
    const int r = tid - g * kRows;             // row inside the tile (inner layers) / output channel (last layer)
    // ---- weights: split into tf32 hi/lo, canonical K-major layout.  Inner layers: B operand
    //      [npad x kpad] (LBO = npad*16); last layer: A operand [128 x kpad] (LBO = 128*16), zero rows
    //      beyond cout.  SBO = 128 either way.  Biases are added in fp32 by the epilogues.
    for (int l = 0; l < p.L; ++l) {
        const int cin = p.ch[l], cout = p.ch[l + 1], kp = lay.kpad[l];
        const int np = l == p.L - 1 ? kRows : lay.npad[l];
        for (int e = tid; e < np * kp; e += kThreads) {
            const int n = e / kp, k = e - n * kp;
            const float w = (n < cout && k < cin) ? __ldg(p.W[l] + static_cast<size_t>(n) * cin + k) : 0.f;
            uint32_t hi, lo;
            split_tf32(w, hi, lo);
            const uint32_t off = static_cast<uint32_t>(k >> 2) * (np * 16) + n * 16 + (k & 3) * 4;
            *reinterpret_cast<uint32_t*>(smem + lay.w_hi[l] + off) = hi;
            *reinterpret_cast<uint32_t*>(smem + lay.w_lo[l] + off) = lo;
        }
    }
    proxy_fence_async();
    __syncthreads();
    const uint32_t a_hi = sbase + lay.a_hi[g], a_lo = sbase + lay.a_lo[g];

    const int cout_last = p.ch[p.L];
    const int total_tiles = lay.tiles_per_cloud * p.B;
    const int tile_step = gridDim.x * kGroups;
    const int xoff = p.xyz_first ? 0 : p.D;       // first channel of the xyz_rel block
    const int foff = p.xyz_first ? 3 : 0;         // first channel of the feature block
    const int r_div_k = r / p.K;                  // neighbourhood of this thread's row inside a tile
    // t / tiles_per_cloud without an integer division (magic = floor(2^32 / d) is off by at most one)
    auto cloud_of = [&](int t) -> int {
        int q = static_cast<int>(__umulhi(static_cast<unsigned>(t), lay.tpc_magic));
        if (t - q * lay.tiles_per_cloud >= lay.tiles_per_cloud) ++q;
        return q;
    };
    // neighbour index of this thread's row in tile `t` (-1 past the end / past the rows of the tile)
    auto load_index = [&](int t) -> int {
        if (t >= total_tiles) return -1;
        const int tb = cloud_of(t);
        const int ts0 = (t - tb * lay.tiles_per_cloud) * lay.gpt;
        if (r >= min(lay.gpt, p.S - ts0) * p.K) return -1;
        return __ldg(p.gidx + (static_cast<size_t>(tb) * p.S + ts0) * p.K + r);
    };
    // the 16-wide zero-padded [xyz_rel | feats] (or [feats | xyz_rel]) row of this thread in tile `t`
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
    const bool fast_rows = lay.kpad[0] == 16;     // the whole padded input row fits 16 registers
    float row[16];
    int j_next;
    {
        const int t0 = blockIdx.x * kGroups + g;
        if (fast_rows) {
            load_row16(t0, load_index(t0), row);
            j_next = load_index(t0 + tile_step);
        } else {
#pragma unroll
            for (int c = 0; c < 16; ++c) row[c] = 0.f;
            j_next = load_index(t0);
        }
    }

    for (int tile = blockIdx.x * kGroups + g; tile < total_tiles; tile += tile_step) {
        const int b = cloud_of(tile);
        const int s0 = (tile - b * lay.tiles_per_cloud) * lay.gpt;
        const int groups = min(lay.gpt, p.S - s0);
        const int rows = groups * p.K;

        // ---- layer-0 operand: this thread's grouped row --------------------------------------------
        if (fast_rows) {
            // the 16-wide padded row was loaded into registers while the previous tile computed
#pragma unroll
            for (int kc = 0; kc < 4; ++kc) {
                uint32_t hi[4], lo[4];
#pragma unroll
                for (int i = 0; i < 4; ++i) split_tf32(row[4 * kc + i], hi[i], lo[i]);
                const uint32_t off = kc * kChunkStrideA + r * 16;
                st_shared_v4(a_hi + off, hi[0], hi[1], hi[2], hi[3]);
                st_shared_v4(a_lo + off, lo[0], lo[1], lo[2], lo[3]);
            }
            load_row16(tile + tile_step, j_next, row);          // consumed one tile later: latency hidden
            j_next = load_index(tile + 2 * tile_step);
        } else {
            int j = j_next;                               // index prefetched while the previous tile computed
            const int s = s0 + (r < rows ? r_div_k : 0);
            if (r >= rows || j < 0 || j >= p.N) j = -1;
            const int jj = j < 0 ? 0 : j;
            const float* px = p.xyz + 3 * (static_cast<size_t>(b) * p.N + jj);
            const float* pc = p.new_xyz + 3 * (static_cast<size_t>(b) * p.S + s);
            const float* pf = p.feats ? p.feats + (static_cast<size_t>(b) * p.N + jj) * p.D : px;
            const float rel0 = __fsub_rn(__ldg(px), __ldg(pc)), rel1 = __fsub_rn(__ldg(px + 1), __ldg(pc + 1)),
                        rel2 = __fsub_rn(__ldg(px + 2), __ldg(pc + 2));
            for (int kc = 0; kc < lay.kpad[0] / 4; ++kc) {
                uint32_t hi[4], lo[4];
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const int c = 4 * kc + i;
                    const int xc = c - xoff;
                    float v = xc == 0 ? rel0 : (xc == 1 ? rel1 : rel2);
                    if (static_cast<unsigned>(xc) > 2u) {
                        const unsigned fc = static_cast<unsigned>(c - foff);
                        v = fc < static_cast<unsigned>(p.D) ? __ldg(pf + fc) : 0.f;
                    }
                    if (j < 0) v = 0.f;
                    split_tf32(v, hi[i], lo[i]);
                }
                const uint32_t off = kc * kChunkStrideA + r * 16;
                st_shared_v4(a_hi + off, hi[0], hi[1], hi[2], hi[3]);
                st_shared_v4(a_lo + off, lo[0], lo[1], lo[2], lo[3]);
            }
            j_next = load_index(tile + tile_step);
        }

        for (int l = 0; l < p.L; ++l) {
            const int kp = lay.kpad[l], np = lay.npad[l];
            proxy_fence_async();           // this thread's operand stores -> visible to the tensor core
            group_sync(g);
            if (l < p.L - 1) {
                const uint32_t whi = sbase + lay.w_hi[l], wlo = sbase + lay.w_lo[l];
                for (int h = 0; h < 2 && 64 * h < rows; ++h) {          // tile-uniform
                    switch (np) {
                        case 16: inner_layer<16>(h, kp, a_hi, a_lo, whi, wlo, p.bias[l], p.ch[l + 1], g); break;
                        case 32: inner_layer<32>(h, kp, a_hi, a_lo, whi, wlo, p.bias[l], p.ch[l + 1], g); break;
                        case 48: inner_layer<48>(h, kp, a_hi, a_lo, whi, wlo, p.bias[l], p.ch[l + 1], g); break;
                        case 64: inner_layer<64>(h, kp, a_hi, a_lo, whi, wlo, p.bias[l], p.ch[l + 1], g); break;
                        case 80: inner_layer<80>(h, kp, a_hi, a_lo, whi, wlo, p.bias[l], p.ch[l + 1], g); break;
                        case 96: inner_layer<96>(h, kp, a_hi, a_lo, whi, wlo, p.bias[l], p.ch[l + 1], g); break;
                        case 112: inner_layer<112>(h, kp, a_hi, a_lo, whi, wlo, p.bias[l], p.ch[l + 1], g); break;
                        default: inner_layer<128>(h, kp, a_hi, a_lo, whi, wlo, p.bias[l], p.ch[l + 1], g); break;
                    }
                }
            } else {
                // D^T[channel, row] += W[channel, k] * X[row, k], one 64-channel slice at a time
                float* ob = p.out + (static_cast<size_t>(b) * p.out_c_total + p.out_c_offset) * p.S;
                for (int hc = 0; 64 * hc < cout_last; ++hc) {
                    uint64_t d_whi = make_smem_desc(sbase + lay.w_hi[l] + hc * 64 * 16, kChunkStrideA);
                    uint64_t d_wlo = make_smem_desc(sbase + lay.w_lo[l] + hc * 64 * 16, kChunkStrideA);
                    uint64_t d_xhi = make_smem_desc(a_hi, kChunkStrideA), d_xlo = make_smem_desc(a_lo, kChunkStrideA);
                    float acc[64];
#pragma unroll
                    for (int i = 0; i < 64; ++i) acc[i] = 0.f;
                    fence_regs(acc);
                    wgmma_fence();
                    for (int ks = 0; ks < kp / 8; ++ks) {
                        wgmma_tf32<128>(acc, d_whi, d_xhi, ks > 0);
                        wgmma_tf32<128>(acc, d_whi, d_xlo, true);
                        wgmma_tf32<128>(acc, d_wlo, d_xhi, true);
                        d_xhi += desc_step(2 * kChunkStrideA); d_xlo += desc_step(2 * kChunkStrideA);
                        d_whi += desc_step(2 * kChunkStrideA); d_wlo += desc_step(2 * kChunkStrideA);
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

bool make_layout(const SaParams& p, TcLayout& lay, int kGroups = kMaxGroups)
{
    lay.groups = kGroups;
    if (p.K > kRows || p.K < 1) return false;
    int kmax = 0;
    uint32_t off = 0;
    auto take = [&off](uint32_t bytes, uint32_t align) {
        off = (off + align - 1) / align * align;
        const uint32_t o = off;
        off += bytes;
        return o;
    };
    for (int l = 0; l < p.L; ++l) {
        lay.kpad[l] = l == 0 ? (p.ch[0] + 7) / 8 * 8 : lay.npad[l - 1];
        lay.npad[l] = (p.ch[l + 1] + 15) / 16 * 16;
        if (lay.npad[l] > 128 || lay.kpad[l] > 128) return false;
        kmax = std::max(kmax, lay.kpad[l]);
    }
    const uint32_t a_bytes = static_cast<uint32_t>(kmax / 4) * kChunkStrideA;
    for (int g = 0; g < kGroups; ++g) {
        lay.a_hi[g] = take(a_bytes, 128);
        lay.a_lo[g] = take(a_bytes, 128);
    }
    for (int l = 0; l < p.L; ++l) {
        const int rows_w = l == p.L - 1 ? kRows : lay.npad[l];      // the last layer's weights are a 128-row A operand
        const uint32_t wb = static_cast<uint32_t>(rows_w) * lay.kpad[l] * 4;
        lay.w_hi[l] = take(wb, 128);
        lay.w_lo[l] = take(wb, 128);
    }
    lay.total = off;
    lay.gpt = kRows / p.K;
    lay.tiles_per_cloud = (p.S + lay.gpt - 1) / lay.gpt;
    lay.tpc_magic = static_cast<uint32_t>(std::min<unsigned long long>((1ull << 32) / static_cast<unsigned long long>(lay.tiles_per_cloud), 0xFFFFFFFFull));
    return lay.total <= 220u * 1024;
}

}  // namespace

bool sa_mlp_tc_supported(const SaParams& p)
{
    TcLayout lay{};
    return make_layout(p, lay, kMaxGroups) || make_layout(p, lay, 2);
}

template <int kGroups>
int launch_tc(const SaParams& p, const TcLayout& lay, cudaStream_t st)
{
    const int rc_attr = ensure_dynamic_smem(reinterpret_cast<const void*>(sa_mlp_tc_kernel<kGroups>), lay.total);
    if (rc_attr != TGN_OK) return rc_attr;
    // persistent CTAs: one of 4 tile groups per SM, or two of 2 groups
    const long long tiles = static_cast<long long>(lay.tiles_per_cloud) * p.B;
    const int grid = static_cast<int>(std::min<long long>((tiles + kGroups - 1) / kGroups, static_cast<long long>(sm_count()) * (kMaxGroups / kGroups)));
    sa_mlp_tc_kernel<kGroups><<<grid, kRows * kGroups, lay.total, st>>>(p, lay);
    return check_launch("sa_mlp_tc_kernel");
}

// groups_per_cta: 4 = one CTA owns the SM (all 64K registers); 2 = half-size CTAs (32K registers) that can share an SM with
// the CTAs of another stream's kernels -- the host pipeline keeps the FPS of the
// next chunk resident, and a full-size CTA would wait for it to drain.  (Two half CTAs fit one SM only when the operand
// tiles are small; with the bench shape the weights of the 128-row last layer make it one per SM.)
int sa_mlp_tc_launch(SaParams p, cudaStream_t st, int groups_per_cta)
{
    TcLayout lay{};
    if (groups_per_cta == 2 && make_layout(p, lay, 2)) return launch_tc<2>(p, lay, st);
    if (!make_layout(p, lay, kMaxGroups)) {
        if (make_layout(p, lay, 2)) return launch_tc<2>(p, lay, st);       // operand tiles too large for four groups
        set_error("sa_group_mlp_max: shape not supported by the tensor-core engine");
        return TGN_ERR_INVALID;
    }
    return launch_tc<kMaxGroups>(p, lay, st);
}

}  // namespace tgn
