// sa_mlp_tc.cu -- warpgroup-MMA (wgmma) tensor-core engine of the fused set-abstraction body.
//
// Same contract as the fp32 engine in sa_mlp.cu, but the per-layer contraction
//      D[128 rows, N] = A[128 rows, K] * W[N, K]^T
// runs on the tensor cores with the accumulator in registers:
//   * a CTA is up to 4 independent TILE GROUPS of 128 threads (one warpgroup each); a group owns one 128-row tile
//     (128/K neighbourhoods) at a time.  Thread r of the group gathers row r's [xyz_rel | feats] row into the
//     first layer's operand (the row of the NEXT tile is loaded into registers while this one computes); every
//     layer then runs as two 64-row wgmma slices, and each slice's epilogue adds the bias, applies ReLU and writes
//     the next layer's operand from its accumulator fragments -- the grouped tensor and the inter-layer
//     activations never leave the SM.  The groups share the weights but nothing else (own operand buffers, named
//     barriers instead of __syncthreads), so while one group waits for its gather or its MMAs the others fill the
//     issue slots and the tensor pipe;
//   * inside a group the slices are software-pipelined as one chain (0,0) (0,1) (1,0) (1,1) ...: each slice's
//     epilogue runs while the next slice's MMAs are in flight (slice h of layer l+1 only needs slice h of layer l,
//     so it is issued as soon as that epilogue is stored).  Every wgmma sits in control flow that is uniform over
//     the warpgroup (the group index comes out of a shuffle, loop bounds out of the kernel parameters); partial
//     tiles run both slices on zero rows and drop them at the store;
//   * the inner (hidden) layers all run at one padded width NP (16/32/48/64, a template parameter) with
//     zero-padded weights and biases, so the accumulators are fixed-size arrays and the kernel does not spill;
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
constexpr int kInCols = 16;                           // the gathered input row, zero-padded: 3 + D <= 16
constexpr uint32_t kChunkStrideA = kRows * 16;        // LBO of the A operand: one 16-byte K-chunk of all rows

struct TcLayout {
    int kpad[kSaMaxLayers];          // K of layer l: 3 + D rounded up to 8, then the previous layer's width rounded up to 16
    int np;                          // N of every inner layer (the kernel's template width)
    uint32_t w_hi[kSaMaxLayers], w_lo[kSaMaxLayers];   // byte offsets in dynamic smem
    uint32_t bias;                   // inner layers' biases, np floats each, zero-padded
    uint32_t a_hi[kMaxGroups], a_lo[kMaxGroups];   // per group activation operands (A of the inner layers, B of the last)
    int groups;                      // tile groups per CTA
    uint32_t total;
    int tiles_per_cloud, gpt;
    uint32_t tpc_magic;              // floor(2^32 / tiles_per_cloud): t / tiles_per_cloud by IMAD.HI + one fix-up
};

// Issue the 3xTF32 MMAs of one inner layer on one 64-row slice (rows 64h..64h+63) of a group's tile as one wgmma group:
// acc = X[rows, 0..kp) * W[NP, 0..kp)^T.  The first MMA writes acc without reading it, so acc is not cleared: an
// instruction that wrote it while the other slice's MMAs are in flight would make the compiler serialise them.
template <int NP>
__device__ __forceinline__ void issue_slice(float (&acc)[NP / 2], int h, int kp, uint32_t a_hi, uint32_t a_lo, uint32_t w_hi,
                                            uint32_t w_lo)
{
    constexpr uint32_t lbo_w = NP * 16;
    uint64_t d_xhi = make_smem_desc(a_hi + h * 64 * 16, kChunkStrideA), d_xlo = make_smem_desc(a_lo + h * 64 * 16, kChunkStrideA);
    uint64_t d_whi = make_smem_desc(w_hi, lbo_w), d_wlo = make_smem_desc(w_lo, lbo_w);
    wgmma_fence();
    wgmma_tf32_zero<NP>(acc, d_xhi, d_whi);
    wgmma_tf32<NP>(acc, d_xlo, d_whi, true);
    wgmma_tf32<NP>(acc, d_xhi, d_wlo, true);
    for (int ks = 1; ks < kp / 8; ++ks) {
        d_xhi += desc_step(2 * kChunkStrideA); d_xlo += desc_step(2 * kChunkStrideA);
        d_whi += desc_step(2 * lbo_w); d_wlo += desc_step(2 * lbo_w);
        wgmma_tf32<NP>(acc, d_xhi, d_whi, true);
        wgmma_tf32<NP>(acc, d_xlo, d_whi, true);
        wgmma_tf32<NP>(acc, d_xhi, d_wlo, true);
    }
    wgmma_commit();
}

// Epilogue of one finished slice: + bias, ReLU, tf32 hi/lo split and 8-byte stores of the fragment pairs into the next
// layer's K-major operand (the same buffers: the slice only overwrites its own rows, which no other slice reads).
template <int NP>
__device__ __forceinline__ void store_slice(const float (&acc)[NP / 2], int h, uint32_t a_hi, uint32_t a_lo, const float* bias)
{
    const int lane = threadIdx.x & 31, w = (threadIdx.x >> 5) & 3;
    const int row = h * 64 + w * 16 + (lane >> 2);
#pragma unroll
    for (int i = 0; i < NP / 8; ++i) {
        const int c = 8 * i + 2 * (lane & 3);
        const float b0 = bias[c], b1 = bias[c + 1];
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

template <int kGroups, int NP>
__global__ void __launch_bounds__(kRows * kGroups, 4 / kGroups)
sa_mlp_tc_kernel(const SaParams p, const TcLayout lay)
{
    constexpr int kThreads = kRows * kGroups;
    extern __shared__ __align__(1024) uint8_t smem[];
    const uint32_t sbase = smem_u32(smem);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    // tile group, read through a shuffle so that the compiler sees it (and everything derived from it: the tile
    // loop, every wgmma) as warp-uniform -- otherwise it serialises the asynchronous MMAs
    const int g = __shfl_sync(0xffffffffu, tid / kRows, 0);
    const int r = tid - g * kRows;             // row inside the tile (inner layers) / output channel (last layer)
    // ---- weights: split into tf32 hi/lo, canonical K-major layout.  Inner layers: B operand
    //      [NP x kpad] (LBO = NP*16); last layer: A operand [128 x kpad] (LBO = 128*16).  Zero rows
    //      beyond cout.  SBO = 128 either way.  Biases are added in fp32 by the epilogues.
    float* bias_s = reinterpret_cast<float*>(smem + lay.bias);
    for (int l = 0; l < p.L; ++l) {
        const int cin = p.ch[l], cout = p.ch[l + 1], kp = lay.kpad[l];
        const int np = l == p.L - 1 ? kRows : NP;
        for (int e = tid; e < np * kp; e += kThreads) {
            const int n = e / kp, k = e - n * kp;
            const float w = (n < cout && k < cin) ? __ldg(p.W[l] + static_cast<size_t>(n) * cin + k) : 0.f;
            uint32_t hi, lo;
            split_tf32(w, hi, lo);
            const uint32_t off = static_cast<uint32_t>(k >> 2) * (np * 16) + n * 16 + (k & 3) * 4;
            *reinterpret_cast<uint32_t*>(smem + lay.w_hi[l] + off) = hi;
            *reinterpret_cast<uint32_t*>(smem + lay.w_lo[l] + off) = lo;
        }
        if (l < p.L - 1)
            for (int c = tid; c < NP; c += kThreads) bias_s[l * NP + c] = c < cout ? __ldg(p.bias[l] + c) : 0.f;
    }
    proxy_fence_async();
    __syncthreads();
    const uint32_t a_hi = sbase + lay.a_hi[g], a_lo = sbase + lay.a_lo[g];

    const int n_inner = p.L - 1;
    const int cout_last = p.ch[p.L];
    const int total_tiles = lay.tiles_per_cloud * p.B;
    const int tile_step = gridDim.x * kGroups;
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
    auto load_row16 = [&](int t, int j, float (&out)[kInCols]) {
#pragma unroll
        for (int c = 0; c < kInCols; ++c) out[c] = 0.f;
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
                for (int i = 0; i < kInCols - 3; ++i)
                    if (i < p.D) out[3 + i] = __ldg(pf + i);
            } else {
#pragma unroll
                for (int c = 0; c < kInCols; ++c) {
                    if (c < p.D) out[c] = __ldg(pf + c);
                    else if (c == p.D) out[c] = rel0;
                    else if (c == p.D + 1) out[c] = rel1;
                    else if (c == p.D + 2) out[c] = rel2;
                }
            }
        }
    };
    float row[kInCols];
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

        // ---- layer-0 operand: this thread's grouped row, loaded into registers while the previous tile computed
#pragma unroll
        for (int kc = 0; kc < kInCols / 4; ++kc) {
            uint32_t hi[4], lo[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) split_tf32(row[4 * kc + i], hi[i], lo[i]);
            const uint32_t off = kc * kChunkStrideA + r * 16;
            st_shared_v4(a_hi + off, hi[0], hi[1], hi[2], hi[3]);
            st_shared_v4(a_lo + off, lo[0], lo[1], lo[2], lo[3]);
        }
        load_row16(tile + tile_step, j_next, row);          // consumed one tile later: latency hidden
        j_next = load_index(tile + 2 * tile_step);
        proxy_fence_async();               // this thread's operand stores -> visible to the tensor core
        group_sync(g);

        // ---- inner layers: each slice's epilogue runs under the MMAs of the next slice in the chain
        //      (l,0) (l,1) (l+1,0) (l+1,1) ...; slice h of layer l+1 only needs slice h of layer l.  Every epilogue
        //      follows a wait for ALL issued MMAs and the next slice is issued after it: the compiler serialises
        //      the MMAs when an accumulator is read while a group issued before it is still open, or when the
        //      open groups differ between paths (hence the last inner layer is peeled).
        if (n_inner > 0) {
            float acc0[NP / 2], acc1[NP / 2];
            auto finish = [&](const float (&acc)[NP / 2], int h, int l) {
                group_sync(g);             // every warp's MMAs have read the slice's rows before any of them is overwritten
                store_slice<NP>(acc, h, a_hi, a_lo, bias_s + l * NP);
                proxy_fence_async();
                group_sync(g);
            };
            issue_slice<NP>(acc0, 0, lay.kpad[0], a_hi, a_lo, sbase + lay.w_hi[0], sbase + lay.w_lo[0]);
            int l = 0;
            for (; l < n_inner - 1; ++l) {
                const uint32_t whi = sbase + lay.w_hi[l], wlo = sbase + lay.w_lo[l];
                wgmma_wait<0>();
                fence_regs(acc0);
                issue_slice<NP>(acc1, 1, lay.kpad[l], a_hi, a_lo, whi, wlo);
                finish(acc0, 0, l);
                wgmma_wait<0>();
                fence_regs(acc1);
                issue_slice<NP>(acc0, 0, lay.kpad[l + 1], a_hi, a_lo, sbase + lay.w_hi[l + 1], sbase + lay.w_lo[l + 1]);
                finish(acc1, 1, l);
            }
            wgmma_wait<0>();
            fence_regs(acc0);
            issue_slice<NP>(acc1, 1, lay.kpad[l], a_hi, a_lo, sbase + lay.w_hi[l], sbase + lay.w_lo[l]);
            finish(acc0, 0, l);
            wgmma_wait<0>();
            fence_regs(acc1);
            finish(acc1, 1, l);
        }

        // ---- last layer: D^T[channel, row] += W[channel, k] * X[row, k], one 64-channel slice at a time
        const int l = p.L - 1, kp = lay.kpad[l];
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
        group_sync(g);                     // the next tile's first-layer stores overwrite the operand these MMAs read
    }
}

// Inner layers run at the narrowest of 16/32/48/64 that holds every hidden width; 0 when one is wider.
int inner_width(const SaParams& p)
{
    int w = 16;
    for (int l = 1; l < p.L; ++l) w = std::max(w, (p.ch[l] + 15) / 16 * 16);
    return w <= 64 ? w : 0;
}

bool make_layout(const SaParams& p, TcLayout& lay, int kGroups = kMaxGroups)
{
    lay.groups = kGroups;
    if (p.K > kRows || p.K < 1) return false;
    if (p.ch[0] > kInCols) return false;                 // the gathered row is built in 16 registers
    lay.np = inner_width(p);
    if (lay.np == 0) return false;
    int kmax = kInCols;
    uint32_t off = 0;
    auto take = [&off](uint32_t bytes, uint32_t align) {
        off = (off + align - 1) / align * align;
        const uint32_t o = off;
        off += bytes;
        return o;
    };
    for (int l = 0; l < p.L; ++l) {
        lay.kpad[l] = l == 0 ? (p.ch[0] + 7) / 8 * 8 : (p.ch[l] + 15) / 16 * 16;
        kmax = std::max(kmax, lay.kpad[l]);
    }
    kmax = std::max(kmax, p.L > 1 ? lay.np : 0);       // the inner layers' epilogues write np columns
    const uint32_t a_bytes = static_cast<uint32_t>(kmax / 4) * kChunkStrideA;
    for (int g = 0; g < kGroups; ++g) {
        lay.a_hi[g] = take(a_bytes, 128);
        lay.a_lo[g] = take(a_bytes, 128);
    }
    for (int l = 0; l < p.L; ++l) {
        const int rows_w = l == p.L - 1 ? kRows : lay.np;      // the last layer's weights are a 128-row A operand
        const uint32_t wb = static_cast<uint32_t>(rows_w) * lay.kpad[l] * 4;
        lay.w_hi[l] = take(wb, 128);
        lay.w_lo[l] = take(wb, 128);
    }
    lay.bias = take(static_cast<uint32_t>(std::max(p.L - 1, 1) * lay.np) * 4, 16);
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

template <int kGroups, int NP>
int launch_tc_np(const SaParams& p, const TcLayout& lay, cudaStream_t st)
{
    const int rc_attr = ensure_dynamic_smem(reinterpret_cast<const void*>(sa_mlp_tc_kernel<kGroups, NP>), lay.total);
    if (rc_attr != TGN_OK) return rc_attr;
    // persistent CTAs: one of 4 tile groups per SM, or two of 2 groups
    const long long tiles = static_cast<long long>(lay.tiles_per_cloud) * p.B;
    const int grid = static_cast<int>(std::min<long long>((tiles + kGroups - 1) / kGroups, static_cast<long long>(sm_count()) * (kMaxGroups / kGroups)));
    sa_mlp_tc_kernel<kGroups, NP><<<grid, kRows * kGroups, lay.total, st>>>(p, lay);
    return check_launch("sa_mlp_tc_kernel");
}

template <int kGroups>
int launch_tc(const SaParams& p, const TcLayout& lay, cudaStream_t st)
{
    switch (lay.np) {
        case 16: return launch_tc_np<kGroups, 16>(p, lay, st);
        case 32: return launch_tc_np<kGroups, 32>(p, lay, st);
        case 48: return launch_tc_np<kGroups, 48>(p, lay, st);
        default: return launch_tc_np<kGroups, 64>(p, lay, st);
    }
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
