// sa_mlp_tc.cu -- warpgroup-MMA (wgmma) tensor-core engine of the fused set-abstraction body.
//
// Same contract as the fp32 engine in sa_mlp.cu, but every layer's contraction runs on the tensor cores TRANSPOSED,
//      D^T[channel, row] = W[channel, K] * X[row, K]^T,
// with the weights as the A operand (channels on M), the activation tile as the B operand (N = the 128 rows of a
// tile) and the accumulator in registers: one m64n128k8 wgmma does the work of four m64n32k8 ones of the row-major
// form, so a layer is a few wide MMAs instead of many narrow ones, and the fixed issue and completion latency of
// each MMA is spread over 4x the work.
//   * a CTA is up to 4 independent TILE GROUPS of 128 threads (one warpgroup each); a group owns one 128-row tile
//     (128/K neighbourhoods) at a time.  Thread r of the group gathers row r's [xyz_rel | feats] row into the
//     first layer's operand (the row of the NEXT tile is loaded into registers while this one computes); each
//     inner layer's epilogue adds the bias, applies ReLU and writes the next layer's operand from its
//     channel-major accumulator fragments -- the grouped tensor and the inter-layer activations never leave the
//     SM.  The groups share the weights but nothing else (own operand buffers, named barriers instead of
//     __syncthreads), so while one group waits for its gather, its MMAs or its epilogue the others fill the issue
//     slots and the tensor pipe.  Every wgmma sits in control flow that is uniform over the warpgroup (the group
//     index comes out of a shuffle, loop bounds out of the kernel parameters); partial tiles run on zero rows and
//     drop them at the store;
//   * fp32 fidelity: inputs are split a = a_hi + a_lo with a_hi the tf32 truncation, and each K-step issues
//     tf32 MMAs for hi*hi + lo*hi + hi*lo ("3xTF32"), so the result carries ~2^-21 relative error instead of
//     tf32's 2^-10 -- the reference's own default for these 1x1 convolutions is plain TF32 (SURVEY.md 7.1);
//   * the inner (hidden) layers all run at one padded width NP (16/32/48/64, a template parameter) with
//     zero-padded weights and biases, on M = 64 weight rows.  Up to 32 channels the rows are PACKED: rows
//     16w..16w+7 hold W_hi of channels 8w..8w+7 and rows 16w+8..16w+15 their W_lo, so one MMA against X_hi yields
//     hi*hi and lo*hi of a channel in the same thread, and a second against X_lo with the W_lo rows zero adds
//     hi*lo: two m64n128k8 per K-step instead of three on a half-empty M.  Wider layers run one channel per row,
//     three MMAs per K-step;
//   * operands live in shared memory in the canonical K-major, no-swizzle layout (8x16-byte core matrices;
//     element (r,k) at (k/4)*LBO + r*16 + (k%4)*4 with SBO = 128 B).  The activation tile's LBO is 128*16 + 16
//     bytes: an epilogue's 4-byte stores of one warp (8 channels x 4 rows) then fall in 32 distinct banks;
//   * the LAST layer's weights are zero-padded to 64 or 128 channels and run 64 channels at a time, so a thread's
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
constexpr int kInnerM = 64;                           // weight rows (M) of an inner layer's MMA
constexpr uint32_t kActChunk = kRows * 16 + 16;       // LBO of the activation tile: one 16-byte K-chunk of all rows + 16
                                                      // bytes, so that the epilogue's stores do not collide in banks

struct TcLayout {
    int kpad[kSaMaxLayers];          // K of layer l: 3 + D rounded up to 8, then the previous layer's width rounded up to 16
    int np;                          // padded width of every inner layer (the kernel's template width)
    int last_rows;                   // weight rows of the last layer: its width rounded up to 64
    uint32_t w_a[kSaMaxLayers], w_b[kSaMaxLayers];     // byte offsets in dynamic smem of layer l's two A operands
    uint32_t bias;                   // inner layers' biases, np floats each, zero-padded
    uint32_t a_hi[kMaxGroups], a_lo[kMaxGroups];   // per group activation tile (B operand of every layer), hi / lo
    int groups;                      // tile groups per CTA
    uint32_t total;
    int tiles_per_cloud, gpt;
    uint32_t tpc_magic;              // floor(2^32 / tiles_per_cloud): t / tiles_per_cloud by IMAD.HI + one fix-up
};

// Inner layers of width <= 32 pack W_hi and W_lo of a channel into one 64-row A operand (file comment).
template <int NP>
constexpr bool kPacked = NP <= 32;

// Issue the 3xTF32 MMAs of one inner layer on a group's whole tile as one wgmma group: acc = W[64, 0..kp) *
// X[128 rows, 0..kp)^T.  The first MMA writes acc without reading it, so acc is not cleared.
template <int NP>
__device__ __forceinline__ void issue_inner(float (&acc)[64], int kp, uint32_t x_hi, uint32_t x_lo, uint32_t w_a, uint32_t w_b)
{
    constexpr uint32_t lbo_w = kInnerM * 16;
    uint64_t d_xhi = make_smem_desc(x_hi, kActChunk), d_xlo = make_smem_desc(x_lo, kActChunk);
    uint64_t d_wa = make_smem_desc(w_a, lbo_w), d_wb = make_smem_desc(w_b, lbo_w);
    auto rest = [&] {
        if (kPacked<NP>) {
            wgmma_tf32<128>(acc, d_wb, d_xlo, true);            // [W_hi | 0] * X_lo
        } else {
            wgmma_tf32<128>(acc, d_wa, d_xlo, true);            // W_hi * X_lo
            wgmma_tf32<128>(acc, d_wb, d_xhi, true);            // W_lo * X_hi
        }
    };
    wgmma_fence();
    wgmma_tf32_zero<128>(acc, d_wa, d_xhi);
    rest();
    for (int ks = 1; ks < kp / 8; ++ks) {
        d_xhi += desc_step(2 * kActChunk); d_xlo += desc_step(2 * kActChunk);
        d_wa += desc_step(2 * lbo_w); d_wb += desc_step(2 * lbo_w);
        wgmma_tf32<128>(acc, d_wa, d_xhi, true);
        rest();
    }
    wgmma_commit();
}

// Epilogue of a finished inner layer: + bias, ReLU, tf32 hi/lo split and 4-byte stores of the thread's channels
// across the tile's rows into the next layer's K-major operand (the same buffers, rewritten after every warp's MMAs
// have read them).  Channels from NP on are never read, so the warps that hold only those store nothing.
template <int NP>
__device__ __forceinline__ void store_inner(const float (&acc)[64], uint32_t x_hi, uint32_t x_lo, const float* bias)
{
    const int lane = threadIdx.x & 31, w = (threadIdx.x >> 5) & 3;
    const int r0 = 2 * (lane & 3);                 // the thread's rows: 8i + r0 + e
    auto put = [&](float v, uint32_t o) {
        uint32_t hi, lo;
        split_tf32(fmaxf(v, 0.f), hi, lo);
        st_shared_b32(x_hi + o, hi);
        st_shared_b32(x_lo + o, lo);
    };
    if (kPacked<NP>) {
        // rows 16w + lane/4 (hi*hi + hi*lo) and 16w + 8 + lane/4 (lo*hi) of D^T are the parts of channel 8w + lane/4
        if (8 * w >= NP) return;
        const int c = 8 * w + (lane >> 2);
        const float b = bias[c];
        const uint32_t off = static_cast<uint32_t>(c >> 2) * kActChunk + (c & 3) * 4 + r0 * 16;
#pragma unroll
        for (int i = 0; i < 16; ++i)
#pragma unroll
            for (int e = 0; e < 2; ++e) put((acc[4 * i + e] + acc[4 * i + 2 + e]) + b, off + (8 * i + e) * 16);
    } else {
        // rows 16w + lane/4 and 16w + 8 + lane/4 of D^T are channels c and c + 8
        if (16 * w >= NP) return;
        const bool second = 16 * w + 8 < NP;
        const int c = 16 * w + (lane >> 2);
        const float b0 = bias[c], b1 = second ? bias[c + 8] : 0.f;
        const uint32_t off0 = static_cast<uint32_t>(c >> 2) * kActChunk + (c & 3) * 4 + r0 * 16;
        const uint32_t off1 = off0 + 2 * kActChunk;
#pragma unroll
        for (int i = 0; i < 16; ++i)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                put(acc[4 * i + e] + b0, off0 + (8 * i + e) * 16);
                if (second) put(acc[4 * i + 2 + e] + b1, off1 + (8 * i + e) * 16);
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
    const int r = tid - g * kRows;             // row of the tile this thread gathers
    // ---- weights: split into tf32 hi/lo, canonical K-major A operands [M x kpad] (LBO = M*16, SBO = 128): M = 64
    //      for the inner layers (packed or one channel per row, see the file comment), 64 or 128 for the last layer
    //      (w_a = W_hi, w_b = W_lo).  Zero rows beyond cout.  Biases are added in fp32 by the epilogues.
    float* bias_s = reinterpret_cast<float*>(smem + lay.bias);
    for (int l = 0; l < p.L; ++l) {
        const int cin = p.ch[l], cout = p.ch[l + 1], kp = lay.kpad[l];
        const bool inner = l < p.L - 1, packed = inner && kPacked<NP>;
        const int m_rows = inner ? kInnerM : lay.last_rows;
        for (int e = tid; e < m_rows * kp; e += kThreads) {
            const int m = e / kp, k = e - m * kp;
            const int n = packed ? (m >> 4) * 8 + (m & 7) : m;          // channel of weight row m
            const bool lo_row = packed && (m & 8);
            const float w = (n < cout && k < cin) ? __ldg(p.W[l] + static_cast<size_t>(n) * cin + k) : 0.f;
            uint32_t hi, lo;
            split_tf32(w, hi, lo);
            const uint32_t off = static_cast<uint32_t>(k >> 2) * (m_rows * 16) + m * 16 + (k & 3) * 4;
            *reinterpret_cast<uint32_t*>(smem + lay.w_a[l] + off) = lo_row ? lo : hi;
            *reinterpret_cast<uint32_t*>(smem + lay.w_b[l] + off) = packed ? (lo_row ? 0u : hi) : lo;
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
            const uint32_t off = kc * kActChunk + r * 16;
            st_shared_v4(a_hi + off, hi[0], hi[1], hi[2], hi[3]);
            st_shared_v4(a_lo + off, lo[0], lo[1], lo[2], lo[3]);
        }
        load_row16(tile + tile_step, j_next, row);          // consumed one tile later: latency hidden
        j_next = load_index(tile + 2 * tile_step);
        proxy_fence_async();               // this thread's operand stores -> visible to the tensor core
        group_sync(g);

        // ---- inner layers: the whole tile's MMAs as one group, then the epilogue rewrites the operand in place
        for (int l = 0; l < n_inner; ++l) {
            float acc[64];
            issue_inner<NP>(acc, lay.kpad[l], a_hi, a_lo, sbase + lay.w_a[l], sbase + lay.w_b[l]);
            wgmma_wait<0>();
            fence_regs(acc);
            group_sync(g);                 // every warp's MMAs have read the tile before any of it is overwritten
            store_inner<NP>(acc, a_hi, a_lo, bias_s + l * NP);
            proxy_fence_async();
            group_sync(g);
        }

        // ---- last layer: D^T[channel, row] += W[channel, k] * X[row, k], one 64-channel slice at a time
        const int l = p.L - 1, kp = lay.kpad[l];
        float* ob = p.out + (static_cast<size_t>(b) * p.out_c_total + p.out_c_offset) * p.S;
        const uint32_t lbo_w = lay.last_rows * 16;
        for (int hc = 0; 64 * hc < cout_last; ++hc) {
            uint64_t d_whi = make_smem_desc(sbase + lay.w_a[l] + hc * 64 * 16, lbo_w);
            uint64_t d_wlo = make_smem_desc(sbase + lay.w_b[l] + hc * 64 * 16, lbo_w);
            uint64_t d_xhi = make_smem_desc(a_hi, kActChunk), d_xlo = make_smem_desc(a_lo, kActChunk);
            float acc[64];
#pragma unroll
            for (int i = 0; i < 64; ++i) acc[i] = 0.f;
            fence_regs(acc);
            wgmma_fence();
            for (int ks = 0; ks < kp / 8; ++ks) {
                wgmma_tf32<128>(acc, d_whi, d_xhi, ks > 0);
                wgmma_tf32<128>(acc, d_whi, d_xlo, true);
                wgmma_tf32<128>(acc, d_wlo, d_xhi, true);
                d_xhi += desc_step(2 * kActChunk); d_xlo += desc_step(2 * kActChunk);
                d_whi += desc_step(2 * lbo_w); d_wlo += desc_step(2 * lbo_w);
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
    lay.last_rows = (p.ch[p.L] + 63) / 64 * 64;
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
    const uint32_t a_bytes = static_cast<uint32_t>(kmax / 4) * kActChunk;
    for (int g = 0; g < kGroups; ++g) {
        lay.a_hi[g] = take(a_bytes, 128);
        lay.a_lo[g] = take(a_bytes, 128);
    }
    for (int l = 0; l < p.L; ++l) {
        const int rows_w = l == p.L - 1 ? lay.last_rows : kInnerM;
        const uint32_t wb = static_cast<uint32_t>(rows_w) * lay.kpad[l] * 4;
        lay.w_a[l] = take(wb, 128);
        lay.w_b[l] = take(wb, 128);
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
// tiles are small: with the bench shape each takes 105 KB of shared memory, so two do.)
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
