// sa_mlp_tc.cu -- warpgroup-MMA (wgmma) tensor-core engine of the fused set-abstraction body (engines 2 and 5).
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
//   * fp32 fidelity, split fp16: inputs are split a = a_hi + a_lo' * 2^-11 with a_hi = fp16(a) and a_lo' = fp16((a - a_hi)
//     * 2^11), so the pair carries ~22 bits; each K-step of 16 issues f16 MMAs (m64n128k16) for hi*hi + lo'*hi + hi*lo', the
//     dropped lo*lo term is ~2^-22 of the product, and the result stays inside the 3xTF32 engine's bound (DESIGN.md 3.3).  The
//     reference's own default for these 1x1 convolutions is plain TF32 (SURVEY.md 7.1);
//   * range guard, per tile: a layer-0 input or inner activation that is non-finite, at least 2^15 in magnitude, or (where
//     the consuming layer's biases do not cover the absolute error of tiny operands) nonzero below 2^-14 flags its tile, and
//     a weight out of range flags every tile.  The flags ride on the group barriers the schedule already has (bar.red.or),
//     so they are known before the last layer: a flagged tile writes nothing and is appended to a device list, which
//     sa_mlp_tc3_kernel -- the previous 3xTF32 kernel ("3xTF32": tf32 hi/lo, hi*hi + lo*hi + hi*lo) -- runs in a second
//     launch on the same stream.  That launch exits at once when the list is empty.  A tile never straddles two clouds,
//     so a cloud's result depends on that cloud alone;
//   * the inner (hidden) layers all run at one padded width NP (16/32/48/64, a template parameter) with
//     zero-padded weights and biases, on M = 64 weight rows.  Up to 32 channels the rows are PACKED: rows
//     16w..16w+7 hold W_hi of channels 8w..8w+7 and rows 16w+8..16w+15 their W_lo', so one MMA against X_hi yields
//     hi*hi (hi rows) and lo'*hi (lo rows) of a channel in the same thread, and a second, [0 ; W_hi] against X_lo',
//     adds hi*lo' into the lo rows; the epilogue takes hi + 2^-11 lo: two MMAs per K-step instead of three on a
//     half-empty M.  Wider layers and the last layer run one channel per row with one accumulator, (2^11 W_hi) X_hi
//     + W_lo' X_hi + W_hi X_lo' (three MMAs per K-step, 2^11 times the product; the epilogue scales it back exactly);
//   * operands live in shared memory in the canonical K-major, no-swizzle layout (8x16-byte core matrices; fp16
//     element (r,k) at (k/8)*LBO + r*16 + (k%8)*2 with SBO = 128 B; tf32 (k/4)*LBO + r*16 + (k%4)*4).  The inner
//     epilogue writes the packed f16x2 fragments with stmatrix.trans, 8 rows of 16 contiguous bytes per matrix (no bank
//     conflicts); the activation tile's LBO is 128*16 + 16 bytes, so the fallback's 4-byte stores of one warp (8
//     channels x 4 rows) fall in 32 distinct banks;
//   * the LAST layer's weights are zero-padded to 64 or 128 channels and run 64 channels at a time, so a thread's
//     accumulator fragment holds two channels across all rows of the tile; the max over the K rows of a
//     neighbourhood is a chain of max inside the thread plus two shuffles across its quad.
// Weights are split and laid out once per CTA; CTAs are persistent over tiles.
#include <algorithm>

#include <cuda_fp16.h>

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
    uint32_t w_a[kSaMaxLayers], w_b[kSaMaxLayers];     // byte offsets in dynamic smem of layer l's A operands: two (3xTF32,
    uint32_t w_c[kSaMaxLayers];                        // packed fp16) or three (fp16 one channel per row)
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

// The 3xTF32 fallback: runs the tiles the split-fp16 kernel listed (list[0] = count, then tile ids) and nothing else.
template <int kGroups, int NP>
__global__ void __launch_bounds__(kRows * kGroups, 4 / kGroups)
sa_mlp_tc3_kernel(const SaParams p, const TcLayout lay, const int* __restrict__ list)
{
    // read through a shuffle so that the tile loop's bound is seen as warp-uniform (see g below)
    const int count = __shfl_sync(0xffffffffu, __ldg(list), 0);
    if (count == 0) return;
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
    // tile id of list entry i (total_tiles, i.e. no tile, past the end)
    auto tile_at = [&](int i) -> int { return i < count ? __ldg(list + 1 + i) : total_tiles; };
    float row[kInCols];
    int j_next;
    {
        const int i0 = blockIdx.x * kGroups + g;
        load_row16(tile_at(i0), load_index(tile_at(i0)), row);
        j_next = load_index(tile_at(i0 + tile_step));
    }

    for (int i = blockIdx.x * kGroups + g; i < count; i += tile_step) {
        const int tile = tile_at(i);
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
        load_row16(tile_at(i + tile_step), j_next, row);          // consumed one tile later: latency hidden
        j_next = load_index(tile_at(i + 2 * tile_step));
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

// ---------------------------------------------------------------------------------------------- split-fp16 engine
// a = hi + lo' * 2^-11 with hi = fp16(a) and lo' = fp16((a - hi) * 2^11): a - hi is exact in fp32, and the power-of-two scale
// keeps lo' out of fp16's subnormal range wherever |a| >= 2^-3 (DESIGN.md 3.3 has the error bound, tiny |a| included)
__device__ __forceinline__ void split_f16(float a, uint32_t& hi, uint32_t& lo)
{
    const __half h = __float2half_rn(a);
    hi = __half_as_ushort(h);
    lo = __half_as_ushort(__float2half_rn(__fmul_rn(__fsub_rn(a, __half2float(h)), 2048.f)));
}
// split_f16 of two values at once, packed as f16x2 (a0 in the low half): one cvt.rn.f16x2.f32 per part, bit for bit the same
__device__ __forceinline__ void split_f16x2(float a0, float a1, uint32_t& hi, uint32_t& lo)
{
    const __half2 h = __floats2half2_rn(a0, a1);
    const float2 hf = __half22float2(h);
    const __half2 l = __floats2half2_rn(__fmul_rn(__fsub_rn(a0, hf.x), 2048.f), __fmul_rn(__fsub_rn(a1, hf.y), 2048.f));
    hi = *reinterpret_cast<const uint32_t*>(&h);
    lo = *reinterpret_cast<const uint32_t*>(&l);
}
// an operand the split cannot carry within the engine's bound: non-finite, |v| >= 2^15, or -- only where the consuming
// layer's biases do not cover the absolute error of tiny operands -- nonzero below fp16's normal range
__device__ __forceinline__ bool f16_out_of_range(float v, bool tiny_bad)
{
    const float a = fabsf(v);
    return !(a < 32768.f) || (tiny_bad && a != 0.f && a < 0x1p-14f);
}
// bar.sync of tile group g that also returns the OR of `v` over its 128 threads
__device__ __forceinline__ bool group_sync_or(int g, bool v)
{
    uint32_t out;
    asm volatile("{\n\t.reg .pred p, q;\n\tsetp.ne.u32 q, %1, 0;\n\tbar.red.or.pred p, %2, %3, q;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(out) : "r"(static_cast<uint32_t>(v)), "r"(g + 1), "r"(kRows) : "memory");
    return out != 0;
}
// four 8x8 b16 matrices, each stored transposed: lane l's register j holds (row l/4, columns 2(l%4), +1) of matrix j, and
// lanes 8j..8j+7 give the addresses of the stored matrix j's rows (= the register matrix's columns)
__device__ __forceinline__ void stmatrix_x4_trans(uint32_t addr, const uint32_t (&v)[4])
{
    asm volatile("stmatrix.sync.aligned.m8n8.x4.trans.shared.b16 [%0], {%1, %2, %3, %4};"
                 ::"r"(addr), "r"(v[0]), "r"(v[1]), "r"(v[2]), "r"(v[3]) : "memory");
}

// The split-fp16 MMAs of one inner layer on a group's whole tile, K = 16 per instruction.  Packed (NP <= 32):
// [W_hi ; W_lo'] * X_hi, then [0 ; W_hi] * X_lo', so the hi rows hold hi*hi and the lo rows lo'*hi + hi*lo'.  One channel
// per row: (2^11 W_hi) * X_hi + W_lo' * X_hi + W_hi * X_lo' in one accumulator, 2^11 times the product.
template <int NP>
__device__ __forceinline__ void issue_inner16(float (&acc)[64], int kp, uint32_t x_hi, uint32_t x_lo, uint32_t w_a, uint32_t w_b,
                                              uint32_t w_c)
{
    constexpr uint32_t lbo_w = kInnerM * 16;
    uint64_t d_xhi = make_smem_desc(x_hi, kActChunk), d_xlo = make_smem_desc(x_lo, kActChunk);
    uint64_t d_wa = make_smem_desc(w_a, lbo_w), d_wb = make_smem_desc(w_b, lbo_w), d_wc = make_smem_desc(w_c, lbo_w);
    auto rest = [&] {
        if (kPacked<NP>) {
            wgmma_f16<128>(acc, d_wb, d_xlo, true);             // [0 ; W_hi] * X_lo'
        } else {
            wgmma_f16<128>(acc, d_wb, d_xhi, true);             // W_lo' * X_hi
            wgmma_f16<128>(acc, d_wc, d_xlo, true);             // W_hi * X_lo'
        }
    };
    wgmma_fence();
    wgmma_f16_zero<128>(acc, d_wa, d_xhi);
    rest();
    for (int ks = 1; ks < kp / 16; ++ks) {
        d_xhi += desc_step(2 * kActChunk); d_xlo += desc_step(2 * kActChunk);
        d_wa += desc_step(2 * lbo_w); d_wb += desc_step(2 * lbo_w); d_wc += desc_step(2 * lbo_w);
        wgmma_f16<128>(acc, d_wa, d_xhi, true);
        rest();
    }
    wgmma_commit();
}

// Epilogue of a finished inner layer: y = hi part + 2^-11 lo part + bias, ReLU, fp16 hi/lo' split, and stmatrix.trans of
// the packed f16x2 pairs into the next layer's K-major operand (each 8x8 matrix is 8 rows of 16 contiguous bytes: no bank
// conflicts).  Returns whether any value is out of the split's range.
// The ReLU's fmaxf turns NaN into 0, so a value is out of range exactly when it is >= 2^15 (+Inf included): one running
// max covers the whole epilogue.  kTiny (the next layer's biases do not cover tiny operands) adds the per-value test.
template <int NP, bool kTiny>
__device__ __forceinline__ bool store_inner16(const float (&acc)[64], uint32_t x_hi, uint32_t x_lo, const float* bias)
{
    const int lane = threadIdx.x & 31, w = (threadIdx.x >> 5) & 3;
    float vmax = 0.f;
    bool tiny = false;
    auto pair = [&](float y0, float y1, uint32_t& hi, uint32_t& lo) {
        y0 = fmaxf(y0, 0.f);
        y1 = fmaxf(y1, 0.f);
        vmax = fmaxf(vmax, fmaxf(y0, y1));
        if (kTiny) tiny |= (y0 != 0.f && y0 < 0x1p-14f) | (y1 != 0.f && y1 < 0x1p-14f);
        split_f16x2(y0, y1, hi, lo);
    };
    const uint32_t row_off = static_cast<uint32_t>(8 * (lane >> 3) + (lane & 7)) * 16;     // stmatrix row of this lane
    if (kPacked<NP>) {
        // rows 16w + lane/4 (hi*hi) and 16w + 8 + lane/4 (lo'*hi + hi*lo') of D^T are the parts of channel 8w + lane/4
        if (8 * w >= NP) return false;
        const float b = bias[8 * w + (lane >> 2)];
        const uint32_t base = static_cast<uint32_t>(w) * kActChunk + row_off;
#pragma unroll
        for (int q = 0; q < 4; ++q) {                       // 8-row blocks 4q..4q+3 of the tile
            uint32_t hi[4], lo[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int i = 4 * q + j;
                pair(fmaf(acc[4 * i + 2], 0x1p-11f, acc[4 * i]) + b, fmaf(acc[4 * i + 3], 0x1p-11f, acc[4 * i + 1]) + b, hi[j], lo[j]);
            }
            stmatrix_x4_trans(x_hi + base + q * 512, hi);
            stmatrix_x4_trans(x_lo + base + q * 512, lo);
        }
    } else {
        // rows 16w + lane/4 and 16w + 8 + lane/4 of D^T are channels c and c + 8, each 2^11 times its product
        if (16 * w >= NP) return false;
        const bool second = 16 * w + 8 < NP;
        const int c = 16 * w + (lane >> 2);
        const float b0 = bias[c], b1 = second ? bias[c + 8] : 0.f;
        const uint32_t base0 = static_cast<uint32_t>(2 * w) * kActChunk + row_off;
        // one 8-channel K-chunk at a time (accumulator entries 4i + a0, +1): fewer live registers than both at once
        auto chunk = [&](int a0, float bb, uint32_t base) {
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                uint32_t hi[4], lo[4];
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const int i = 4 * q + j;
                    pair(fmaf(acc[4 * i + a0], 0x1p-11f, bb), fmaf(acc[4 * i + a0 + 1], 0x1p-11f, bb), hi[j], lo[j]);
                }
                stmatrix_x4_trans(x_hi + base + q * 512, hi);
                stmatrix_x4_trans(x_lo + base + q * 512, lo);
            }
        };
        chunk(0, b0, base0);
        if (second) chunk(2, b1, base0 + kActChunk);
    }
    return !(vmax < 32768.f) || tiny;
}

// Split-fp16 engine: the schedule of the 3xTF32 kernel above with fp16 operands.  A tile whose operands leave the split's
// range writes nothing and is appended to `list` (list[0] = count) for sa_mlp_tc3_kernel, launched next on the stream.
template <int kGroups, int NP>
__global__ void __launch_bounds__(kRows * kGroups, 4 / kGroups)
sa_mlp_tc_kernel(const SaParams p, const TcLayout lay, int* __restrict__ list)
{
    constexpr int kThreads = kRows * kGroups;
    extern __shared__ __align__(1024) uint8_t smem[];
    __shared__ int range_state;        // bit 0: a weight out of range (every tile falls back); bit 1 + l: see below
    const uint32_t sbase = smem_u32(smem);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int g = __shfl_sync(0xffffffffu, tid / kRows, 0);      // warp-uniform, as in the 3xTF32 kernel
    const int r = tid - g * kRows;
    if (tid == 0) range_state = 0;
    __syncthreads();
    // ---- weights: fp16 hi/lo' split, canonical K-major A operands [M x kpad] of 2-byte elements (element (m, k) at
    //      (k/8)*M*16 + m*16 + (k%8)*2).  Packed inner layers: w_a = [W_hi ; W_lo'], w_b = [0 ; W_hi] per 16 rows.  One
    //      channel per row (wide inner layers, the last layer): w_a = 2^11 W_hi, w_b = W_lo', w_c = W_hi.
    float* bias_s = reinterpret_cast<float*>(smem + lay.bias);
    int state = 0;
    for (int l = 0; l < p.L; ++l) {
        const int cin = p.ch[l], cout = p.ch[l + 1], kp = lay.kpad[l];
        const bool inner = l < p.L - 1, packed = inner && kPacked<NP>;
        const int m_rows = inner ? kInnerM : lay.last_rows;
        for (int e = tid; e < m_rows * kp; e += kThreads) {
            const int m = e / kp, k = e - m * kp;
            const int n = packed ? (m >> 4) * 8 + (m & 7) : m;
            const bool lo_row = packed && (m & 8);
            const float w = (n < cout && k < cin) ? __ldg(p.W[l] + static_cast<size_t>(n) * cin + k) : 0.f;
            const float aw = fabsf(w);
            if (!(aw < 16.f) || (aw != 0.f && aw < 0x1p-16f)) state |= 1;      // 2^11 W_hi stays finite in fp16
            uint32_t hi, lo;
            split_f16(w, hi, lo);
            const uint32_t off = static_cast<uint32_t>(k >> 3) * (m_rows * 16) + m * 16 + (k & 7) * 2;
            if (packed) {
                *reinterpret_cast<uint16_t*>(smem + lay.w_a[l] + off) = static_cast<uint16_t>(lo_row ? lo : hi);
                *reinterpret_cast<uint16_t*>(smem + lay.w_b[l] + off) = static_cast<uint16_t>(lo_row ? hi : 0u);
            } else {
                const float hs = __half2float(__ushort_as_half(static_cast<unsigned short>(hi))) * 2048.f;     // exact
                *reinterpret_cast<uint16_t*>(smem + lay.w_a[l] + off) = __half_as_ushort(__float2half_rn(hs));
                *reinterpret_cast<uint16_t*>(smem + lay.w_b[l] + off) = static_cast<uint16_t>(lo);
                *reinterpret_cast<uint16_t*>(smem + lay.w_c[l] + off) = static_cast<uint16_t>(hi);
            }
        }
        // bit 1 + l: some channel's bias is below 2^-11 |W_c|_1, so layer l's operands must not be tiny (DESIGN.md 3.3)
        for (int c = tid; c < cout; c += kThreads) {
            float s = 0.f;
            for (int k = 0; k < cin; ++k) s += fabsf(__ldg(p.W[l] + static_cast<size_t>(c) * cin + k));
            if (!(fabsf(__ldg(p.bias[l] + c)) >= 0x1p-11f * s)) state |= 2 << l;
        }
        if (inner)
            for (int c = tid; c < NP; c += kThreads) bias_s[l * NP + c] = c < cout ? __ldg(p.bias[l] + c) : 0.f;
    }
    if (state) atomicOr(&range_state, state);
    proxy_fence_async();
    __syncthreads();
    const int range = range_state;
    const uint32_t a_hi = sbase + lay.a_hi[g], a_lo = sbase + lay.a_lo[g];

    const int n_inner = p.L - 1;
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

        // ---- layer-0 operand: 16 fp16 hi and 16 lo' of this thread's row, two 16-byte K-chunks each
        bool bad = range & 1;
#pragma unroll
        for (int kc = 0; kc < kInCols / 8; ++kc) {
            uint32_t hi[4], lo[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const float v0 = row[8 * kc + 2 * i], v1 = row[8 * kc + 2 * i + 1];
                bad |= f16_out_of_range(v0, range & 2) | f16_out_of_range(v1, range & 2);
                split_f16x2(v0, v1, hi[i], lo[i]);
            }
            const uint32_t off = kc * kActChunk + r * 16;
            st_shared_v4(a_hi + off, hi[0], hi[1], hi[2], hi[3]);
            st_shared_v4(a_lo + off, lo[0], lo[1], lo[2], lo[3]);
        }
        load_row16(tile + tile_step, j_next, row);
        j_next = load_index(tile + 2 * tile_step);
        proxy_fence_async();
        // the group's flag rides on the barrier; read back through a shuffle so that the wgmma below stay warp-uniform
        bool flagged = __shfl_sync(0xffffffffu, static_cast<int>(group_sync_or(g, bad)), 0) != 0;

        // ---- inner layers, as in the 3xTF32 kernel; each epilogue's range flag rides on its closing barrier
        for (int l = 0; l < n_inner && !flagged; ++l) {
            float acc[64];
            issue_inner16<NP>(acc, lay.kpad[l], a_hi, a_lo, sbase + lay.w_a[l], sbase + lay.w_b[l], sbase + lay.w_c[l]);
            wgmma_wait<0>();
            fence_regs(acc);
            group_sync(g);
            const bool out_bad = (range >> (l + 2)) & 1 ? store_inner16<NP, true>(acc, a_hi, a_lo, bias_s + l * NP)
                                                        : store_inner16<NP, false>(acc, a_hi, a_lo, bias_s + l * NP);
            proxy_fence_async();
            flagged = __shfl_sync(0xffffffffu, static_cast<int>(group_sync_or(g, out_bad)), 0) != 0;
        }

        if (flagged) {
            // every flag is known before the last layer: this tile writes nothing here, the 3xTF32 kernel computes it
            if (r == 0) list[1 + atomicAdd(list, 1)] = tile;
        } else {
            // ---- last layer: (2^11 W_hi) X_hi + W_lo' X_hi + W_hi X_lo', one 64-channel slice at a time
            const int l = p.L - 1, kp = lay.kpad[l];
            float* ob = p.out + (static_cast<size_t>(b) * p.out_c_total + p.out_c_offset) * p.S;
            const uint32_t lbo_w = lay.last_rows * 16;
            for (int hc = 0; 64 * hc < cout_last; ++hc) {
                uint64_t d_wa = make_smem_desc(sbase + lay.w_a[l] + hc * 64 * 16, lbo_w);
                uint64_t d_wb = make_smem_desc(sbase + lay.w_b[l] + hc * 64 * 16, lbo_w);
                uint64_t d_wc = make_smem_desc(sbase + lay.w_c[l] + hc * 64 * 16, lbo_w);
                uint64_t d_xhi = make_smem_desc(a_hi, kActChunk), d_xlo = make_smem_desc(a_lo, kActChunk);
                float acc[64];
                wgmma_fence();
                wgmma_f16_zero<128>(acc, d_wa, d_xhi);
                wgmma_f16<128>(acc, d_wb, d_xhi, true);
                wgmma_f16<128>(acc, d_wc, d_xlo, true);
                for (int ks = 1; ks < kp / 16; ++ks) {
                    d_xhi += desc_step(2 * kActChunk); d_xlo += desc_step(2 * kActChunk);
                    d_wa += desc_step(2 * lbo_w); d_wb += desc_step(2 * lbo_w); d_wc += desc_step(2 * lbo_w);
                    wgmma_f16<128>(acc, d_wa, d_xhi, true);
                    wgmma_f16<128>(acc, d_wb, d_xhi, true);
                    wgmma_f16<128>(acc, d_wc, d_xlo, true);
                }
                wgmma_commit();
                wgmma_wait<0>();
                fence_regs(acc);
                // max, then the exact 2^-11 and the bias
                store_neighbourhood_max(acc, 64 * hc + 16 * (warp & 3) + (lane >> 2), cout_last, p.bias[l], ob, p.S, s0, p.K, groups,
                                        0x1p-11f);
            }
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

// f16: the split-fp16 kernel's layout (2-byte operands, K-chunks of 8, layer 0 padded to K = 16); otherwise the 3xTF32
// fallback's, which also decides whether the engine takes a shape at all (it is the larger of the two)
bool make_layout(const SaParams& p, TcLayout& lay, int kGroups, bool f16)
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
        lay.kpad[l] = l == 0 && !f16 ? (p.ch[0] + 7) / 8 * 8 : (p.ch[l] + 15) / 16 * 16;
        kmax = std::max(kmax, lay.kpad[l]);
    }
    kmax = std::max(kmax, p.L > 1 ? lay.np : 0);       // the inner layers' epilogues write np columns
    const int esize = f16 ? 2 : 4;
    const uint32_t a_bytes = static_cast<uint32_t>(kmax * esize / 16) * kActChunk;
    for (int g = 0; g < kGroups; ++g) {
        lay.a_hi[g] = take(a_bytes, 128);
        lay.a_lo[g] = take(a_bytes, 128);
    }
    for (int l = 0; l < p.L; ++l) {
        const int rows_w = l == p.L - 1 ? lay.last_rows : kInnerM;
        const uint32_t wb = static_cast<uint32_t>(rows_w) * lay.kpad[l] * esize;
        lay.w_a[l] = take(wb, 128);
        lay.w_b[l] = take(wb, 128);
        lay.w_c[l] = f16 && !(l < p.L - 1 && lay.np <= 32) ? take(wb, 128) : 0;
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
    return make_layout(p, lay, kMaxGroups, false) || make_layout(p, lay, 2, false);
}

template <int kGroups, int NP>
int launch_tc_np(const SaParams& p, const TcLayout& lay, const TcLayout& lay3, cudaStream_t st)
{
    int rc = ensure_dynamic_smem(reinterpret_cast<const void*>(sa_mlp_tc_kernel<kGroups, NP>), lay.total);
    if (rc != TGN_OK) return rc;
    rc = ensure_dynamic_smem(reinterpret_cast<const void*>(sa_mlp_tc3_kernel<kGroups, NP>), lay3.total);
    if (rc != TGN_OK) return rc;
    // persistent CTAs: one of 4 tile groups per SM, or two of 2 groups
    const long long tiles = static_cast<long long>(lay.tiles_per_cloud) * p.B;
    const int grid = static_cast<int>(std::min<long long>((tiles + kGroups - 1) / kGroups, static_cast<long long>(sm_count()) * (kMaxGroups / kGroups)));
    // the tiles the fp16 kernel leaves to the 3xTF32 one: a count and their ids, stream-ordered
    keep_async_pool();
    int* list = nullptr;
    cudaError_t e = cudaMallocAsync(reinterpret_cast<void**>(&list), static_cast<size_t>(tiles + 1) * sizeof(int), st);
    if (e == cudaSuccess) e = cudaMemsetAsync(list, 0, sizeof(int), st);
    if (e != cudaSuccess) {
        set_error("sa_group_mlp_max: fallback tile list: %s", cudaGetErrorString(e));
        (void)cudaGetLastError();
        if (list) (void)cudaFreeAsync(list, st);
        return TGN_ERR_CUDA;
    }
    sa_mlp_tc_kernel<kGroups, NP><<<grid, kRows * kGroups, lay.total, st>>>(p, lay, list);
    rc = check_launch("sa_mlp_tc_kernel");
    if (rc == TGN_OK) {
        sa_mlp_tc3_kernel<kGroups, NP><<<grid, kRows * kGroups, lay3.total, st>>>(p, lay3, list);
        rc = check_launch("sa_mlp_tc3_kernel");
    }
    (void)cudaFreeAsync(list, st);
    return rc;
}

template <int kGroups>
int launch_tc(const SaParams& p, cudaStream_t st)
{
    TcLayout lay{}, lay3{};
    make_layout(p, lay3, kGroups, false);
    make_layout(p, lay, kGroups, true);       // fits wherever the 3xTF32 layout does: every operand is half the bytes
    switch (lay.np) {
        case 16: return launch_tc_np<kGroups, 16>(p, lay, lay3, st);
        case 32: return launch_tc_np<kGroups, 32>(p, lay, lay3, st);
        case 48: return launch_tc_np<kGroups, 48>(p, lay, lay3, st);
        default: return launch_tc_np<kGroups, 64>(p, lay, lay3, st);
    }
}

// groups_per_cta: 4 = one CTA owns the SM (all 64K registers); 2 = half-size CTAs (32K registers) that can share an SM with
// the CTAs of another stream's kernels -- the host pipeline keeps the FPS of the
// next chunk resident, and a full-size CTA would wait for it to drain.  (Two half CTAs fit one SM only when the operand
// tiles are small: with the bench shape each takes 105 KB of shared memory, so two do.)
int sa_mlp_tc_launch(SaParams p, cudaStream_t st, int groups_per_cta)
{
    TcLayout lay{};
    if (groups_per_cta == 2 && make_layout(p, lay, 2, false)) return launch_tc<2>(p, st);
    if (!make_layout(p, lay, kMaxGroups, false)) {
        if (make_layout(p, lay, 2, false)) return launch_tc<2>(p, st);       // operand tiles too large for four groups
        set_error("sa_group_mlp_max: shape not supported by the tensor-core engine");
        return TGN_ERR_INVALID;
    }
    return launch_tc<kMaxGroups>(p, st);
}

}  // namespace tgn
