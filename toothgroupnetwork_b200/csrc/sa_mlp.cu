// sa_mlp.cu -- fused set-abstraction body (gather -> shared MLP -> max over neighbours),
// fp32 CUDA-core engine + the dispatcher of tgn_sa_group_mlp_max.
//
// The reference runs this as separate PyTorch ops: two advanced-index gathers, a subtract, a
// cat, a permute, then per layer Conv2d(1x1) + BatchNorm2d + ReLU over a materialised
// (B, C, K, S) tensor, then torch.max (external_libs/pointnet2_utils/pointnet2_utils.py:160-170,
// 227-237, 276-294).  Here one CTA takes a tile of up to 128 grouped rows, builds the
// [xyz_rel | feats] rows in shared memory straight from the index table, runs every layer out
// of shared memory (ping-pong activation buffers, weights staged per layer) and reduces the K
// rows of each group before anything is written: HBM sees the inputs once and (B, C_out, S) once.
//
// This engine is exact fp32 FMA arithmetic and handles any K and any widths <= 128; it is the
// numerical reference for, and the fallback of, the tensor-core engine in sa_mlp_tc.cu.
#include <algorithm>

#include "common.cuh"
#include "sa_mlp.cuh"
#include "tgn_b200.h"

namespace tgn {
namespace {

constexpr int kRowsMax = 128;
constexpr int kThreads = 512;        // 16 warps: enough warps per scheduler to cover the shared-memory latency of the FMA loop
constexpr int kWarps = kThreads / 32;

// Build activation rows [xyz_rel | feats] (or [feats | xyz_rel]) for `rows` grouped rows.
__device__ __forceinline__ void gather_rows_to_smem(const SaParams& p, int b, int s0, int row0_in_group, int rows,
                                                    const int* jrow, float* act, int cs)
{
    const int cin = p.ch[0];
    const float* xyz = p.xyz + 3 * static_cast<size_t>(b) * p.N;
    const float* feats = p.feats ? p.feats + static_cast<size_t>(b) * p.N * p.D : nullptr;
    for (int e = threadIdx.x; e < rows * cin; e += kThreads) {
        const int r = e / cin, c = e - r * cin;
        const int j = jrow[r];
        const int s = s0 + (p.K <= kRowsMax ? r / p.K : 0);
        const int xc = p.xyz_first ? c : c - p.D;          // channel inside the xyz block, if any
        float v = 0.f;
        if (j >= 0 && j < p.N) {
            if (xc >= 0 && xc < 3)
                v = __fsub_rn(__ldg(xyz + 3 * static_cast<size_t>(j) + xc),
                              __ldg(p.new_xyz + 3 * (static_cast<size_t>(b) * p.S + s) + xc));
            else
                v = __ldg(feats + static_cast<size_t>(j) * p.D + (p.xyz_first ? c - 3 : c));
        }
        act[r * cs + c] = v;
    }
    (void)row0_in_group;
}

// Output columns per warp CPW (kWarps warps): 4 rows x CPW columns per thread.  The accumulators are packed
// fp32 pairs of adjacent output columns (two IEEE fp32 FMAs each, rounding like the scalar op); the weight pairs
// come straight out of the 16-byte shared loads.
template <int CPW>
__device__ __forceinline__ void dense_layer(const float* __restrict__ act_in, float* __restrict__ act_out, const float* wt,
                                            const float* __restrict__ bias, int cin, int cout, int cout_pad, int cs)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int c0 = warp * CPW;
    if (c0 >= cout) return;
    uint64_t acc[4][CPW / 2];
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int c = 0; c < CPW / 2; ++c) acc[r][c] = 0ull;          // (+0.f, +0.f)
#pragma unroll 2
    for (int ci = 0; ci < cin; ++ci) {
        uint64_t a[4];
#pragma unroll
        for (int r = 0; r < 4; ++r) {
            const float v = act_in[(lane + 32 * r) * cs + ci];
            a[r] = pack2(v, v);
        }
#pragma unroll
        for (int c4 = 0; c4 < CPW / 4; ++c4) {
            const ulonglong2 w = *reinterpret_cast<const ulonglong2*>(wt + ci * cout_pad + c0 + 4 * c4);
#pragma unroll
            for (int r = 0; r < 4; ++r) {
                acc[r][2 * c4 + 0] = fma2(a[r], w.x, acc[r][2 * c4 + 0]);
                acc[r][2 * c4 + 1] = fma2(a[r], w.y, acc[r][2 * c4 + 1]);
            }
        }
    }
#pragma unroll
    for (int c = 0; c < CPW / 2; ++c) {
        const int co = c0 + 2 * c;
        const float b0 = co < cout ? __ldg(bias + co) : 0.f, b1 = co + 1 < cout ? __ldg(bias + co + 1) : 0.f;
#pragma unroll
        for (int r = 0; r < 4; ++r) {
            float v0, v1;
            unpack2(acc[r][c], v0, v1);
            if (co < cout) act_out[(lane + 32 * r) * cs + co] = fmaxf(v0 + b0, 0.f);
            if (co + 1 < cout) act_out[(lane + 32 * r) * cs + co + 1] = fmaxf(v1 + b1, 0.f);
        }
    }
}

__global__ void __launch_bounds__(kThreads)
sa_mlp_fp32_kernel(const SaParams p)
{
    extern __shared__ __align__(16) float smem[];
    const int cs = p.cstride;
    float* act0 = smem;
    float* act1 = act0 + kRowsMax * cs;
    float* wt = act1 + kRowsMax * cs;                          // [cin][cout_pad] of the current layer
    int* jrow = reinterpret_cast<int*>(wt + p.wt_floats);

    auto stage_weights = [&](int l, float* dst) {             // W[l] (cout x cin, row-major) -> [cin][cout_pad]
        const int cin = p.ch[l], cout = p.ch[l + 1];
        const int cout_pad = (cout + 15) & ~15;
        for (int e = threadIdx.x; e < cin * cout_pad; e += kThreads) {
            const int ci = e / cout_pad, co = e - ci * cout_pad;
            dst[e] = co < cout ? __ldg(p.W[l] + static_cast<size_t>(co) * cin + ci) : 0.f;
        }
    };
    if (p.wt_resident)                                        // once per (persistent) CTA
        for (int l = 0; l < p.L; ++l) stage_weights(l, wt + p.wt_off[l]);

    const long long total_tiles = static_cast<long long>(p.tiles_x) * p.B;
    for (long long tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        const int b = static_cast<int>(tile / p.tiles_x);
        const int bx = static_cast<int>(tile - static_cast<long long>(b) * p.tiles_x);
        int s0, rows, k0 = 0;
        if (p.K <= kRowsMax) {
            s0 = bx * p.gpt;
            rows = min(p.gpt, p.S - s0) * p.K;
        } else {
            s0 = bx / p.chunks;
            k0 = (bx % p.chunks) * kRowsMax;
            rows = min(kRowsMax, p.K - k0);
        }
        __syncthreads();                                        // the previous tile is done with act / jrow
        const int* gi = p.gidx + (static_cast<size_t>(b) * p.S + s0) * p.K + k0;
        for (int r = threadIdx.x; r < kRowsMax; r += kThreads) jrow[r] = r < rows ? __ldg(gi + r) : -1;
        __syncthreads();
        gather_rows_to_smem(p, b, s0, k0, rows, jrow, act0, cs);
        // rows past `rows` are never read back; zero them once so the FMAs stay finite
        for (int e = threadIdx.x + rows * cs; e < kRowsMax * cs; e += kThreads) act0[e] = 0.f;

        float* cur = act0;
        float* nxt = act1;
        for (int l = 0; l < p.L; ++l) {
            const int cin = p.ch[l], cout = p.ch[l + 1];
            const int cout_pad = (cout + 15) & ~15;
            __syncthreads();                                    // previous layer done with wt / cur ready
            const float* wl = wt + (p.wt_resident ? p.wt_off[l] : 0);
            if (!p.wt_resident) {
                stage_weights(l, wt);
                __syncthreads();
            }
            const int cpw = (cout + kWarps - 1) / kWarps;
            if (cpw <= 4) dense_layer<4>(cur, nxt, wl, p.bias[l], cin, cout, cout_pad, cs);
            else if (cpw <= 8) dense_layer<8>(cur, nxt, wl, p.bias[l], cin, cout, cout_pad, cs);
            else dense_layer<16>(cur, nxt, wl, p.bias[l], cin, cout, cout_pad, cs);
            float* t = cur; cur = nxt; nxt = t;
        }
        __syncthreads();

        // ---- max over the K rows of each group, channel-first store --------------------------------
        const int cout = p.ch[p.L];
        float* ob = p.out + (static_cast<size_t>(b) * p.out_c_total + p.out_c_offset) * p.S;
        if (p.K <= kRowsMax) {
            const int groups = rows / p.K;
            for (int e = threadIdx.x; e < groups * cout; e += kThreads) {
                const int g = e / cout, co = e - g * cout;
                float m = cur[(g * p.K) * cs + co];
                for (int k = 1; k < p.K; ++k) m = fmaxf(m, cur[(g * p.K + k) * cs + co]);
                ob[static_cast<size_t>(co) * p.S + s0 + g] = m;
            }
        } else {
            for (int co = threadIdx.x; co < cout; co += kThreads) {
                float m = cur[co];
                for (int k = 1; k < rows; ++k) m = fmaxf(m, cur[k * cs + co]);
                // post-ReLU values are >= 0, so integer order == float order and 0 is the identity
                atomicMax(reinterpret_cast<int*>(ob + static_cast<size_t>(co) * p.S + s0), __float_as_int(m));
            }
        }
    }
}

}  // namespace

int sa_mlp_fp32_launch(SaParams p, cudaStream_t st)
{
    int cmax = 0, wmax = 0, wsum = 0;
    for (int l = 0; l <= p.L; ++l) cmax = std::max(cmax, p.ch[l]);
    for (int l = 0; l < p.L; ++l) {
        const int wl = p.ch[l] * ((p.ch[l + 1] + 15) & ~15);
        p.wt_off[l] = wsum;
        wmax = std::max(wmax, wl);
        wsum += (wl + 3) & ~3;
    }
    p.cstride = cmax | 1;                       // odd row stride: conflict-free column walks
    // every layer's weights resident in shared memory when they fit next to the two activation buffers
    // (then a persistent CTA stages them once); else one layer at a time, re-staged per tile
    const size_t fixed = 2ull * kRowsMax * p.cstride * sizeof(float) + kRowsMax * sizeof(int);
    p.wt_resident = fixed + static_cast<size_t>(wsum) * sizeof(float) <= 226 * 1024 ? 1 : 0;
    p.wt_floats = p.wt_resident ? wsum : ((wmax + 3) & ~3);
    const size_t smem = fixed + static_cast<size_t>(p.wt_floats) * sizeof(float);
    if (smem > 227 * 1024) { set_error("sa_group_mlp_max: %zu bytes of shared memory needed", smem); return TGN_ERR_INVALID; }
    const int rc_attr = ensure_dynamic_smem(reinterpret_cast<const void*>(sa_mlp_fp32_kernel), smem);
    if (rc_attr != TGN_OK) return rc_attr;
    if (p.K <= kRowsMax) {
        p.gpt = kRowsMax / p.K;
        p.chunks = 1;
        p.tiles_x = (p.S + p.gpt - 1) / p.gpt;
    } else {
        p.gpt = 1;
        p.chunks = (p.K + kRowsMax - 1) / kRowsMax;
        p.tiles_x = p.S * p.chunks;
        // partial maxima are merged with atomicMax: clear this branch's slice of out first
        const cudaError_t e = cudaMemset2DAsync(p.out + static_cast<size_t>(p.out_c_offset) * p.S,
                                                static_cast<size_t>(p.out_c_total) * p.S * sizeof(float), 0,
                                                static_cast<size_t>(p.ch[p.L]) * p.S * sizeof(float), p.B, st);
        if (e != cudaSuccess) { set_error("cudaMemset2DAsync: %s", cudaGetErrorString(e)); return TGN_ERR_CUDA; }
    }
    // persistent CTAs (as many per SM as shared memory and the 2048-thread limit allow) over the flattened tile list
    const long long total_tiles = static_cast<long long>(p.tiles_x) * p.B;
    const long long per_sm = std::max<long long>(1, std::min<long long>(2048 / kThreads, (227 * 1024) / (smem + 1024)));
    const dim3 grid(static_cast<unsigned>(std::min<long long>(total_tiles, per_sm * sm_count())));
    sa_mlp_fp32_kernel<<<grid, kThreads, smem, st>>>(p);
    return check_launch("sa_mlp_fp32_kernel");
}

}  // namespace tgn

extern "C" int tgn_sa_group_mlp_max(int B, int N, int S, int K, int D, const float* xyz, const float* feats,
                                    const float* new_xyz, const int* group_idx, int xyz_first, int n_layers,
                                    const int* channels, const float* const* weights, const float* const* biases,
                                    float* out, int out_c_total, int out_c_offset, int engine, void* stream)
{
    using namespace tgn;
    if (B <= 0 || S <= 0) return TGN_OK;
    if (N <= 0 || K <= 0) { set_error("sa_group_mlp_max: N and K must be positive"); return TGN_ERR_INVALID; }
    if (B > 65535) { set_error("sa_group_mlp_max: B=%d exceeds gridDim.y", B); return TGN_ERR_INVALID; }
    if (n_layers < 1 || n_layers > kSaMaxLayers) { set_error("sa_group_mlp_max: 1..%d layers supported, got %d", kSaMaxLayers, n_layers); return TGN_ERR_INVALID; }
    if (D < 0 || (D > 0 && !feats)) { set_error("sa_group_mlp_max: feats missing for D=%d", D); return TGN_ERR_INVALID; }
    if (channels[0] != 3 + D) { set_error("sa_group_mlp_max: channels[0]=%d but 3+D=%d", channels[0], 3 + D); return TGN_ERR_INVALID; }
    SaParams p{};
    p.B = B; p.N = N; p.S = S; p.K = K; p.D = D;
    p.xyz = xyz; p.feats = feats; p.new_xyz = new_xyz; p.gidx = group_idx;
    p.xyz_first = xyz_first; p.L = n_layers;
    for (int l = 0; l <= n_layers; ++l) {
        p.ch[l] = channels[l];
        if (channels[l] < 1 || channels[l] > kSaMaxWidth) {
            set_error("sa_group_mlp_max: layer width %d outside [1,%d]", channels[l], kSaMaxWidth);
            return TGN_ERR_INVALID;
        }
    }
    for (int l = 0; l < n_layers; ++l) { p.W[l] = weights[l]; p.bias[l] = biases[l]; }
    p.out = out; p.out_c_total = out_c_total; p.out_c_offset = out_c_offset;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    // auto: the 3xTF32 tensor-core engine when the shape fits it (widths <= 64), else the wide tensor-core
    // engine (tf32 first layer, bf16x2-split later layers: ~1e-5 relative, inside the 1e-4 bar), else the
    // exact-FMA CUDA-core engine (any K, widths <= 128)
    if (engine < 0 || engine > 5 || engine == 4) { set_error("sa_group_mlp_max: unknown engine %d", engine); return TGN_ERR_INVALID; }
    if (engine == 2 || engine == 5 || (engine == 0 && sa_mlp_tc_supported(p))) {
        if (!sa_mlp_tc_supported(p)) { set_error("sa_group_mlp_max: shape not supported by the tensor-core engine"); return TGN_ERR_INVALID; }
        return sa_mlp_tc_launch(p, st, engine == 5 ? 2 : 4);     // 5: half-size CTAs (two per SM; share an SM with other streams' kernels)
    }
    if (engine == 3 || (engine == 0 && sa_mlp_tcw_supported(p))) {
        if (!sa_mlp_tcw_supported(p)) { set_error("sa_group_mlp_max: shape not supported by the wide tensor-core engine"); return TGN_ERR_INVALID; }
        return sa_mlp_tcw_launch(p, st);
    }
    return sa_mlp_fp32_launch(p, st);
}
