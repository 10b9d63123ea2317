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
// The kernel itself is in pw_layer.cuh; `accum` = 1 launches its promoted-accumulation form (pw_mlp_promoted.cu).
#include <algorithm>
#include <cmath>

#include "common.cuh"
#include "pw_bn.cuh"
#include "pw_layer.cuh"
#include "tgn_b200.h"

namespace tgn {
namespace {

using namespace pw;

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
    if (L.accum != 0 && L.accum != 1) { set_error("pw_layer_forward: unknown accum %d", L.accum); return TGN_ERR_INVALID; }
    if (L.ymax) {
        if (!L.ymin || L.group < 1 || L.rows % L.group != 0) { set_error("pw_layer_forward: bad extrema arguments"); return TGN_ERR_INVALID; }
        a.n_groups = L.rows / L.group;
    }
    if (L.accum == 1) return pw_layer_launch_promoted(a, static_cast<cudaStream_t>(stream));
    return pw_layer_launch<256, 0>(a, static_cast<cudaStream_t>(stream), "pw_layer_kernel");
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
