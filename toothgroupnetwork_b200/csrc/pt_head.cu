// pt_head.cu -- the point-transformer network's decoder and heads (models/modules/cbl_point_transformer/blocks.py:82-111,
// heads.py:13-61) after their Linear layers have run on the layer chain (pw_mlp.cu).
//
//   * pt_up_apply_kernel: the last BatchNorm + ReLU of TransitionUp.linear1 with the k = 3 interpolation of linear2's output
//     added in the same pass, in torch's order (pointops.interpolation accumulates into zeros, one rounded product at a time,
//     and blocks.py:110 adds the result).  A 32-row x 32-channel tile goes through shared memory so that the channel-major
//     chain output is read and the row-major result written with whole-warp transactions, and the gathered source rows are
//     read 32 channels at a time.
//   * head_classify_kernel: MultiHead's cls Linear over the concatenation of every level's latent upsampled to level 0.  For
//     k = 1 the reference's interpolation weight is x / x = 1.0 and 0 + v * 1.0 = v, so its upsampled copies are exactly
//     lat_s[nn_s]: one thread per level-0 row gathers them and runs the product, weights broadcast from shared memory; neither
//     the (n0, 32 levels) concatenation nor the per-level copies are written.
#include <algorithm>

#include "common.cuh"
#include "pw_bn.cuh"
#include "tgn_b200.h"

namespace tgn {
namespace {

constexpr int kTile = 32;          // rows and channels per tile of the interpolating apply
constexpr int kTileRowsPerPass = 8;
constexpr int kHeadThreads = 128;
constexpr int kLatent = 32;        // channels of a level's latent (config.base_fdim)

__global__ void __launch_bounds__(kTile * kTileRowsPerPass) pt_up_apply_kernel(const tgn_pt_up_apply_t p)
{
    __shared__ float tile[kTile][kTile + 1];
    __shared__ float4 aff[kTile];
    const tgn_pw_apply_t& a = p.apply;
    const int r0 = blockIdx.x * kTile, c0 = blockIdx.y * kTile, tx = threadIdx.x, ty = threadIdx.y;
    if (ty == 0 && c0 + tx < a.channels) {
        const int c = c0 + tx;
        aff[tx] = a.affine ? bn_scale_shift(a.affine, c, a.channels, a.stats, static_cast<double>(a.stat_rows), a.gamma, a.beta, a.eps,
                                            a.running_mean, a.running_var)
                           : make_float4(0.f, 0.f, 1.f, 0.f);
        if (a.affine == 1 && a.update_running && blockIdx.x == 0)
            bn_update_running(c, a.channels, a.stats, static_cast<double>(a.stat_rows), a.momentum, a.running_mean, a.running_var);
    }
    __syncthreads();
    for (int cc = ty; cc < kTile; cc += kTileRowsPerPass) {
        const int c = c0 + cc, r = r0 + tx;
        if (c < a.channels && r < a.rows) {
            float v = bn_apply(a.src[static_cast<size_t>(c) * a.rows + r], aff[cc]);
            if (a.act == 1) v = leaky_relu(v, a.act_slope);
            else if (a.relu) v = fmaxf(v, 0.f);
            tile[cc][tx] = v;
        }
    }
    __syncthreads();
    const int c = c0 + tx;
    if (c >= a.channels) return;
    for (int rr = ty; rr < kTile; rr += kTileRowsPerPass) {
        const int r = r0 + rr;
        if (r >= a.rows) break;
        float v = tile[tx][rr];
        if (p.f) {
            float s = 0.f;
#pragma unroll
            for (int j = 0; j < 3; ++j) {
                const int i = __ldg(p.idx + 3 * static_cast<size_t>(r) + j);
                const float w = __ldg(p.w + 3 * static_cast<size_t>(r) + j);
                s = __fadd_rn(s, __fmul_rn(__ldg(p.f + static_cast<size_t>(i) * a.channels + c), w));
            }
            v = __fadd_rn(v, s);
        }
        a.out[static_cast<size_t>(r) * a.channels + c] = v;
    }
}

// KB: outputs held per thread (the smallest of 4, 8, 16, 32 that covers k)
template <int KB>
__global__ void __launch_bounds__(kHeadThreads) head_classify_kernel(const tgn_head_classify_t p)
{
    __shared__ float ws[TGN_HEAD_MAX_LEVELS * kLatent * KB];     // ws[col * KB + j] = W[j, col]
    const int cols = p.levels * kLatent;
    for (int e = threadIdx.x; e < cols * KB; e += blockDim.x) {
        const int col = e / KB, j = e - col * KB;
        ws[e] = j < p.k ? __ldg(p.w + static_cast<size_t>(j) * cols + col) : 0.f;
    }
    __syncthreads();
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= p.n0) return;
    float acc[KB];
#pragma unroll
    for (int j = 0; j < KB; ++j) acc[j] = 0.f;
    for (int s = 0; s < p.levels; ++s) {
        const int rs = p.nn[s] ? __ldg(p.nn[s] + r) : r;
        const float* x = p.lat[s] + rs;
        const size_t ns = static_cast<size_t>(p.n[s]);
        const float* wl = ws + s * kLatent * KB;
#pragma unroll 4
        for (int c = 0; c < kLatent; ++c) {
            const float v = __ldg(x + c * ns);
#pragma unroll
            for (int j = 0; j < KB; ++j) acc[j] = __fmaf_rn(wl[c * KB + j], v, acc[j]);
        }
    }
    float* o = p.out + static_cast<size_t>(r) * p.k;
#pragma unroll
    for (int j = 0; j < KB; ++j)
        if (j < p.k) o[j] = p.b ? __fadd_rn(acc[j], __ldg(p.b + j)) : acc[j];
}

}  // namespace
}  // namespace tgn

extern "C" {

int tgn_pt_head_struct_size(int which)
{
    return which == 0 ? static_cast<int>(sizeof(tgn_pt_up_apply_t)) : static_cast<int>(sizeof(tgn_head_classify_t));
}

int tgn_pt_up_apply(const tgn_pt_up_apply_t* p, void* stream)
{
    using namespace tgn;
    if (!p) { set_error("pt_up_apply: null descriptor"); return TGN_ERR_INVALID; }
    const tgn_pw_apply_t& a = p->apply;
    if (!a.src || !a.out || a.rows < 1 || a.channels < 1 || a.ymin) { set_error("pt_up_apply: bad arguments"); return TGN_ERR_INVALID; }
    if (a.affine == 1 && !a.stats) { set_error("pt_up_apply: affine=1 needs stats"); return TGN_ERR_INVALID; }
    if (a.affine == 2 && (!a.running_mean || !a.running_var)) { set_error("pt_up_apply: affine=2 needs running statistics"); return TGN_ERR_INVALID; }
    if (p->f && (!p->idx || !p->w || p->f_rows < 1)) { set_error("pt_up_apply: the addend needs idx, w and f_rows >= 1"); return TGN_ERR_INVALID; }
    dim3 grid((a.rows + kTile - 1) / kTile, (a.channels + kTile - 1) / kTile);
    pt_up_apply_kernel<<<grid, dim3(kTile, kTileRowsPerPass), 0, static_cast<cudaStream_t>(stream)>>>(*p);
    return check_launch("pt_up_apply_kernel");
}

int tgn_head_classify(const tgn_head_classify_t* p, void* stream)
{
    using namespace tgn;
    if (!p || !p->w || !p->out || p->n0 < 1 || p->k < 1 || p->k > 32 || p->levels < 1 || p->levels > TGN_HEAD_MAX_LEVELS) {
        set_error("head_classify: bad arguments (need 1 <= k <= 32, 1 <= levels <= %d)", TGN_HEAD_MAX_LEVELS);
        return TGN_ERR_INVALID;
    }
    for (int s = 0; s < p->levels; ++s) {
        if (!p->lat[s] || p->n[s] < 1 || (!p->nn[s] && p->n[s] != p->n0)) {
            set_error("head_classify: level %d needs a latent, n >= 1, and nn unless n == n0", s);
            return TGN_ERR_INVALID;
        }
    }
    const int blocks = (p->n0 + kHeadThreads - 1) / kHeadThreads;
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (p->k <= 4) head_classify_kernel<4><<<blocks, kHeadThreads, 0, st>>>(*p);
    else if (p->k <= 8) head_classify_kernel<8><<<blocks, kHeadThreads, 0, st>>>(*p);
    else if (p->k <= 16) head_classify_kernel<16><<<blocks, kHeadThreads, 0, st>>>(*p);
    else head_classify_kernel<32><<<blocks, kHeadThreads, 0, st>>>(*p);
    return check_launch("head_classify_kernel");
}

}  // extern "C"
