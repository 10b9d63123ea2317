// pt_block.cu -- the end of PointTransformerBlock.forward (models/modules/cbl_point_transformer/blocks.py:132-134): bn3 of linear3's
// channel-major output from the layer chain (pw_mlp.cu), the residual add and the ReLU, written row-major.
//
// torch rounds bn3's output to fp32 before the in-place `x += identity`, then applies the ReLU, so the kernel does the same: the
// subtract-first BatchNorm of pw_bn.cuh, one fp32 add, then the ReLU.  A 32-row x 32-channel tile goes through shared memory so
// that the channel-major source is read and the row-major result and identity are touched with whole-warp transactions, as in
// pt_head.cu's interpolating apply.
#include "common.cuh"
#include "pw_bn.cuh"
#include "tgn_b200.h"

namespace tgn {
namespace {

constexpr int kTile = 32;
constexpr int kTileRowsPerPass = 8;

__global__ void __launch_bounds__(kTile * kTileRowsPerPass) pt_res_apply_kernel(const tgn_pt_res_apply_t p)
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
        if (c < a.channels && r < a.rows) tile[cc][tx] = bn_apply(a.src[static_cast<size_t>(c) * a.rows + r], aff[cc]);
    }
    __syncthreads();
    const int c = c0 + tx;
    if (c >= a.channels) return;
    for (int rr = ty; rr < kTile; rr += kTileRowsPerPass) {
        const int r = r0 + rr;
        if (r >= a.rows) break;
        float v = __fadd_rn(tile[tx][rr], __ldg(p.identity + static_cast<size_t>(r) * p.identity_row_stride + c));
        if (a.relu) v = fmaxf(v, 0.f);
        a.out[static_cast<size_t>(r) * a.channels + c] = v;
    }
}

}  // namespace
}  // namespace tgn

extern "C" {

int tgn_pt_res_apply_struct_size(void) { return static_cast<int>(sizeof(tgn_pt_res_apply_t)); }

int tgn_pt_res_apply(const tgn_pt_res_apply_t* p, void* stream)
{
    using namespace tgn;
    if (!p) { set_error("pt_res_apply: null descriptor"); return TGN_ERR_INVALID; }
    const tgn_pw_apply_t& a = p->apply;
    if (!a.src || !a.out || !p->identity || a.rows < 1 || a.channels < 1 || a.ymin || a.act || p->identity_row_stride < a.channels) {
        set_error("pt_res_apply: bad arguments");
        return TGN_ERR_INVALID;
    }
    if (a.affine == 1 && !a.stats) { set_error("pt_res_apply: affine=1 needs stats"); return TGN_ERR_INVALID; }
    if (a.affine == 2 && (!a.running_mean || !a.running_var)) { set_error("pt_res_apply: affine=2 needs running statistics"); return TGN_ERR_INVALID; }
    dim3 grid((a.rows + kTile - 1) / kTile, (a.channels + kTile - 1) / kTile);
    pt_res_apply_kernel<<<grid, dim3(kTile, kTileRowsPerPass), 0, static_cast<cudaStream_t>(stream)>>>(*p);
    return check_launch("pt_res_apply_kernel");
}

}  // extern "C"
