// pw_transform.cu -- PointNet's learned per-cloud transforms (torch.bmm(x^T, T_b)^T) in FFMA, next to the layer chain of pw_mlp.cu.
//
//      out[b, j, n]       = sum_{i < ct} x[b, i, n] * T_b[i, j]        j < ct
//      out[b, ct + c, n]  = x[b, ct + c, n]                            c < cpass (copied bit for bit)
//
// PointNet applies T_b twice per forward (external_libs/pointnet2_utils/pointnet_utils.py:104-121): the 3 x 3 input transform to
// xyz with the normals passed through (ct = 3, cpass = 3), and the 128 x 128 feature transform (ct = 128, cpass = 0).  At
// ct = 128 this is 0.79 GFLOP per 24 000-point cloud, a few microseconds of FFMA, so it stays off the tensor cores.  It is not
// folded into the next layer's weights either: a 256-row tile of pw_layer_kernel can straddle two clouds.
//
// CTA = 128 points x 32 output channels of one cloud.  The CTA's 32 columns of T_b (all ct rows) are staged in shared memory;
// each thread owns one point and keeps its 32 sums in registers.  Summation order: every sum starts at +0 and takes
// acc = fmaf(x[i], T_b[i, j], acc) for i = 0, 1, ..., ct - 1, so |out - exact| <= ct * 2^-24 * sum_i |x_i| |T_ij| (plus the
// rounding of an fp64 truth to fp32).  x and out are read and written through (batch, channel, point) strides, so the
// permute(0, 2, 1) view of a point-major cloud needs no copy.
#include "common.cuh"
#include "tgn_b200.h"

namespace tgn {
namespace {

constexpr int kTP = 128;          // points per CTA (one per thread)
constexpr int kTJ = 32;           // output channels per CTA
constexpr int kTMax = 128;        // largest ct

__global__ void __launch_bounds__(kTP) pw_cloud_transform_kernel(int N, int ct, int cpass, const float* __restrict__ x, long long xs_b,
                                                                 long long xs_c, long long xs_n, const float* __restrict__ t,
                                                                 long long t_batch_stride, float* __restrict__ out, long long os_b,
                                                                 long long os_c, long long os_n)
{
    __shared__ __align__(16) float ts[kTMax * kTJ];            // ts[i * kTJ + jj] = T_b[i, j0 + jj], zero for j0 + jj >= ct
    const int b = blockIdx.z, j0 = blockIdx.y * kTJ;
    const float* tb = t + b * t_batch_stride;
    for (int e = threadIdx.x; e < ct * kTJ; e += kTP) {
        const int i = e / kTJ, j = j0 + (e - i * kTJ);
        ts[e] = j < ct ? __ldg(tb + static_cast<long long>(i) * ct + j) : 0.f;
    }
    __syncthreads();
    const int n = blockIdx.x * kTP + threadIdx.x;
    if (n >= N) return;
    const float* xp = x + b * xs_b + n * xs_n;
    float acc[kTJ];
#pragma unroll
    for (int jj = 0; jj < kTJ; ++jj) acc[jj] = 0.f;
    for (int i = 0; i < ct; ++i) {
        const float v = __ldg(xp + i * xs_c);
        const float4* row = reinterpret_cast<const float4*>(ts + i * kTJ);
#pragma unroll
        for (int q = 0; q < kTJ / 4; ++q) {
            const float4 w = row[q];
            acc[4 * q] = fmaf(v, w.x, acc[4 * q]);
            acc[4 * q + 1] = fmaf(v, w.y, acc[4 * q + 1]);
            acc[4 * q + 2] = fmaf(v, w.z, acc[4 * q + 2]);
            acc[4 * q + 3] = fmaf(v, w.w, acc[4 * q + 3]);
        }
    }
    float* op = out + b * os_b + n * os_n;
#pragma unroll
    for (int jj = 0; jj < kTJ; ++jj)
        if (j0 + jj < ct) op[(j0 + jj) * os_c] = acc[jj];
    if (blockIdx.y == 0)
        for (int c = ct; c < ct + cpass; ++c) op[c * os_c] = __ldg(xp + c * xs_c);
}

}  // namespace
}  // namespace tgn

extern "C" int tgn_pw_cloud_transform(int B, int N, int ct, int cpass, const float* x, long long xs_b, long long xs_c, long long xs_n,
                                      const float* t, long long t_batch_stride, float* out, long long os_b, long long os_c,
                                      long long os_n, void* stream)
{
    using namespace tgn;
    if (B < 1 || B > 65535 || N < 1 || ct < 1 || ct > kTMax || cpass < 0 || !x || !t || !out || t_batch_stride < 0) {
        set_error("pw_cloud_transform: bad arguments (need 1 <= B <= 65535, N >= 1, 1 <= ct <= %d, cpass >= 0)", kTMax);
        return TGN_ERR_INVALID;
    }
    dim3 grid((N + kTP - 1) / kTP, (ct + kTJ - 1) / kTJ, B);
    pw_cloud_transform_kernel<<<grid, kTP, 0, static_cast<cudaStream_t>(stream)>>>(N, ct, cpass, x, xs_b, xs_c, xs_n, t, t_batch_stride,
                                                                                    out, os_b, os_c, os_n);
    return check_launch("pw_cloud_transform_kernel");
}
