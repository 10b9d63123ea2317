// pw_bn.cuh -- BatchNorm + activation epilogue of the layer chain (pw_mlp.cu), shared with the decoder's interpolating apply
// (pt_head.cu) so that both evaluate a BatchNorm channel with the same operations.
#pragma once
#include <cuda_runtime.h>

namespace tgn {

// BatchNorm channel from batch sums (mode 1) or running statistics (mode 2), applied as (x - mean) * scale + beta with the mean
// carried as hi + lo floats: folding it into a shift (x * scale + (beta - mean * scale)) costs |mean| / std ulps on the result.
// .x = mean_hi, .y = mean_lo, .z = scale, .w = beta
__device__ __forceinline__ float4 bn_scale_shift(int mode, int c, int cn, const double* stats, double count, const float* gamma,
                                                 const float* beta, float eps, const float* rmean, const float* rvar)
{
    double mean, var;
    if (mode == 1) {
        mean = stats[c] / count;
        var = fmax(stats[cn + c] / count - mean * mean, 0.0);
    } else {
        mean = static_cast<double>(rmean[c]);
        var = static_cast<double>(rvar[c]);
    }
    float4 a;
    a.x = static_cast<float>(mean);
    a.y = static_cast<float>(mean - static_cast<double>(a.x));
    a.z = static_cast<float>(static_cast<double>(gamma ? gamma[c] : 1.f) / sqrt(var + static_cast<double>(eps)));
    a.w = beta ? beta[c] : 0.f;
    return a;
}
__device__ __forceinline__ float bn_apply(float x, const float4& a) { return fmaf((x - a.x) - a.y, a.z, a.w); }
// torch's leaky_relu kernel: keeps the sign of a zero, and NaN stays NaN
__device__ __forceinline__ float leaky_relu(float v, float slope) { return v > 0.f ? v : v * slope; }
// torch's training-mode side effect: running = (1-m) running + m batch (variance unbiased)
__device__ __forceinline__ void bn_update_running(int c, int cn, const double* stats, double count, float momentum, float* rmean, float* rvar)
{
    const double mean = stats[c] / count;
    const double var = fmax(stats[cn + c] / count - mean * mean, 0.0);
    const double unbiased = count > 1.0 ? var * count / (count - 1.0) : var;
    rmean[c] = (1.f - momentum) * rmean[c] + momentum * static_cast<float>(mean);
    rvar[c] = (1.f - momentum) * rvar[c] + momentum * static_cast<float>(unbiased);
}

}  // namespace tgn
