// gather.cu -- the gather / scatter family of the pointops API for sm_90a.
//
// Replaces pointops/src/{grouping,interpolation,subtraction,aggregation}/*_cuda_kernel.cu of
// the reference (one thread per output ELEMENT, three integer divisions and one index load per
// element).  These are HBM/L2 gather-bandwidth kernels: here a thread owns one (row, 4-channel)
// vector when c % 4 == 0 (128-bit loads/stores, one index load per vector) and falls back to
// scalar elements otherwise; grids are sized in multiples of the SM count with grid-stride loops.
// Forward results are bit-identical to the reference (same fma chains); the scatter-add
// backwards use fp32 atomics like the reference (summation order unspecified there too).
#include <algorithm>

#include "common.cuh"
#include "tgn_b200.h"

// The reference's launchers return void: a rejected call cannot be signalled to the caller, so say it on stderr
// instead of returning with the outputs untouched (ADVICE r1).
#ifndef TGN_REPORT
#include <cstdio>
#define TGN_REPORT(call) do { if ((call) != TGN_OK) std::fprintf(stderr, "libtgn_b200: %s\n", tgn_last_error()); } while (0)
#endif

namespace tgn {
namespace {

inline int grid_for(size_t work_items, int threads)
{
    const size_t want = (work_items + threads - 1) / threads;
    const size_t cap = static_cast<size_t>(sm_count()) * 16;
    return static_cast<int>(std::max<size_t>(1, std::min(want, cap)));
}

// out[g, :] = in[idx[g], :]    g over m*nsample rows                (grouping_cuda_kernel.cu:5-14)
template <int VEC>
__global__ void __launch_bounds__(256)
rows_gather_kernel(size_t rows, int c, const float* __restrict__ in, const int* __restrict__ idx, float* __restrict__ out)
{
    const int cv = c / VEC;
    const size_t total = rows * cv;
    for (size_t e = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; e < total;
         e += static_cast<size_t>(gridDim.x) * blockDim.x) {
        const size_t g = e / cv;
        const int v = static_cast<int>(e - g * cv);
        const size_t src = static_cast<size_t>(__ldg(idx + g)) * c + static_cast<size_t>(v) * VEC;
        if (VEC == 4) *reinterpret_cast<float4*>(out + g * c + v * 4) = __ldg(reinterpret_cast<const float4*>(in + src));
        else out[g * c + v] = __ldg(in + src);
    }
}

// grad_in[idx[g], :] += grad_out[g, :]                              (grouping_cuda_kernel.cu:16-25)
__global__ void __launch_bounds__(256)
rows_scatter_add_kernel(size_t rows, int c, const float* __restrict__ grad_out, const int* __restrict__ idx,
                        float* __restrict__ grad_in)
{
    const size_t total = rows * c;
    for (size_t e = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; e < total;
         e += static_cast<size_t>(gridDim.x) * blockDim.x) {
        const size_t g = e / c;
        const int ch = static_cast<int>(e - g * c);
        atomicAdd(grad_in + static_cast<size_t>(__ldg(idx + g)) * c + ch, __ldg(grad_out + e));
    }
}

// out[n,c] += sum_i in[idx[n,i],c] * w[n,i]  as an fma chain in neighbour order
// (interpolation_cuda_kernel.cu:5-18; the reference's "+=" contracts to FFMA).
__global__ void __launch_bounds__(256)
interp_forward_kernel(int n, int c, int k, const float* __restrict__ in, const int* __restrict__ idx,
                      const float* __restrict__ w, float* __restrict__ out, bool fused)
{
    const size_t total = static_cast<size_t>(n) * c;
    for (size_t e = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; e < total;
         e += static_cast<size_t>(gridDim.x) * blockDim.x) {
        const size_t p = e / c;
        const int ch = static_cast<int>(e - p * c);
        float acc = out[e];
        if (fused) {
            for (int i = 0; i < k; ++i)
                acc = __fmaf_rn(__ldg(in + static_cast<size_t>(__ldg(idx + p * k + i)) * c + ch), __ldg(w + p * k + i), acc);
        } else {      // pointops.interpolation (pointops.py:177-179) accumulates with torch ops: product rounded, then added
            for (int i = 0; i < k; ++i)
                acc = __fadd_rn(acc, __fmul_rn(__ldg(in + static_cast<size_t>(__ldg(idx + p * k + i)) * c + ch), __ldg(w + p * k + i)));
        }
        out[e] = acc;
    }
}

// grad_in[idx[n,i],c] += grad_out[n,c] * w[n,i]                     (interpolation_cuda_kernel.cu:20-33)
__global__ void __launch_bounds__(256)
interp_backward_kernel(int n, int c, int k, const float* __restrict__ grad_out, const int* __restrict__ idx,
                       const float* __restrict__ w, float* __restrict__ grad_in)
{
    const size_t total = static_cast<size_t>(n) * c;
    for (size_t e = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; e < total;
         e += static_cast<size_t>(gridDim.x) * blockDim.x) {
        const size_t p = e / c;
        const int ch = static_cast<int>(e - p * c);
        const float g = __ldg(grad_out + e);
        for (int i = 0; i < k; ++i)
            atomicAdd(grad_in + static_cast<size_t>(__ldg(idx + p * k + i)) * c + ch, __fmul_rn(g, __ldg(w + p * k + i)));
    }
}

// out[n,s,c] = in1[n,c] - in2[idx[n,s],c]                           (subtraction_cuda_kernel.cu:5-16)
template <int VEC>
__global__ void __launch_bounds__(256)
subtraction_forward_kernel(int n, int nsample, int c, const float* __restrict__ in1, const float* __restrict__ in2,
                           const int* __restrict__ idx, float* __restrict__ out)
{
    const int cv = c / VEC;
    const size_t rows = static_cast<size_t>(n) * nsample, total = rows * cv;
    for (size_t e = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; e < total;
         e += static_cast<size_t>(gridDim.x) * blockDim.x) {
        const size_t g = e / cv;
        const int v = static_cast<int>(e - g * cv);
        const size_t p = g / nsample;
        const size_t a = p * c + static_cast<size_t>(v) * VEC;
        const size_t b = static_cast<size_t>(__ldg(idx + g)) * c + static_cast<size_t>(v) * VEC;
        if (VEC == 4) {
            const float4 x = __ldg(reinterpret_cast<const float4*>(in1 + a)), y = __ldg(reinterpret_cast<const float4*>(in2 + b));
            *reinterpret_cast<float4*>(out + g * c + v * 4) = make_float4(x.x - y.x, x.y - y.y, x.z - y.z, x.w - y.w);
        } else {
            out[g * c + v] = __ldg(in1 + a) - __ldg(in2 + b);
        }
    }
}

// grad_in1[n,c] += g ; grad_in2[idx[n,s],c] += -g                   (subtraction_cuda_kernel.cu:18-30)
// grad_in1 is a plain per-(n,c) sum over s, so it is reduced in registers (deterministic) and
// only grad_in2 needs atomics.
__global__ void __launch_bounds__(256)
subtraction_backward_kernel(int n, int nsample, int c, const int* __restrict__ idx, const float* __restrict__ grad_out,
                            float* __restrict__ grad_in1, float* __restrict__ grad_in2)
{
    const size_t total = static_cast<size_t>(n) * c;
    for (size_t e = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; e < total;
         e += static_cast<size_t>(gridDim.x) * blockDim.x) {
        const size_t p = e / c;
        const int ch = static_cast<int>(e - p * c);
        float acc = 0.f;
        for (int s = 0; s < nsample; ++s) {
            const size_t g = p * nsample + s;
            const float go = __ldg(grad_out + g * c + ch);
            acc += go;
            atomicAdd(grad_in2 + static_cast<size_t>(__ldg(idx + g)) * c + ch, -go);
        }
        grad_in1[e] += acc;             // accumulate-into semantics of the reference (caller pre-zeroes)
    }
}

// out[n,c] += sum_s (in[idx[n,s],c] + pos[n,s,c]) * w[n,s,c % w_c]  (aggregation_cuda_kernel.cu:5-20)
__global__ void __launch_bounds__(256)
aggregation_forward_kernel(int n, int nsample, int c, int w_c, const float* __restrict__ in, const float* __restrict__ pos,
                           const float* __restrict__ w, const int* __restrict__ idx, float* __restrict__ out)
{
    const size_t total = static_cast<size_t>(n) * c;
    for (size_t e = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; e < total;
         e += static_cast<size_t>(gridDim.x) * blockDim.x) {
        const size_t p = e / c;
        const int ch = static_cast<int>(e - p * c);
        const int wc = ch % w_c;
        float acc = out[e];
        for (int s = 0; s < nsample; ++s) {
            const size_t g = p * nsample + s;
            const float v = __fadd_rn(__ldg(in + static_cast<size_t>(__ldg(idx + g)) * c + ch), __ldg(pos + g * c + ch));
            acc = __fmaf_rn(v, __ldg(w + g * w_c + wc), acc);
        }
        out[e] = acc;
    }
}

// aggregation_cuda_kernel.cu:22-39
__global__ void __launch_bounds__(256)
aggregation_backward_kernel(int n, int nsample, int c, int w_c, const float* __restrict__ in, const float* __restrict__ pos,
                            const float* __restrict__ w, const int* __restrict__ idx, const float* __restrict__ grad_out,
                            float* __restrict__ grad_in, float* __restrict__ grad_pos, float* __restrict__ grad_w)
{
    const size_t total = static_cast<size_t>(n) * c;
    for (size_t e = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; e < total;
         e += static_cast<size_t>(gridDim.x) * blockDim.x) {
        const size_t p = e / c;
        const int ch = static_cast<int>(e - p * c);
        const int wc = ch % w_c;
        const float go = __ldg(grad_out + e);
        for (int s = 0; s < nsample; ++s) {
            const size_t g = p * nsample + s;
            const size_t src = static_cast<size_t>(__ldg(idx + g)) * c + ch;
            const float wv = __ldg(w + g * w_c + wc);
            const float gw = __fmul_rn(go, wv);
            atomicAdd(grad_in + src, gw);
            grad_pos[g * c + ch] = gw;
            atomicAdd(grad_w + g * w_c + wc, __fmul_rn(go, __fadd_rn(__ldg(in + src), __ldg(pos + g * c + ch))));
        }
    }
}

// Batched row gather with a per-batch base (pointnet2_utils.index_points, pointnet2_utils.py:44-61)
template <int VEC>
__global__ void __launch_bounds__(256)
batched_rows_gather_kernel(int N, int M, int c, const float* __restrict__ points, const int* __restrict__ idx,
                           float* __restrict__ out)
{
    const int b = blockIdx.y;
    const int cv = c / VEC;
    const size_t total = static_cast<size_t>(M) * cv;
    const float* src0 = points + static_cast<size_t>(b) * N * c;
    const int* ib = idx + static_cast<size_t>(b) * M;
    float* ob = out + static_cast<size_t>(b) * M * c;
    for (size_t e = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; e < total;
         e += static_cast<size_t>(gridDim.x) * blockDim.x) {
        const size_t g = e / cv;
        const int v = static_cast<int>(e - g * cv);
        const size_t src = static_cast<size_t>(__ldg(ib + g)) * c + static_cast<size_t>(v) * VEC;
        if (VEC == 4) *reinterpret_cast<float4*>(ob + g * c + v * 4) = __ldg(reinterpret_cast<const float4*>(src0 + src));
        else ob[g * c + v] = __ldg(src0 + src);
    }
}

// (B, R, C) -> (B, C, R) tiled transpose through shared memory (32x33 tile, coalesced both ways).
__global__ void __launch_bounds__(256)
transpose_kernel(int R, int C, const float* __restrict__ in, float* __restrict__ out)
{
    __shared__ float tile[32][33];
    const int b = blockIdx.z;
    const float* ib = in + static_cast<size_t>(b) * R * C;
    float* ob = out + static_cast<size_t>(b) * R * C;
    const int c0 = blockIdx.x * 32, r0 = blockIdx.y * 32;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;   // 32 x 8
    for (int i = ty; i < 32; i += 8) {
        const int r = r0 + i, c = c0 + tx;
        if (r < R && c < C) tile[i][tx] = __ldg(ib + static_cast<size_t>(r) * C + c);
    }
    __syncthreads();
    for (int i = ty; i < 32; i += 8) {
        const int c = c0 + i, r = r0 + tx;
        if (r < R && c < C) ob[static_cast<size_t>(c) * R + r] = tile[tx][i];
    }
}

// Same transpose when one side is tiny (xyz: 3, xyz+normals: 6 ...): a 32x32 tile would be mostly
// padding.  One thread per long-axis index; the long axis is the coalesced one on both sides
// (reads of a short row are contiguous per thread and contiguous across neighbouring threads).
template <int MAXS>
__global__ void __launch_bounds__(256)
transpose_short_rows_kernel(int R, int C, const float* __restrict__ in, float* __restrict__ out)
{   // in (R, C) with R <= MAXS short, C long  ->  out (C, R)
    const int b = blockIdx.y;
    const float* ib = in + static_cast<size_t>(b) * R * C;
    float* ob = out + static_cast<size_t>(b) * R * C;
    for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < C; c += gridDim.x * blockDim.x) {
        float v[MAXS];
#pragma unroll
        for (int r = 0; r < MAXS; ++r) v[r] = r < R ? __ldg(ib + static_cast<size_t>(r) * C + c) : 0.f;
#pragma unroll
        for (int r = 0; r < MAXS; ++r)
            if (r < R) ob[static_cast<size_t>(c) * R + r] = v[r];
    }
}
template <int MAXS>
__global__ void __launch_bounds__(256)
transpose_short_cols_kernel(int R, int C, const float* __restrict__ in, float* __restrict__ out)
{   // in (R, C) with R long, C <= MAXS short  ->  out (C, R)
    const int b = blockIdx.y;
    const float* ib = in + static_cast<size_t>(b) * R * C;
    float* ob = out + static_cast<size_t>(b) * R * C;
    for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < R; r += gridDim.x * blockDim.x) {
        float v[MAXS];
#pragma unroll
        for (int c = 0; c < MAXS; ++c) v[c] = c < C ? __ldg(ib + static_cast<size_t>(r) * C + c) : 0.f;
#pragma unroll
        for (int c = 0; c < MAXS; ++c)
            if (c < C) ob[static_cast<size_t>(c) * R + r] = v[c];
    }
}

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

}  // namespace
}  // namespace tgn

extern "C" {
using namespace tgn;

int tgn_grouping_forward(int m, int nsample, int c, const float* input, const int* idx, float* output, void* stream)
{
    const size_t rows = static_cast<size_t>(m) * nsample;
    if (!rows || c <= 0) return TGN_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (c % 4 == 0 && aligned16(input) && aligned16(output))
        rows_gather_kernel<4><<<grid_for(rows * (c / 4), 256), 256, 0, st>>>(rows, c, input, idx, output);
    else
        rows_gather_kernel<1><<<grid_for(rows * c, 256), 256, 0, st>>>(rows, c, input, idx, output);
    return check_launch("rows_gather_kernel");
}

int tgn_grouping_backward(int m, int nsample, int c, const float* grad_output, const int* idx, float* grad_input, void* stream)
{
    const size_t rows = static_cast<size_t>(m) * nsample;
    if (!rows || c <= 0) return TGN_OK;
    rows_scatter_add_kernel<<<grid_for(rows * c, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(rows, c, grad_output, idx, grad_input);
    return check_launch("rows_scatter_add_kernel");
}

int tgn_interpolation_forward(int n, int c, int k, const float* input, const int* idx, const float* weight, float* output, void* stream)
{
    if (n <= 0 || c <= 0) return TGN_OK;
    interp_forward_kernel<<<grid_for(static_cast<size_t>(n) * c, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(n, c, k, input, idx, weight, output, true);
    return check_launch("interp_forward_kernel");
}

int tgn_weighted_gather(int n, int c, int k, const float* input, const int* idx, const float* weight, float* output, int fused, void* stream)
{
    if (n <= 0 || c <= 0) return TGN_OK;
    interp_forward_kernel<<<grid_for(static_cast<size_t>(n) * c, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(n, c, k, input, idx, weight, output, fused != 0);
    return check_launch("interp_forward_kernel");
}

int tgn_interpolation_backward(int n, int c, int k, const float* grad_output, const int* idx, const float* weight, float* grad_input, void* stream)
{
    if (n <= 0 || c <= 0) return TGN_OK;
    interp_backward_kernel<<<grid_for(static_cast<size_t>(n) * c, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(n, c, k, grad_output, idx, weight, grad_input);
    return check_launch("interp_backward_kernel");
}

int tgn_subtraction_forward(int n, int nsample, int c, const float* input1, const float* input2, const int* idx, float* output, void* stream)
{
    const size_t rows = static_cast<size_t>(n) * nsample;
    if (!rows || c <= 0) return TGN_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (c % 4 == 0 && aligned16(input1) && aligned16(input2) && aligned16(output))
        subtraction_forward_kernel<4><<<grid_for(rows * (c / 4), 256), 256, 0, st>>>(n, nsample, c, input1, input2, idx, output);
    else
        subtraction_forward_kernel<1><<<grid_for(rows * c, 256), 256, 0, st>>>(n, nsample, c, input1, input2, idx, output);
    return check_launch("subtraction_forward_kernel");
}

int tgn_subtraction_backward(int n, int nsample, int c, const int* idx, const float* grad_output, float* grad_input1, float* grad_input2, void* stream)
{
    if (n <= 0 || c <= 0 || nsample <= 0) return TGN_OK;
    subtraction_backward_kernel<<<grid_for(static_cast<size_t>(n) * c, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(n, nsample, c, idx, grad_output, grad_input1, grad_input2);
    return check_launch("subtraction_backward_kernel");
}

int tgn_aggregation_forward(int n, int nsample, int c, int w_c, const float* input, const float* position, const float* weight,
                            const int* idx, float* output, void* stream)
{
    if (n <= 0 || c <= 0) return TGN_OK;
    if (w_c <= 0) { set_error("aggregation: w_c must be positive"); return TGN_ERR_INVALID; }
    aggregation_forward_kernel<<<grid_for(static_cast<size_t>(n) * c, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(n, nsample, c, w_c, input, position, weight, idx, output);
    return check_launch("aggregation_forward_kernel");
}

int tgn_aggregation_backward(int n, int nsample, int c, int w_c, const float* input, const float* position, const float* weight,
                             const int* idx, const float* grad_output, float* grad_input, float* grad_position,
                             float* grad_weight, void* stream)
{
    if (n <= 0 || c <= 0) return TGN_OK;
    if (w_c <= 0) { set_error("aggregation: w_c must be positive"); return TGN_ERR_INVALID; }
    aggregation_backward_kernel<<<grid_for(static_cast<size_t>(n) * c, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(n, nsample, c, w_c, input, position, weight, idx, grad_output, grad_input, grad_position, grad_weight);
    return check_launch("aggregation_backward_kernel");
}

int tgn_gather_rows(int B, int N, int M, int C, const float* points, const int* idx, float* out, void* stream)
{
    if (B <= 0 || M <= 0 || C <= 0) return TGN_OK;
    if (B > 65535) { set_error("gather_rows: B=%d exceeds gridDim.y", B); return TGN_ERR_INVALID; }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (C % 4 == 0 && aligned16(points) && aligned16(out)) {
        dim3 grid(grid_for(static_cast<size_t>(M) * (C / 4), 256), B);
        batched_rows_gather_kernel<4><<<grid, 256, 0, st>>>(N, M, C, points, idx, out);
    } else {
        dim3 grid(grid_for(static_cast<size_t>(M) * C, 256), B);
        batched_rows_gather_kernel<1><<<grid, 256, 0, st>>>(N, M, C, points, idx, out);
    }
    return check_launch("batched_rows_gather_kernel");
}

int tgn_transpose_cn(int B, int C, int N, const float* in, float* out, void* stream)
{
    // in (B, C, N) -> out (B, N, C): rows R = C, cols = N in the kernel's naming
    if (B <= 0 || C <= 0 || N <= 0) return TGN_OK;
    if (B > 65535 || (C + 31) / 32 > 65535) { set_error("transpose: shape exceeds grid limits"); return TGN_ERR_INVALID; }
    // in (B, C rows, N cols): rows = C, cols = N in the kernels' naming
    if (C <= 8 && N >= 256) {
        dim3 g(std::min((N + 255) / 256, 4 * sm_count()), B);
        transpose_short_rows_kernel<8><<<g, 256, 0, static_cast<cudaStream_t>(stream)>>>(C, N, in, out);
        return check_launch("transpose_short_rows_kernel");
    }
    if (N <= 8 && C >= 256) {
        dim3 g(std::min((C + 255) / 256, 4 * sm_count()), B);
        transpose_short_cols_kernel<8><<<g, 256, 0, static_cast<cudaStream_t>(stream)>>>(C, N, in, out);
        return check_launch("transpose_short_cols_kernel");
    }
    dim3 grid((N + 31) / 32, (C + 31) / 32, B);
    transpose_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(C, N, in, out);
    return check_launch("transpose_kernel");
}

// ---- the reference's own launcher names (legacy default stream, no status) -----------------
void grouping_forward_cuda_launcher(int m, int nsample, int c, const float* input, const int* idx, float* output)
{ TGN_REPORT(tgn_grouping_forward(m, nsample, c, input, idx, output, nullptr)); }
void grouping_backward_cuda_launcher(int m, int nsample, int c, const float* grad_output, const int* idx, float* grad_input)
{ TGN_REPORT(tgn_grouping_backward(m, nsample, c, grad_output, idx, grad_input, nullptr)); }
void interpolation_forward_cuda_launcher(int n, int c, int k, const float* input, const int* idx, const float* weight, float* output)
{ TGN_REPORT(tgn_interpolation_forward(n, c, k, input, idx, weight, output, nullptr)); }
void interpolation_backward_cuda_launcher(int n, int c, int k, const float* grad_output, const int* idx, const float* weight, float* grad_input)
{ TGN_REPORT(tgn_interpolation_backward(n, c, k, grad_output, idx, weight, grad_input, nullptr)); }
void subtraction_forward_cuda_launcher(int n, int nsample, int c, const float* input1, const float* input2, const int* idx, float* output)
{ TGN_REPORT(tgn_subtraction_forward(n, nsample, c, input1, input2, idx, output, nullptr)); }
void subtraction_backward_cuda_launcher(int n, int nsample, int c, const int* idx, const float* grad_output, float* grad_input1, float* grad_input2)
{ TGN_REPORT(tgn_subtraction_backward(n, nsample, c, idx, grad_output, grad_input1, grad_input2, nullptr)); }
void aggregation_forward_cuda_launcher(int n, int nsample, int c, int w_c, const float* input, const float* position, const float* weight, const int* idx, float* output)
{ TGN_REPORT(tgn_aggregation_forward(n, nsample, c, w_c, input, position, weight, idx, output, nullptr)); }
void aggregation_backward_cuda_launcher(int n, int nsample, int c, int w_c, const float* input, const float* position, const float* weight, const int* idx, const float* grad_output, float* grad_input, float* grad_position, float* grad_weight)
{ TGN_REPORT(tgn_aggregation_backward(n, nsample, c, w_c, input, position, weight, idx, grad_output, grad_input, grad_position, grad_weight, nullptr)); }

}  // extern "C"
