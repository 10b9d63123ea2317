// ballquery.cuh -- internal interface between the ball-query kernels.
#pragma once
#include <cuda_runtime.h>

namespace tgn {

// |p|^2 as torch.sum(p ** 2, -1) rounds it ON THE GPU (square_distance :39-40), measured with torch 2.11
// (scripts/diag_sumsq.py): a strided reduction (the permuted views the reference's modules
// pass) accumulates in index order, (x*x + y*y) + z*z -- the same as torch on the CPU; a CONTIGUOUS (..., 3) tensor
// (e.g. new_xyz fresh out of index_points) goes through the vectorised reduce path and comes out as
// (x*x + z*z) + y*y.  `alt` selects the second form; the Python layer derives it from the layout the reference's
// own call would see, per operand.
__device__ __forceinline__ float sq_norm_unfused(float x, float y, float z, bool alt) {
    return alt ? __fadd_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(z, z)), __fmul_rn(y, y))
               : __fadd_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)), __fmul_rn(z, z));
}
__device__ __forceinline__ float sq_dist_expanded(float ax, float ay, float az, float an, float bx, float by, float bz,
                                                  float bn) {
    float dot = __fmul_rn(ax, bx);
    dot = __fmaf_rn(ay, by, dot);
    dot = __fmaf_rn(az, bz, dot);
    float d = __fmul_rn(-2.0f, dot);
    d = __fadd_rn(d, an);
    return __fadd_rn(d, bn);
}

// Per-call scratch of the grid ball query (ballquery_grid.cu), all per cloud b.
struct BqGridWs {
    float4* rec;       // [B][N]    points sorted by (index window, cell): (x, y, z, bits of the original index)
    int* cell_start;   // [B][kMaxCells + 1]  first sorted position of key window * cells + cell
    float4* org;       // [B]      grid origin x, y, z, 1 / cell size
    int4* dim;         // [B]      nx, ny, nz, log2 of the index-window size
    float4* bnd;       // [B]      max |p|^2, max |coordinate|
    int* flag;         // [B]      1: answered by the grid kernel, 0: left to the tile kernel
};

int bq_grid_max_points();
// Byte size of the scratch; fills `offsets` with the byte offsets of the arrays (as pointers from 0).
size_t bq_grid_workspace_bytes(int B, int N, BqGridWs* offsets);
// force: 0 = per-cloud estimate decides, 1 = every cloud takes the grid kernel.
// order: bit 0 / bit 1 = |new_xyz|^2 / |xyz|^2 rounded as torch's contiguous reduce does (see ballquery.cu).
int bq_grid_launch(int B, int N, int S, float r2, int nsample, const float* xyz, const float* new_xyz, void* group_idx,
                   bool idx64, int force, int order, const BqGridWs& ws, cudaStream_t st);

}  // namespace tgn
