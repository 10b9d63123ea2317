// sa_mlp.cuh -- parameter block shared by the two engines of the fused set-abstraction body.
#pragma once
#include <cuda_runtime.h>

namespace tgn {

constexpr int kSaMaxLayers = 4;
constexpr int kSaMaxWidth = 128;

struct SaParams {
    int B, N, S, K, D;
    const float* xyz;        // (B,N,3)
    const float* feats;      // (B,N,D) point-major, or nullptr
    const float* new_xyz;    // (B,S,3)
    const int* gidx;         // (B,S,K)
    int xyz_first;           // 1: [xyz_rel, feats]  0: [feats, xyz_rel]
    int L;
    int ch[kSaMaxLayers + 1];
    const float* W[kSaMaxLayers];      // (C_{l+1}, C_l) row-major, BatchNorm folded
    const float* bias[kSaMaxLayers];
    float* out;              // (B, out_c_total, S)
    int out_c_total, out_c_offset;
    // filled by the launchers
    int cstride, wt_floats, gpt, chunks;
    int wt_resident;                 // fp32 engine: 1 = the weights of all layers stay in shared memory (wt_off), 0 = staged per layer
    int wt_off[kSaMaxLayers];        // float offsets of the layers' [cin][cout_pad] blocks
    int tiles_x;                     // fp32 engine: tiles per cloud (grid is flattened and persistent)
};

int sa_mlp_fp32_launch(SaParams p, cudaStream_t st);
bool sa_mlp_tc_supported(const SaParams& p);
int sa_mlp_tc_launch(SaParams p, cudaStream_t st, int groups_per_cta = 4);
bool sa_mlp_tcw_supported(const SaParams& p);     // wide hidden layers: tf32 first layer, bf16x2-split later layers
int sa_mlp_tcw_launch(SaParams p, cudaStream_t st);

}  // namespace tgn
