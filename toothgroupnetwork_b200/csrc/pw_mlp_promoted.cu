// pw_mlp_promoted.cu -- the promoted-accumulation form of the layer kernel (pw_layer.cuh), launched by tgn_pw_layer_forward for
// accum = 1: tiles of 128 channels x 128 rows, each consumer warpgroup's m64n128 chunk accumulator added into an fp32 register
// total with a round-to-nearest FADD every kPromoteSteps K-steps of 16 (6 MMAs per chunk).  Kept in a
// translation unit of its own so that the accumulate-everything form in pw_mlp.cu compiles exactly as before.
#include "pw_layer.cuh"

namespace tgn {
namespace pw {

// K-steps of 16 per promoted chunk.  Two (one pipeline stage, 12 MMAs) left DGCNN's eval-mode conv8 up to 2.1x the reference fp32
// run's distance from float64 on an H100; one step (6 MMAs, a second wait inside each stage) is what DESIGN §3.12 records.
constexpr int kPromoteSteps = 1;

int pw_layer_launch_promoted(PwArgs& a, cudaStream_t stream)
{
    return pw_layer_launch<kPromoteNT, kPromoteSteps>(a, stream, "pw_layer_kernel (promoted)");
}

}  // namespace pw
}  // namespace tgn
