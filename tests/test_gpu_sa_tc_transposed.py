"""GPU: the 3xTF32 group-MLP engine's transposed inner layers (csrc/sa_mlp_tc.cu) at the edges of their schedule, one launch
at a time against the float64 restatement (oracle/sa_group.py), with the per-engine bound of test_gpu_sa_group.py.

Every inner layer runs as D^T[channel, row] = W * X^T on 64 weight rows and the tile's 128 rows:
* inner widths up to 32 pack W_hi and W_lo of a channel into one 64-row operand and add the two halves in the epilogue;
  wider ones hold one channel per row.  Each case below names the padded width NP it runs at, with the real widths
  short of NP (padded channels), and channel counts that end inside a warp's 8 or 16 channels;
* the epilogue rewrites the tile's operand in place, so chains of two and three inner layers are covered;
* K of 1, 7, 32, 100 and 128 (128 / K neighbourhoods per tile, a partial last tile when S is not a multiple of it).
Engine 5 (half-size CTAs) must equal engine 2 bit for bit, and each cloud of a launch must equal its own launch."""
import pytest
import torch

from test_gpu_sa_group import TC, TC_HALF, Inputs, launch, make_net, run_engines

pytestmark = pytest.mark.gpu

# (inner widths + last width, NP)
NETS = [
    ([16, 16], 16),            # packed, no padding
    ([9, 5, 40], 16),          # packed, padded, two inner layers, the last layer's channels end inside a warp
    ([24, 64], 32),            # packed, channels 16..23 in warp 2, warp 3 only padding
    ([32, 32, 32, 64], 32),    # packed, three inner layers
    ([40, 100], 48),           # one channel per row, padded to 48; 64-row M holds 48 channels
    ([57, 33], 64),            # one channel per row, channels 57..63 padded
    ([64, 64], 64),            # one channel per row, no padding
    ([33, 128], 48),           # one past the packed limit; two 64-channel passes of the last layer
]


def _cases():
    out = []
    for i, (widths, np_) in enumerate(NETS):
        for j, K in enumerate((1, 7, 32, 100, 128)):
            gpt = 128 // K
            S = 3 * gpt + 1 + (i + j) % max(gpt - 1, 1) if gpt > 1 else 5      # a partial last tile unless K divides 128 exactly
            out.append((1 + (i + j) % 3, K, S, 6 if (i + j) % 2 else 13, (i + j) % 2, widths, np_))
    return out


@pytest.mark.parametrize("B,K,S,D,xyz_first,widths,np_", _cases())
def test_transposed_inner_layers_against_float64(B, K, S, D, xyz_first, widths, np_):
    inp = Inputs(B, 2000, S, K, D, seed=17 * K + S + D, kind="arch" if K % 2 == 0 else "offset")
    ws, bs = make_net([3 + D] + widths, seed=7 * len(widths) + K)
    outs, truth = run_engines(inp, ws, bs, xyz_first, (TC, TC_HALF), f"NP={np_} B={B} S={S} K={K} D={D} w={widths}")
    assert torch.equal(outs[TC_HALF], outs[TC])
    for b in range(B):
        assert torch.equal(outs[TC][b:b + 1], launch(inp.cloud(b), ws, bs, TC, xyz_first)), f"cloud {b}"


def test_many_tiles_per_group():
    """more tiles than the persistent CTAs' groups: each group runs its chain over many tiles, the operand rewritten
    between them; the 128-row tiles of K = 32 and a partial one at the end of every cloud"""
    inp = Inputs(4, 6000, 1023, 32, 6, seed=5)
    ws, bs = make_net([9, 32, 32, 64], seed=11)
    outs, _ = run_engines(inp, ws, bs, 1, (TC, TC_HALF), "many tiles")
    assert torch.equal(outs[TC_HALF], outs[TC])
    assert torch.equal(outs[TC][3:4], launch(inp.cloud(3), ws, bs, TC))
