"""GPU: the split-fp16 group-MLP kernel (csrc/sa_mlp_tc.cu) at the edges of its range guard, one launch at a time against the
float64 restatement (oracle/sa_group.py) with the per-engine bound of test_gpu_sa_group.py.

A tile is computed in split fp16 unless one of its layer-0 inputs or inner activations is non-finite or |v| >= 2^15, or is
nonzero below 2^-14 where the consuming layer's biases do not cover the absolute error of such tiny operands; a weight out of
range (non-finite, |w| >= 2^4, or nonzero below 2^-16) sends every tile to the 3xTF32 kernel.  Both paths must meet the same
bound, engine 5 must equal engine 2 bit for bit, and a cloud must equal its own launch whichever of its tiles fall back."""
import pytest
import torch

from test_gpu_sa_group import TC, TC_HALF, Inputs, check_bound, launch, make_net, truth_of

pytestmark = pytest.mark.gpu


def _bits(t):
    return t.contiguous().view(torch.int32)


def _set_feats(inp, feats):
    inp.feats = feats.contiguous()
    inp.dev[1] = inp.feats.cuda()


def _covering_biases(bs, floor=0.05):
    """biases at least `floor` in magnitude: every layer's biases cover the error of tiny operands"""
    return [torch.where(b.abs() < floor, torch.full_like(b, floor), b) for b in bs]


def _check(inp, ws, bs, tag, xyz_first=1, clouds_alone=True):
    truth, mag = truth_of(inp, ws, bs, xyz_first)
    ch = [3 + inp.D] + [w.shape[0] for w in ws]
    outs = {}
    for e in (TC, TC_HALF):
        got = launch(inp, ws, bs, e, xyz_first)
        check_bound(got, truth, mag, e, ch, tag)
        assert torch.equal(_bits(got), _bits(launch(inp, ws, bs, e, xyz_first))), f"engine {e}: two launches differ"
        outs[e] = got
    assert torch.equal(_bits(outs[TC_HALF]), _bits(outs[TC]))
    if clouds_alone:
        for b in range(inp.B):
            assert torch.equal(_bits(outs[TC][b:b + 1]), _bits(launch(inp.cloud(b), ws, bs, TC, xyz_first))), f"{tag}: cloud {b}"
    return outs


# ------------------------------------------------------------------------------------------------- the |v| >= 2^15 guard
@pytest.mark.parametrize("value", [32767.0, 32768.0, 32769.0, -32767.5, -40000.0])
def test_inputs_around_two_to_the_fifteen(value):
    inp = Inputs(3, 2000, 61, 32, 6, seed=41)
    f = inp.feats.clone()
    f[1, ::37, 4] = value                      # cloud 1 only: some of its tiles take the fallback above 2^15
    _set_feats(inp, f)
    ws, bs = make_net([9, 32, 32, 64], seed=5)
    _check(inp, ws, bs, f"input {value}")


@pytest.mark.parametrize("scale", [1.0, 4.0, 12.0])
def test_inner_activations_around_two_to_the_fifteen(scale):
    """features up to ~5e3 (logspace(-3, 3)) through a layer-0 weight scaled up: the first hidden layer's activations straddle
    2^15, so whole tiles flip between the split-fp16 and the 3xTF32 path"""
    inp = Inputs(3, 2000, 77, 16, 6, seed=43)
    ws, bs = make_net([9, 32, 48, 64], seed=6)
    ws[0] = ws[0] * scale
    _check(inp, ws, bs, f"layer-0 weights x{scale}")


@pytest.mark.parametrize("widths", [[32, 32, 64], [48, 64], [64]])
def test_one_large_weight_flags_every_tile(widths):
    inp = Inputs(3, 2000, 61, 32, 6, seed=44)
    ws, bs = make_net([9] + widths, seed=7)
    ws[-1][1, 2] = 40000.0
    _check(inp, ws, bs, f"w={widths} one weight 4e4")


# ------------------------------------------------------------------------------------------------------ small magnitudes
TINY = [2.0 ** -14 * (1 - 2.0 ** -12), 2.0 ** -14, 2.0 ** -14 * (1 + 2.0 ** -10), 2.0 ** -17, 2.0 ** -24, 2.0 ** -25,
        2.0 ** -30, 1e-30, 1e-40]


@pytest.mark.parametrize("covering", [True, False])
@pytest.mark.parametrize("widths", [[32, 32, 64], [64, 48]])
def test_values_straddling_fp16_normal_range(covering, widths):
    """features and xyz offsets across fp16's subnormal band and below it, with biases that cover the absolute error of tiny
    operands (split-fp16 path) or biases of zero (those tiles fall back)"""
    inp = Inputs(2, 2000, 61, 32, 6, seed=45)
    gen = torch.Generator().manual_seed(3)
    f = inp.feats.clone()
    pick = torch.randint(0, len(TINY), f.shape, generator=gen)
    sign = torch.where(torch.rand(f.shape, generator=gen) < 0.5, -1.0, 1.0)
    tiny = torch.tensor(TINY)[pick] * sign
    mask = torch.rand(f.shape, generator=gen) < 0.5
    f = torch.where(mask, tiny.float(), f)
    _set_feats(inp, f)
    ws, bs = make_net([9] + widths, seed=8, zero_bias=False)
    bs = _covering_biases(bs) if covering else [torch.zeros_like(b) for b in bs]
    _check(inp, ws, bs, f"w={widths} covering={covering}")


def test_tiny_weights():
    """weights in [2^-16, 2^-14) stay on the split-fp16 path; one below 2^-16 sends every tile to the 3xTF32 kernel"""
    inp = Inputs(2, 2000, 61, 32, 6, seed=46)
    ws, bs = make_net([9, 32, 32, 64], seed=9, zero_bias=False)
    bs = _covering_biases(bs)
    ws[1][::5, ::3] = 2.0 ** -15
    _check(inp, ws, bs, "weights 2^-15")
    ws[2][3, 4] = 2.0 ** -20
    _check(inp, ws, bs, "one weight 2^-20")


# ----------------------------------------------------------------------------------------------------- non-finite inputs
@pytest.mark.parametrize("bad", [float("nan"), float("inf"), float("-inf")])
def test_non_finite_inputs(bad):
    """a non-finite input sends its tile to the 3xTF32 kernel: the launch is deterministic, engine 5 equals engine 2 bit for
    bit, the cloud equals its own launch, and the clouds without one stay within the bound"""
    inp = Inputs(3, 2000, 61, 32, 6, seed=47)
    f = inp.feats.clone()
    f[1, 100:2000:97, 2] = bad
    _set_feats(inp, f)
    ws, bs = make_net([9, 32, 32, 64], seed=10)
    outs = {}
    for e in (TC, TC_HALF):
        outs[e] = launch(inp, ws, bs, e)
        assert torch.equal(_bits(outs[e]), _bits(launch(inp, ws, bs, e)))
    assert torch.equal(_bits(outs[TC_HALF]), _bits(outs[TC]))
    for b in range(3):
        assert torch.equal(_bits(outs[TC][b:b + 1]), _bits(launch(inp.cloud(b), ws, bs, TC))), f"cloud {b}"
    for b in (0, 2):
        one = Inputs.__new__(Inputs)
        one.B, one.N, one.S, one.K, one.D = 1, inp.N, inp.S, inp.K, inp.D
        one.xyz, one.feats, one.new_xyz, one.gidx = (t[b:b + 1] for t in (inp.xyz, inp.feats, inp.new_xyz, inp.gidx))
        truth, mag = truth_of(one, ws, bs, 1)
        check_bound(outs[TC][b:b + 1], truth, mag, TC, [9, 32, 32, 64], f"finite cloud {b}")


# ---------------------------------------------------------------------------------- none, some and all tiles flagged
@pytest.mark.parametrize("flagged", ["none", "some", "all"])
@pytest.mark.parametrize("widths", [[32, 32, 64], [48, 48, 128], [16, 40]])
def test_flagged_share(flagged, widths):
    inp = Inputs(4, 4000, 300, 32, 6, seed=48, kind="offset")
    f = inp.feats.clone()
    f[..., 3:] = f[..., 3:].clamp(-1000.0, 1000.0)            # 'none': every operand in range
    f = torch.where(f.abs() < 2.0 ** -10, torch.full_like(f, 2.0 ** -10), f)
    ws, bs = make_net([9] + widths, seed=11, zero_bias=False)
    bs = _covering_biases(bs)
    if flagged == "some":
        f[2, ::50, 5] = 1e5
    if flagged == "all":
        ws[0][0, 0] = float("inf")
    _set_feats(inp, f)
    if flagged == "all":
        # an infinite weight: every engine's result is non-finite somewhere; only determinism and equality are checked
        outs = {e: launch(inp, ws, bs, e) for e in (TC, TC_HALF)}
        assert torch.equal(_bits(outs[TC_HALF]), _bits(outs[TC]))
        assert torch.equal(_bits(outs[TC][1:2]), _bits(launch(inp.cloud(1), ws, bs, TC)))
        return
    _check(inp, ws, bs, f"w={widths} flagged={flagged}")


def test_one_cloud_with_a_flagged_tile():
    """B = 40 clouds, one tile of cloud 17 out of range: every cloud equals its own launch bit for bit"""
    inp = Inputs(40, 600, 40, 32, 6, seed=49, kind="offset", radius=0.1)
    f = inp.feats.clone()
    f[17, 3, 4] = 50000.0
    _set_feats(inp, f)
    ws, bs = make_net([9, 32, 32, 64], seed=12)
    full = launch(inp, ws, bs, TC)
    for b in range(40):
        assert torch.equal(_bits(full[b:b + 1]), _bits(launch(inp.cloud(b), ws, bs, TC))), f"cloud {b}"
    truth, mag = truth_of(inp, ws, bs, 1)
    check_bound(full, truth, mag, TC, [9, 32, 32, 64], "one flagged cloud")
