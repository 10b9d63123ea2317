"""Fused PointTransformerLayer / TransitionDown forwards (csrc/pt_layer.cu, the tensor-core layer chain) against the fixtures written by
the reference's own blocks.py (tests/golden/ref_torch_blocks.npz) and against the oracle's float64 evaluation.  No reference
checkout is needed at run time; tests/test_gpu_reference_live.py holds the live comparisons."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import oracle as O  # noqa: E402
from toothgroupnetwork_b200 import blocks_fused, clouds  # noqa: E402

pytestmark = pytest.mark.gpu
GOLD = os.path.join(ROOT, "tests", "golden")
REL_TOL, FLOOR = 1e-4, 0.05


def elementwise(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float(((a - b).abs() / b.abs().clamp(min=FLOOR * float(b.abs().max()))).max())


class Layer(nn.Module):
    """the attribute layout of blocks.PointTransformerLayer (blocks.py:15-29), so that its state_dict loads"""

    def __init__(self, c, nsample, share=8):
        super().__init__()
        self.mid_planes = self.out_planes = c
        self.share_planes, self.nsample = share, nsample
        self.linear_q, self.linear_k, self.linear_v = nn.Linear(c, c), nn.Linear(c, c), nn.Linear(c, c)
        self.linear_p = nn.Sequential(nn.Linear(3, 3), nn.BatchNorm1d(3), nn.ReLU(inplace=True), nn.Linear(3, c))
        self.linear_w = nn.Sequential(nn.BatchNorm1d(c), nn.ReLU(inplace=True), nn.Linear(c, c // share), nn.BatchNorm1d(c // share),
                                      nn.ReLU(inplace=True), nn.Linear(c // share, c // share))


class Down(nn.Module):
    """blocks.TransitionDown with stride != 1 (blocks.py:48-57)"""

    def __init__(self, cin, cout, stride, nsample):
        super().__init__()
        self.stride, self.nsample = stride, nsample
        self.linear = nn.Linear(3 + cin, cout, bias=False)
        self.bn = nn.BatchNorm1d(cout)


def _state(fix, tag):
    pre = tag + "_state_"
    return {k[len(pre):]: torch.from_numpy(fix[k]) for k in fix.files if k.startswith(pre)}


@pytest.mark.parametrize("c", [32, 64])
@pytest.mark.parametrize("train_bn", [True, False])
def test_fused_layer_against_reference_fixture(c, train_bn):
    fix = np.load(os.path.join(GOLD, "ref_torch_blocks.npz"))
    tag = f"ptl{c}"
    layer = Layer(c, int(fix[tag + "_K"])).cuda().train(train_bn)
    layer.load_state_dict(_state(fix, tag))
    p, o, x = torch.from_numpy(fix["p"]).cuda(), torch.from_numpy(fix["o"]).cuda(), torch.from_numpy(fix[tag + "_x"]).cuda()
    with torch.no_grad():
        assert blocks_fused.pt_layer_fusable(layer, p, x, o)
        got = blocks_fused.pt_layer_forward(layer, [p, x, o])
    want = torch.from_numpy(fix[tag + ("_out_train" if train_bn else "_out_eval")])
    assert elementwise(got, want) < REL_TOL
    if train_bn:
        for k, v in layer.state_dict().items():
            if "running" in k:
                assert elementwise(v, torch.from_numpy(fix[f"{tag}_after_{k}"])) < 1e-4, k
            if "num_batches_tracked" in k:
                assert int(v) == 1


@pytest.fixture(params=[0, 1 << 30], ids=["warp_per_query", "cta_per_query"])
def schedule(request):
    from toothgroupnetwork_b200 import _lib as L
    old = L.load().tgn_pt_layer_set_cta_threshold(request.param)
    yield request.param
    L.load().tgn_pt_layer_set_cta_threshold(old)


@pytest.mark.parametrize("c,K,n", [(32, 36, 6000), (64, 7, 777), (128, 24, 1500), (256, 24, 400), (512, 24, 93)])
@pytest.mark.parametrize("train_bn", [True, False])
def test_fused_layer_against_oracle_float64(c, K, n, train_bn, schedule):
    torch.manual_seed(c)
    layer = Layer(c, K).train(train_bn)
    g = torch.Generator().manual_seed(1)
    for m in layer.modules():
        if isinstance(m, nn.BatchNorm1d):
            with torch.no_grad():
                m.weight.copy_(torch.rand(m.weight.shape, generator=g) + 0.5)
                m.bias.copy_(torch.randn(m.bias.shape, generator=g) * 0.1)
                m.running_mean.copy_(torch.randn(m.running_mean.shape, generator=g) * 0.1)
                m.running_var.copy_(torch.rand(m.running_var.shape, generator=g) + 0.5)
    state = {k: v.clone() for k, v in layer.state_dict().items()}
    p = clouds.dental_arch(n, 4)[0].contiguous()
    x = torch.randn(n, c, generator=g)
    o = torch.tensor([n], dtype=torch.int32)
    truth = O.point_transformer_layer(p, x, o, state, K, 8, train_bn, dtype=torch.float64)
    fp32 = O.point_transformer_layer(p, x, o, state, K, 8, train_bn, dtype=torch.float32)
    layer.cuda()
    with torch.no_grad():
        got = blocks_fused.pt_layer_forward(layer, [p.cuda(), x.cuda(), o.cuda()])
    e_ours, e_fp32 = elementwise(got, truth), elementwise(fp32, truth)
    assert e_ours <= max(REL_TOL, 2.0 * e_fp32), (e_ours, e_fp32)


@pytest.mark.parametrize("train_bn", [True, False])
def test_fused_transition_down_against_reference_fixture(train_bn):
    fix = np.load(os.path.join(GOLD, "ref_torch_blocks.npz"))
    td = Down(32, 64, 4, 16).cuda().train(train_bn)
    td.load_state_dict(_state(fix, "td"))
    p, o, x = torch.from_numpy(fix["p"]).cuda(), torch.from_numpy(fix["o"]).cuda(), torch.from_numpy(fix["td_x"]).cuda()
    with torch.no_grad():
        assert blocks_fused.transition_down_fusable(td, p, x, o)
        n_p, n_x, n_o = blocks_fused.transition_down_forward(td, [p, x, o])
    assert np.array_equal(n_p.cpu().numpy(), fix["td_p"]) and np.array_equal(n_o.cpu().numpy(), fix["td_o"])
    assert elementwise(n_x, torch.from_numpy(fix["td_out_train" if train_bn else "td_out_eval"])) < REL_TOL


def test_fused_paths_step_aside_under_autograd_and_for_other_shapes():
    layer = Layer(32, 16).cuda()
    p, x, o = torch.randn(100, 3).cuda(), torch.randn(100, 32).cuda(), torch.tensor([100], dtype=torch.int32).cuda()
    assert not blocks_fused.pt_layer_fusable(layer, p, x, o)            # parameters require grad and grad mode is on
    with torch.no_grad():
        assert blocks_fused.pt_layer_fusable(layer, p, x, o)
        assert not blocks_fused.pt_layer_fusable(Layer(48, 16).cuda(), p, torch.randn(100, 48).cuda(), o)
        assert not blocks_fused.pt_layer_fusable(layer, p.cpu(), x.cpu(), o.cpu())
