"""GPU: the boundary network's c = 16 point-transformer layers (tgnet_bdl: PointTransformerLayer(16, 16, 8, 36)) on the fused
kernel's half-warp schedule, through blocks_fused -- against the reference's own blocks.py output (tests/golden/
ref_torch_blocks16.npz), against the oracle in float64, under autograd (where the reference's code keeps running) and, when the
reference snapshot is staged, against the reference's layer and the whole boundary network live on the same GPU."""
import os
import sys

import numpy as np
import pytest
import torch

from oracle import ref_cuda, ref_models
from test_gpu_blocks import GOLD, REL_TOL, Layer, _layer_against_oracle, _state, elementwise
from toothgroupnetwork_b200 import _lib as L
from toothgroupnetwork_b200 import blocks_fused, clouds

pytestmark = pytest.mark.gpu
live = pytest.mark.skipif(not (ref_models.available() and ref_cuda.available()), reason="reference snapshot not staged")


@pytest.mark.parametrize("train_bn", [True, False])
def test_fused_c16_layer_against_reference_fixture(train_bn):
    fix = np.load(os.path.join(GOLD, "ref_torch_blocks16.npz"))
    layer = Layer(16, int(fix["ptl16_K"])).cuda().train(train_bn)
    layer.load_state_dict(_state(fix, "ptl16"))
    p, o, x = torch.from_numpy(fix["p"]).cuda(), torch.from_numpy(fix["o"]).cuda(), torch.from_numpy(fix["ptl16_x"]).cuda()
    with torch.no_grad():
        assert blocks_fused.pt_layer_fusable(layer, p, x, o)
        launches = L.launch_count()
        got = blocks_fused.pt_layer_forward(layer, [p, x, o])
        assert L.launch_count() > launches
    assert elementwise(got, torch.from_numpy(fix["ptl16_out_train" if train_bn else "ptl16_out_eval"])) < REL_TOL
    for k, v in layer.state_dict().items():
        if "running" in k:
            want = torch.from_numpy(fix[f"ptl16_after_{k}"] if train_bn else fix[f"ptl16_state_{k}"])
            assert elementwise(v, want) < 1e-4, k
        if "num_batches_tracked" in k:
            assert int(v) == int(train_bn)


@pytest.mark.parametrize("K,n,crops", [(36, 6000, 1), (36, 16 * 384, 16)])
@pytest.mark.parametrize("train_bn", [True, False])
def test_fused_c16_layer_against_oracle_float64(K, n, crops, train_bn):
    _layer_against_oracle(16, K, n, train_bn, offset=0.0, crops=crops)


def test_c16_layer_steps_aside_under_autograd():
    """backward passes stay on the reference's code: with grad enabled and trainable parameters the layer is not fused"""
    layer = Layer(16, 36).cuda()
    p, x, o = torch.randn(100, 3).cuda(), torch.randn(100, 16).cuda(), torch.tensor([100], dtype=torch.int32).cuda()
    assert not blocks_fused.pt_layer_fusable(layer, p, x, o)
    assert not blocks_fused.pt_layer_fusable(layer, p, x.requires_grad_(), o)
    with torch.no_grad():
        assert blocks_fused.pt_layer_fusable(layer, p, x, o)


# ------------------------------------------------------------------------ live, against the reference on the same GPU
_world = {}


@pytest.fixture
def fp32_library():
    """the reference's Linear / Conv layers in plain fp32 (no TF32), as the live comparisons run them"""
    saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved


def world(ops):
    if ops not in _world:
        _world[ops] = ref_models.World(ops)
    return _world[ops]


@live
@pytest.mark.parametrize("train_bn", [True, False])
def test_fused_c16_layer_vs_reference_layer(train_bn, fp32_library):
    """blocks.PointTransformerLayer(16, 16, 8, 36) at n = 24 000 under no_grad: the fused layer against the reference's own layer on
    the reference's operators, and against that layer in float64 with the same neighbour indices (the bar of
    test_gpu_reference_live.test_fused_point_transformer_layer_vs_reference_layer)"""
    c, K, n = 16, 36, 24000
    name = "models.modules.cbl_point_transformer.blocks"
    p = clouds.dental_arch(n, 4)[0].cuda()
    g = torch.Generator(device="cuda").manual_seed(2)
    x = torch.randn(n, c, device="cuda", generator=g)
    o = torch.tensor([n], dtype=torch.int32, device="cuda")
    with world("reference"), torch.no_grad():
        torch.manual_seed(0)
        ref = world("reference").mod(name).PointTransformerLayer(c, c, 8, K).cuda().train(train_bn)
        g2 = torch.Generator().manual_seed(3)
        for b in (ref.linear_p[1], ref.linear_w[0], ref.linear_w[3]):
            b.weight.copy_(torch.rand(b.weight.shape, generator=g2) + 0.5)
            b.bias.copy_(torch.randn(b.bias.shape, generator=g2) * 0.1)
            b.running_mean.copy_(torch.randn(b.running_mean.shape, generator=g2) * 0.1)
            b.running_var.copy_(torch.rand(b.running_var.shape, generator=g2) + 0.5)
        state = {k: v.clone() for k, v in ref.state_dict().items()}
        want = ref([p, x, o])
        ref_state_after = {k: v.clone() for k, v in ref.state_dict().items()}
        ref.load_state_dict(state)
        po = world("reference").mod("external_libs.pointops.functions.pointops")
        saved = po.knnquery
        po.knnquery = lambda k, xyz, new_xyz, off, noff: saved(k, xyz.float().contiguous(), new_xyz.float().contiguous(), off, noff)
        try:
            truth = ref.double()([p.double(), x.double(), o])
        finally:
            po.knnquery = saved
            ref.float()
    with world("b200"), torch.no_grad():
        ours = world("b200").mod(name).PointTransformerLayer(c, c, 8, K).cuda().train(train_bn)
        ours.load_state_dict(state)
        assert blocks_fused.pt_layer_fusable(ours, p, x, o)
        launches = L.launch_count()
        got = ours([p, x, o])
        assert L.launch_count() - launches >= 2
    err, e_ours, e_ref = elementwise(got, want), elementwise(got, truth), elementwise(want, truth)
    assert err < REL_TOL or e_ours <= max(REL_TOL, 2.0 * e_ref), (err, e_ours, e_ref)
    if train_bn:
        for k, v in ref_state_after.items():
            if "running" in k:
                assert elementwise(ours.state_dict()[k], v) < 1e-4, k
            if "num_batches_tracked" in k:
                assert int(ours.state_dict()[k]) == int(v)


@live
def test_boundary_network_vs_reference(fp32_library):
    """GroupingNetworkModule with the boundary network's parameters, no_grad, test=True (as the tgnet inference pipeline calls it),
    train-mode BatchNorm: model_parity's verdict on every output, crops identical"""
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "scripts"))
    import model_parity as mp
    feats, labels = mp.make_inputs(24000)
    res = mp.case_tgn_infer([world("reference"), world("b200")], feats, labels, True, mp.Timer(), params=mp.TGNB_PARAMS, test=True)
    assert res["tensors"]["nn_crop_indexes"]["bitwise"]
    assert res["verdict"]["pass"], res["verdict"]
