"""The reference's CALLERS of the hot path, restated as small models, running on the new ops
(BASELINE configs C3 / C4 at reduced size; the reference's own models/*.py cannot travel to the
GPU box).  Each block is written twice: once on this package's operator API exactly the way the
reference's module calls it, once in the reference's underlying formulation (torch advanced
indexing / dense ops, evaluated on the same device or by the CPU oracle).  Forward values and
gradients must agree.

  * TransitionDown      models/modules/cbl_point_transformer/blocks.py:59-79
  * PointTransformerLayer (grouping / subtraction / aggregation core)   blocks.py:31-44
  * TransitionUp        blocks.py:108-110
  * PointNet++ MSG encoder + FP decoder   models/modules/tsg_centroid_module.py:10-17,30-48
"""
import numpy as np
import pytest
import torch
import torch.nn as nn

from oracle import oracle
from toothgroupnetwork_b200 import clouds, pointops
from toothgroupnetwork_b200 import pointnet2_utils as pn2

pytestmark = pytest.mark.gpu


def rel_err(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).abs().max() / (b.abs().max() + 1e-30))


def _i32(v):
    return torch.tensor(v, dtype=torch.int32, device="cuda")


def test_transition_down_forward_backward():
    """FPS -> gather -> queryandgroup -> Linear -> BN -> ReLU -> MaxPool, two clouds in a batch."""
    torch.manual_seed(0)
    n1, n2, c, k, stride = 3000, 1200, 16, 12, 4
    p = torch.cat([clouds.dental_arch(n1, 1)[0], clouds.dental_arch(n2, 2)[0]]).cuda()
    x = torch.randn(n1 + n2, c, device="cuda")
    o = _i32([n1, n1 + n2])
    n_o = _i32([n1 // stride, n1 // stride + n2 // stride])
    linear = nn.Linear(3 + c, 32, bias=False).cuda()
    bn = nn.BatchNorm1d(32).cuda()
    pool = nn.MaxPool1d(k)

    def block(xin, group_fn):
        idx = pointops.furthestsampling(p, o, n_o)
        n_p = p[idx.long(), :]
        g = group_fn(xin, n_p)
        h = torch.relu(bn(linear(g).transpose(1, 2).contiguous()))
        return pool(h).squeeze(-1), idx

    x1 = x.clone().requires_grad_(True)
    out1, idx1 = block(x1, lambda xin, n_p: pointops.queryandgroup(k, p, n_p, xin, None, o, n_o, use_xyz=True))
    out1.square().sum().backward()
    g_x1, g_w1 = x1.grad.clone(), linear.weight.grad.clone()
    linear.weight.grad = None

    # FPS indices: oracle
    want_idx = oracle.furthestsampling(p.cpu().numpy(), o.cpu().numpy(), n_o.cpu().numpy())
    assert np.array_equal(idx1.cpu().numpy(), want_idx)

    def ref_group(xin, n_p):      # pointops.py:88-100 in the reference's own formulation
        kidx, _ = pointops.knnquery(k, p, n_p, o, n_o)
        gx = p[kidx.view(-1).long(), :].view(-1, k, 3) - n_p.unsqueeze(1)
        gf = xin[kidx.view(-1).long(), :].view(-1, k, c)
        return torch.cat((gx, gf), -1)

    x2 = x.clone().requires_grad_(True)
    out2, _ = block(x2, ref_group)
    out2.square().sum().backward()
    assert rel_err(out1, out2) < 1e-6
    assert rel_err(g_x1, x2.grad) < 1e-4
    assert rel_err(g_w1, linear.weight.grad) < 1e-4


def test_point_transformer_layer_core():
    """Vector attention core: w = softmax(mlp(x_k[idx] - x_q + p_r)); out = sum((x_v[idx] + p_r) * w),
    written with the Subtraction / Aggregation kernels and with dense torch ops."""
    torch.manual_seed(1)
    n, c, k, s = 2500, 32, 16, 8
    p = clouds.dental_arch(n, 3)[0].cuda()
    o = _i32([n])
    x_q = torch.randn(n, c, device="cuda", requires_grad=True)
    x_k = torch.randn(n, c, device="cuda", requires_grad=True)
    x_v = torch.randn(n, c, device="cuda", requires_grad=True)
    p_r = torch.randn(n, k, c, device="cuda", requires_grad=True)
    w_lin = torch.randn(c // s, c, device="cuda") * 0.1
    idx, _ = pointops.knnquery(k, p, p, o, o)

    def finish(diff, v_plus_p=None, use_kernel=False):
        w = torch.softmax((diff + p_r) @ w_lin.t(), dim=1)                    # (n,k,c/s)
        if use_kernel:
            return pointops.aggregation(x_v, p_r, w.contiguous(), idx)
        return ((x_v[idx.long()] + p_r).view(n, k, s, c // s) * w.unsqueeze(2)).sum(1).reshape(n, c)

    out_a = finish(pointops.subtraction(x_k, x_q, idx) * -1.0, use_kernel=True)
    out_a.square().sum().backward()
    grads_a = [t.grad.clone() for t in (x_q, x_k, x_v, p_r)]
    for t in (x_q, x_k, x_v, p_r):
        t.grad = None
    # dense formulation; note subtraction(in1,in2) = in1[n] - in2[idx]: (x_k - x_q[idx]) * -1 == x_q[idx] - x_k[n]
    out_b = finish(x_q[idx.long()] - x_k.unsqueeze(1))
    # aggregation weights cycle over channels as c % w_c (aggregation_cuda_kernel.cu:12): the dense form
    # above views channels as (s, c/s), i.e. weight index = channel % (c/s) as well
    out_b.square().sum().backward()
    assert rel_err(out_a, out_b) < 1e-5
    # x_k[n] is constant along the softmax axis, so its true gradient is 0 (both paths return
    # rounding noise ~1e-8): compare every gradient on the scale of the largest one
    scale = max(float(t.grad.abs().max()) for t in (x_q, x_k, x_v, p_r))
    for ga, t in zip(grads_a, (x_q, x_k, x_v, p_r)):
        assert float((ga - t.grad).abs().max()) < 1e-4 * scale


def test_transition_up_interpolation():
    torch.manual_seed(2)
    n1, n2, c = 4000, 1000, 24
    p1 = clouds.dental_arch(n1, 4)[0].cuda()
    fps = pointops.furthestsampling(p1, _i32([n1]), _i32([n2]))
    p2 = p1[fps.long()].contiguous()
    x2 = torch.randn(n2, c, device="cuda", requires_grad=True)
    up = pointops.interpolation(p2, p1, x2, _i32([n2]), _i32([n1]))
    up.square().sum().backward()
    g_kernel = x2.grad.clone()
    x2.grad = None
    idx, dist = pointops.knnquery(3, p2, p1, _i32([n2]), _i32([n1]))       # pointops.py:170-179
    rec = 1.0 / (dist + 1e-8)
    w = rec / rec.sum(1, keepdim=True)
    ref = torch.zeros(n1, c, device="cuda")
    for i in range(3):
        ref = ref + x2[idx[:, i].long(), :] * w[:, i].unsqueeze(-1)
    ref.square().sum().backward()
    assert rel_err(up, ref) < 1e-5
    assert rel_err(g_kernel, x2.grad) < 1e-4


def _rand_bn(module, gen):
    for m in module.modules():
        if isinstance(m, (nn.BatchNorm1d, nn.BatchNorm2d)):
            with torch.no_grad():
                m.weight.copy_(torch.rand(m.weight.shape, generator=gen) + 0.5)
                m.bias.copy_(torch.randn(m.bias.shape, generator=gen) * 0.1)
                m.running_mean.copy_(torch.randn(m.running_mean.shape, generator=gen) * 0.1)
                m.running_var.copy_(torch.rand(m.running_var.shape, generator=gen) + 0.5)


def _params(convs, bns):
    return [oracle.MlpParams(c.weight.detach().cpu().reshape(c.weight.shape[0], -1), c.bias.detach().cpu(), b.weight.detach().cpu(),
                             b.bias.detach().cpu(), b.running_mean.detach().cpu(), b.running_var.detach().cpu(), b.eps)
            for c, b in zip(convs, bns)]


def test_pointnetpp_msg_encoder_decoder_eval_matches_oracle():
    """tsg_centroid_module-shaped U-Net at reduced size: 3 MSG set abstractions (fused tensor-core /
    fp32 engines, or the unfused CUDA path where widths exceed 128) + 3 feature propagations, eval
    BN; outputs within 1e-4 relative of the CPU oracle stack."""
    torch.manual_seed(3)
    gen = torch.Generator().manual_seed(5)
    B, N = 2, 6000
    feats = torch.cat([clouds.arch_features(N, 30), clouds.arch_features(N, 31)], 0)
    sa1 = pn2.PointNetSetAbstractionMsg(512, [0.05, 0.1], [32, 64], 6, [[32, 32], [32, 32]])
    sa2 = pn2.PointNetSetAbstractionMsg(256, [0.1, 0.2], [32, 64], 64, [[64, 128], [64, 128]])
    sa3 = pn2.PointNetSetAbstractionMsg(64, [0.2, 0.4], [32, 64], 256, [[196, 256], [196, 256]])
    fp3 = pn2.PointNetFeaturePropagation(768, [256, 256])
    fp2 = pn2.PointNetFeaturePropagation(320, [128, 128])
    fp1 = pn2.PointNetFeaturePropagation(128 + 6, [64, 32])
    net = nn.ModuleList([sa1, sa2, sa3, fp3, fp2, fp1])
    _rand_bn(net, gen)
    net = net.cuda().eval()
    with torch.no_grad():
        l0 = feats.cuda()
        x0 = l0[:, :3].contiguous()
        x1, f1 = sa1(x0, l0)
        x2, f2 = sa2(x1, f1)
        x3, f3 = sa3(x2, f2)
        g2 = fp3(x2, x3, f2, f3)
        g1 = fp2(x1, x2, f1, g2)
        g0 = fp1(x0, x1, l0, g1)

    def msg(mod, xyz, pts):
        return oracle.set_abstraction_msg(xyz, pts, mod.npoint, mod.radius_list, mod.nsample_list,
                                          [_params(c, b) for c, b in zip(mod.conv_blocks, mod.bn_blocks)])

    def fp(mod, a, b_, pa, pb):
        return oracle.feature_propagation(a, b_, pa, pb, _params(mod.mlp_convs, mod.mlp_bns))

    c0 = feats
    cx0 = c0[:, :3].contiguous()
    cx1, cf1 = msg(sa1, cx0, c0)
    cx2, cf2 = msg(sa2, cx1, cf1)
    cx3, cf3 = msg(sa3, cx2, cf2)
    cg2 = fp(fp3, cx2, cx3, cf2, cf3)
    cg1 = fp(fp2, cx1, cx2, cf1, cg2)
    cg0 = fp(fp1, cx0, cx1, c0, cg1)
    assert torch.equal(x3.cpu(), cx3) and torch.equal(x1.cpu(), cx1)
    for got, want in ((f1, cf1), (f2, cf2), (f3, cf3), (g2, cg2), (g1, cg1), (g0, cg0)):
        assert rel_err(got, want) < 1e-4


@pytest.mark.gpu
def test_host_pipeline_matches_direct_module_call():
    """pinned host -> chunks -> pinned host gives the same bits as one call on the whole batch
    (indices are per cloud, the fused MLP is per row: chunking must not change anything)."""
    from toothgroupnetwork_b200.pipeline import HostPipeline
    B, N = 10, 6000
    feats = torch.cat([clouds.arch_features(N, 40 + i) for i in range(B)], 0)
    sa = pn2.PointNetSetAbstraction(256, 0.1, 32, 9, [32, 32, 64], False).cuda().eval()
    with torch.no_grad():
        d = feats.cuda()
        want_xyz, want_pts = sa(d[:, :3].contiguous(), d)
    host = feats.pin_memory()
    ox = torch.empty((B, 3, 256)).pin_memory()
    op = torch.empty((B, 64, 256)).pin_memory()
    for groups in ((1,), (2, 1)):
        ox.zero_(); op.zero_()
        HostPipeline(sa, chunk_clouds=3, n_streams=2, groups=groups)(host, ox, op)
        torch.cuda.synchronize()
        assert torch.equal(ox, want_xyz.cpu()) and torch.equal(op, want_pts.cpu())
