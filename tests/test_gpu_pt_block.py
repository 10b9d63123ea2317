"""GPU: the fused PointTransformerBlock one launch at a time -- the transformer layer's output pass with bn2's batch sums
(tgn_pt_layer_forward_sums) and bn3 + residual + ReLU (tgn_pt_res_apply) -- against float64 (oracle/pt_block.py), and the whole
block at the shapes of tgnet's two networks against the float64 block, with its running statistics."""
import ctypes
import types

import pytest
import torch
import torch.nn as nn

from oracle import pt_block as B
from test_cpu_pt_block import Block, _randomise
from toothgroupnetwork_b200 import _lib as L
from toothgroupnetwork_b200 import blocks_fused, clouds, pointops

pytestmark = pytest.mark.gpu
F64 = torch.float64


def _close(got, want, floor=0.05):
    got, want = got.double(), want.double()
    return float(((got - want).abs() / want.abs().clamp(min=floor * float(want.abs().max()))).max())


@pytest.fixture(params=[0, 1 << 30], ids=["warp_per_query", "cta_per_query"])
def schedule(request):
    old = L.load().tgn_pt_layer_set_cta_threshold(request.param)
    yield request.param
    L.load().tgn_pt_layer_set_cta_threshold(old)


def _layer_and_input(c, K, n, seed):
    gen = torch.Generator().manual_seed(seed)
    blk = Block(c, K)
    _randomise(blk, gen)
    layer = blk.transformer2.cuda().eval()
    with torch.no_grad():                                      # channels 0 and 1 of out at |mean| / std of about 100 and 1000
        layer.linear_v.bias[0] = 100.0 * float(layer.linear_v.weight[0].norm())
        layer.linear_v.bias[1] = -1000.0 * float(layer.linear_v.weight[1].norm())
    p = torch.cat([clouds.dental_arch(max(n, 4), seed)[0][:n]]).cuda().contiguous()
    x = torch.randn(n, c, generator=gen).cuda()
    return layer, [p, x, torch.tensor([n], dtype=torch.int32, device="cuda")]


@pytest.mark.parametrize("c", [16, 32, 64, 128, 256, 512])
@pytest.mark.parametrize("K", [1, 24, 64])
def test_output_sums_against_float64_sums_of_the_kernels_own_output(c, K, schedule):
    for n in (1, 2, 3, 31, 33, 1001, 2000):
        layer, pxo = _layer_and_input(c, K, n, c + K + n)
        with torch.no_grad():
            plain = blocks_fused.pt_layer_forward(layer, pxo)
            stats = torch.zeros(2 * c, dtype=F64, device="cuda")
            out = blocks_fused.pt_layer_forward(layer, pxo, stats)
        assert torch.equal(out, plain), (n, "the sums change the output")
        o = out.double()
        mean_w, var_w = o.mean(0), o.var(0, unbiased=False)
        mean_g = stats[:c] / n
        var_g = stats[c:] / n - mean_g * mean_g
        std = var_w.sqrt()
        assert bool(((mean_g - mean_w).abs() <= 1e-6 * std + 1e-12 * mean_w.abs()).all()), (n, float((mean_g - mean_w).abs().max()))
        assert bool(((var_g - var_w).abs() <= 1e-5 * var_w + 8 * 2.0 ** -52 * mean_w ** 2).all()), n


def _res_case(c, n, train, seed):
    gen = torch.Generator().manual_seed(seed)
    bn = nn.BatchNorm1d(c, eps=1e-4, momentum=0.3)
    _randomise(bn, gen)
    with torch.no_grad():
        bn.weight[0] = -abs(float(bn.weight[0])) - 0.5                         # negative gamma
    bn = bn.cuda().train(train)
    y = (torch.randn(c, n, generator=gen) * 3 + torch.randn(c, 1, generator=gen) * 20).cuda()
    y[1] = 2.5                                                                   # a zero-variance channel
    ident = torch.randn(n, c, generator=gen).cuda()
    return bn, y, ident


@pytest.mark.parametrize("c,n", [(16, 2000), (32, 24000), (64, 33), (512, 93), (48, 7)])
@pytest.mark.parametrize("train", [True, False])
def test_residual_apply_against_float64(c, n, train):
    bn, y, ident = _res_case(c, n, train, c + n)
    state = {k: v.clone() for k, v in bn.state_dict().items()}
    yd = y.double()
    stats = torch.cat([yd.sum(1), (yd * yd).sum(1)]).contiguous()
    ident0 = ident.clone()
    guard = 7
    buf = torch.full(((n + 2 * guard) * c,), 1234.5, device="cuda")
    out = buf[guard * c:(guard + n) * c].view(n, c)
    a = L.PwApply()
    a.rows, a.rows_per_batch, a.channels, a.out_channels, a.relu = n, n, c, c, 1
    a.src, a.out = L.ptr(y), L.ptr(out)
    a.affine, a.stats, a.stat_rows = (1 if train else 2), L.ptr(stats), n
    a.gamma, a.beta, a.running_mean, a.running_var = L.ptr(bn.weight), L.ptr(bn.bias), L.ptr(bn.running_mean), L.ptr(bn.running_var)
    a.eps, a.momentum, a.update_running = bn.eps, bn.momentum, int(train)
    r = L.PtResApply()
    r.apply, r.identity, r.identity_row_stride = a, L.ptr(ident), c
    L.call("tgn_pt_res_apply", ctypes.byref(r), L.stream_ptr())
    want, err, _ = B.res_apply(yd, {k: v.double() for k, v in state.items()}, "", ident.double(), train, eps=bn.eps,
                               momentum=bn.momentum)
    assert bool(((out.double() - want).abs() <= err).all()), float(((out.double() - want).abs() / err).max())
    assert torch.equal(ident, ident0)
    assert bool((buf[:guard * c] == 1234.5).all()) and bool((buf[(guard + n) * c:] == 1234.5).all())
    if train:
        mean, var = yd.mean(1), yd.var(1, unbiased=False)
        m = bn.momentum
        for got, old, batch in ((bn.running_mean, state["running_mean"].cuda(), mean.float()),
                                (bn.running_var, state["running_var"].cuda(), (var * n / (n - 1)).float())):
            ref = (1 - m) * old + m * batch
            # ulps of the update's two terms: where they cancel, the result's own ulp is smaller than one rounding of a term
            ulp = torch.finfo(torch.float32).eps * ((1 - m) * old.abs() + m * batch.abs())
            assert bool(((got - ref).abs() <= 4 * ulp).all()), float(((got - ref).abs() / ulp).max())


def _levels(B_, n, strides):
    p = torch.cat([clouds.dental_arch(n, 30 + b)[0] for b in range(B_)]).cuda().contiguous()
    out, per = [], n
    for s in strides:
        per //= s
        p = p.view(B_, -1, 3)[:, ::s][:, :per].reshape(-1, 3).contiguous()
        out.append((p, torch.arange(1, B_ + 1, dtype=torch.int32, device="cuda") * per))
    return out


# (planes, nsample, strides, n per cloud, clouds): tgnet's first network at 1 x 24 000 and on the 16 x 3 072 crop batch, and the
# boundary network's 16 / 32 planes at stride 1
NETS = {
    "first_1x24000": ([32, 64, 128, 256, 512], [36, 24, 24, 24, 24], [1, 4, 4, 4, 4], 24000, 1),
    "first_16x3072": ([32, 64, 128, 256, 512], [36, 24, 24, 24, 24], [1, 4, 4, 4, 4], 3072, 16),
    "boundary_1x24000": ([16, 32], [36, 24], [1, 1], 24000, 1),
    "boundary_16x3072": ([16, 32], [36, 24], [1, 1], 3072, 16),
}


@pytest.mark.parametrize("net", list(NETS))
@pytest.mark.parametrize("train", [True, False])
def test_block_at_network_shapes_against_float64(net, train):
    planes, nsample, strides, n, nb = NETS[net]
    gen = torch.Generator().manual_seed(len(planes) + nb)
    for lvl, ((p, o), c, K) in enumerate(zip(_levels(nb, n, strides), planes, nsample)):
        blk = Block(c, K)
        _randomise(blk, gen)
        blk = blk.cuda().train(train)
        x = (torch.randn(p.shape[0], c, generator=gen) + torch.randn(1, c, generator=gen)).cuda()
        x0 = x.clone()
        state = {k: v.clone() for k, v in blk.state_dict().items()}
        with torch.no_grad():
            # the forward is exact at every width; the drop-in takes it only up to BLOCK_FUSED_MAX_C, where it is faster
            assert blocks_fused.pt_block_fusable(blk, p, x, o) == (c <= blocks_fused.BLOCK_FUSED_MAX_C)
            got = blocks_fused.pt_block_forward(blk, [p, x, o])[1]
        assert torch.equal(x, x0)
        idx, _ = pointops.knn_packed(K, p, p, o, o)
        want, after = B.block({k: v.double() for k, v in state.items()}, p, x, idx, train)
        assert _close(got, want) < 1e-4, (lvl, _close(got, want))
        sd = blk.state_dict()
        if train:
            assert len(after) == 18
            for k, v in after.items():
                if "num_batches" in k:
                    assert int(sd[k]) == int(v) == 1, k
                else:
                    assert _close(sd[k], v) < 1e-4, (lvl, k)
        else:
            assert all(torch.equal(sd[k], state[k]) for k in sd), lvl


def test_autograd_is_bitwise_the_reference_and_other_calls_fall_back():
    calls = []

    class PointTransformerBlock(Block):
        def forward(self, pxo):
            calls.append("original")
            return super().forward(pxo)

    blocks_fused.accelerate_blocks(types.SimpleNamespace(PointTransformerBlock=PointTransformerBlock))
    p, o = _levels(1, 512, [1])[0]
    torch.manual_seed(5)
    ref = Block(32, 16).cuda()
    ours = PointTransformerBlock(32, 16).cuda()
    ours.load_state_dict(ref.state_dict())
    idx, _ = pointops.knn_packed(16, p, p, o, o)
    ref.transformer2.idx = ours.transformer2.idx = idx.long()
    x = torch.randn(512, 32, device="cuda")
    outs, grads = [], []
    for m in (ref, ours):
        xi = x.clone().requires_grad_(True)
        out = m([p, xi, o])[1]
        out.square().sum().backward()
        outs.append(out.detach())
        grads.append([xi.grad] + [q.grad for q in m.parameters()])
    assert calls == ["original"]
    assert torch.equal(outs[0], outs[1]) and all(torch.equal(a, b) for a, b in zip(grads[0], grads[1]))

    def refused(blk, xx):
        before = len(calls)
        with torch.no_grad():
            blk([p, xx, o])
        return len(calls) == before + 1

    x16 = torch.randn(512, 16, device="cuda")                  # 16 channels: within BLOCK_FUSED_MAX_C, refused only for its reason
    assert not refused(PointTransformerBlock(16, 16).cuda(), x16)                       # taken
    above = PointTransformerBlock(64, 16).cuda()
    above.transformer2.idx = idx.long()
    assert refused(above, torch.randn(512, 64, device="cuda"))                          # wider than BLOCK_FUSED_MAX_C
    wide = PointTransformerBlock(24, 16).cuda()
    wide.transformer2.idx = idx.long()
    assert refused(wide, torch.randn(512, 24, device="cuda"))                           # unsupported width
    biased = PointTransformerBlock(16, 16, bias=True).cuda()
    biased.transformer2.idx = idx.long()
    assert refused(biased, x16)                                                         # linear1 with a bias
    cma = PointTransformerBlock(16, 16).cuda()
    cma.bn2 = nn.BatchNorm1d(16, momentum=None).cuda()
    cma.transformer2.idx = idx.long()
    assert refused(cma, x16)                                                            # cumulative moving average
    cpu = PointTransformerBlock(16, 16)
    cpu.transformer2.idx = idx.long().cpu()
    before = len(calls)
    with torch.no_grad():
        cpu([p.cpu(), x16.cpu(), o.cpu()])
    assert len(calls) == before + 1                                                     # CPU tensors
    needs_grad = PointTransformerBlock(16, 16).cuda()
    needs_grad.transformer2.idx = idx.long()
    needs_grad([p, x16, o])                                                             # parameters need gradients
    assert calls[-1] == "original"
