"""The fused point-transformer decoder and heads (csrc/pt_head.cu, blocks_fused.transition_up_forward / multi_head_forward) one
launch at a time against float64 (oracle/pt_decoder.py) and torch, and at module level at the networks' shapes."""
import ctypes
import types

import pytest
import torch

from oracle import pt_decoder as D
from test_cpu_pt_decoder import _MH, _TU
from toothgroupnetwork_b200 import _lib as L
from toothgroupnetwork_b200 import blocks_fused, clouds, pointops

pytestmark = pytest.mark.gpu
F64 = torch.float64
U = 2.0 ** -24


def _rand_bn(module, gen):
    for m in module.modules():
        if isinstance(m, torch.nn.BatchNorm1d):
            with torch.no_grad():
                m.weight.copy_(torch.rand(m.weight.shape, generator=gen) + 0.5)
                m.bias.copy_(torch.randn(m.bias.shape, generator=gen) * 0.1)
                m.running_mean.copy_(torch.randn(m.running_mean.shape, generator=gen) * 0.1)
                m.running_var.copy_(torch.rand(m.running_var.shape, generator=gen) + 0.5)


@pytest.mark.parametrize("levels", [1, 2, 5, 8])
@pytest.mark.parametrize("k", [2, 3, 10, 17, 32])
def test_head_classify_against_float64(levels, k):
    gen = torch.Generator().manual_seed(levels * 100 + k)
    n0 = 1000                                                   # not a multiple of the 128-row block
    ns = [n0] + [max(1, n0 >> (2 * s)) for s in range(1, levels)]
    lats = [torch.rand(32, n, generator=gen).cuda() for n in ns]
    nns = [None]
    for n in ns[1:]:
        nn_s = torch.randint(0, n, (n0,), generator=gen, dtype=torch.int32)
        nn_s[:3], nn_s[-3:] = 0, n - 1                           # both ends of the level
        nns.append(nn_s.cuda())
    w = torch.randn(k, 32 * levels, generator=gen).cuda()
    b = torch.randn(k, generator=gen).cuda()
    out = torch.empty(n0, k, device="cuda")
    d = L.HeadClassify()
    d.n0, d.k, d.levels = n0, k, levels
    for s in range(levels):
        d.lat[s], d.nn[s], d.n[s] = L.ptr(lats[s]), L.ptr(nns[s]), ns[s]
    d.w, d.b, d.out = L.ptr(w), L.ptr(b), L.ptr(out)
    L.call("tgn_head_classify", ctypes.byref(d), L.stream_ptr())
    rows = [l.t().double() if nn is None else l.t().double()[nn.long()] for l, nn in zip(lats, nns)]
    x = torch.cat(rows, 1)
    want = x @ w.double().t() + b.double()
    bound = (32 * levels + 1) * U * (x.abs() @ w.double().abs().t() + b.double().abs())
    assert bool(((out.double() - want).abs() <= bound).all())


def _interp_inputs(gen, n1, n2, c):
    y1 = torch.randn(c, n1, generator=gen).cuda()
    f = torch.randn(n2, c, generator=gen).cuda()
    idx = torch.randint(0, n2, (n1, 3), generator=gen, dtype=torch.int32)
    idx[0], idx[-1] = 0, n2 - 1
    w = torch.rand(n1, 3, generator=gen)
    return y1, f, idx.cuda(), (w / w.sum(1, keepdim=True)).cuda()


def _apply_desc(y1, out, bn, stats=None):
    a = L.PwApply()
    c, n = y1.shape
    a.rows, a.rows_per_batch, a.channels, a.out_channels, a.relu = n, n, c, c, 1
    a.src, a.out = L.ptr(y1), L.ptr(out)
    a.affine = 2 if stats is None else 1
    a.stats, a.stat_rows = L.ptr(stats), n
    a.gamma, a.beta, a.running_mean, a.running_var = L.ptr(bn.weight), L.ptr(bn.bias), L.ptr(bn.running_mean), L.ptr(bn.running_var)
    a.eps, a.momentum = bn.eps, 0.1
    return a


@pytest.mark.parametrize("n1,n2,c", [(1000, 250, 32), (777, 100, 64), (40, 7, 16)])
def test_interpolated_apply_is_torchs_interpolation_plus_add(n1, n2, c):
    gen = torch.Generator().manual_seed(n1 + c)
    y1, f, idx, w = _interp_inputs(gen, n1, n2, c)
    bn = torch.nn.BatchNorm1d(c).cuda().eval()
    _rand_bn(bn, gen)
    bn.cuda()
    u = L.PtUpApply()
    out = torch.empty(n1, c, device="cuda")
    u.apply = _apply_desc(y1, out, bn)
    u.f, u.idx, u.w, u.f_rows = L.ptr(f), L.ptr(idx), L.ptr(w), n2
    L.call("tgn_pt_up_apply", ctypes.byref(u), L.stream_ptr())
    base = torch.empty(1, c, n1, device="cuda")                 # the parent's apply on the same y1
    L.call("tgn_pw_apply", ctypes.byref(_apply_desc(y1, base, bn)), L.stream_ptr())
    want = base[0].t() + pointops._WeightedGather.apply(f, idx, w, False)
    assert torch.equal(out, want)
    u.f = None                                                  # no addend: the parent's apply, row-major
    L.call("tgn_pt_up_apply", ctypes.byref(u), L.stream_ptr())
    assert torch.equal(out, base[0].t())
    with torch.no_grad():                                        # and pointops.interpolation itself with these neighbours
        new = torch.zeros(n1, c, device="cuda")
        for j in range(3):
            new += f[idx[:, j].long(), :] * w[:, j].unsqueeze(-1)
    assert torch.equal(want, base[0].t() + new)


def _levels(B, n, strides):
    """B dental arches of n points, and each coarser level every stride-th point of each cloud -> [(p, o)]"""
    p = torch.cat([clouds.dental_arch(n, 30 + b)[0] for b in range(B)]).cuda().contiguous()
    out, per = [], n
    for s in strides:
        per //= s
        p = p.view(B, -1, 3)[:, ::s][:, :per].reshape(-1, 3).contiguous()
        out.append((p, torch.arange(1, B + 1, dtype=torch.int32, device="cuda") * per))
    return out


def _close(got, want, floor=0.05):
    got, want = got.double(), want.double()
    return float(((got - want).abs() / want.abs().clamp(min=floor * float(want.abs().max()))).max())


def _check_after(module, after):
    sd = module.state_dict()
    for k, v in after.items():
        if "num_batches" in k:
            assert int(sd[k]) == int(v), k
        else:
            assert _close(sd[k], v) < 1e-4, k


# (planes top-down, level sizes top-down, B): the first tgnet network at 24 000 points, the boundary network (16 / 32 planes,
# stride 1), and the 16 x 3 072 crop batch
NETS = {
    "tgnet_fps": ([32, 64, 128, 256, 512], 24000, [1, 4, 4, 4, 4], 1),
    "boundary": ([16, 32], 24000, [1, 1], 1),
    "crops16": ([32, 64, 128, 256, 512], 3072, [1, 4, 4, 4, 4], 16),
    "two_clouds": ([32, 64], 2000, [1, 4], 2),
}


@pytest.mark.parametrize("net", list(NETS))
@pytest.mark.parametrize("train", [True, False])
def test_decoder_and_heads_at_network_shapes(net, train):
    planes, n, strides, B = NETS[net]
    gen = torch.Generator().manual_seed(len(planes) * 7 + B)
    lv = _levels(B, n, strides)
    feats = [torch.randn(p.shape[0], c, generator=gen).cuda() for (p, _), c in zip(lv, planes)]
    if net == "two_clouds":
        feats = [f + torch.arange(f.shape[0], device="cuda").unsqueeze(1).ge(f.shape[0] // 2) * 3.0 for f in feats]
    ups = []
    with torch.no_grad():
        # head form at the coarsest level
        torch.manual_seed(1)
        tu = _TU(planes[-1]).cuda().train(train)
        _rand_bn(tu, gen)
        tu.cuda()
        x = feats[-1]
        state = {k: v.clone() for k, v in tu.state_dict().items()}
        assert blocks_fused.transition_up_fusable(tu, [lv[-1][0], x, lv[-1][1]])
        got = blocks_fused.transition_up_forward(tu, [lv[-1][0], x, lv[-1][1]])
        ends = lv[-1][1].tolist()
        want, _, after = D.transition_up({k: v.double() for k, v in state.items()}, x.double(), ends, train)
        assert _close(got, want) < 1e-4
        if train:
            _check_after(tu, after)
        ups.append(got)
        for lvl in range(len(planes) - 2, -1, -1):
            tu = _TU(planes[lvl + 1], planes[lvl]).cuda().train(train)
            _rand_bn(tu, gen)
            tu.cuda()
            (p1, o1), (p2, o2) = lv[lvl], lv[lvl + 1]
            x1, x2 = feats[lvl], ups[-1]
            state = {k: v.clone() for k, v in tu.state_dict().items()}
            got = blocks_fused.transition_up_forward(tu, [p1, x1, o1], [p2, x2, o2])
            idx, d2 = pointops.knn_packed(3, p2, p1, o2, o1)
            w = pointops._inverse_distance_weights(torch.sqrt(d2))
            want, _, after = D.transition_up({k: v.double() for k, v in state.items()}, x1.double(), o1.tolist(), train,
                                             x2=x2.double(), idx=idx, w=w)
            assert _close(got, want) < 1e-4, lvl
            if train:
                _check_after(tu, after)
            ups.append(got)
        ups = ups[::-1]
        for k in (17, 3):
            mh = _MH(planes, k).cuda().train(train)
            _rand_bn(mh, gen)
            mh.cuda()
            stages = {"up": [{"p_out": p, "f_out": f, "offset": o} for (p, o), f in zip(lv, ups)]}
            state = {kk: v.clone() for kk, v in mh.state_dict().items()}
            assert blocks_fused.multi_head_fusable(mh, stages)
            got, stages = blocks_fused.multi_head_forward(mh, stages)
            nns = [None] + [pointops.knn_packed(1, p, lv[0][0], o, lv[0][1])[0] for p, o in lv[1:]]
            want, _, lats, after = D.multi_head({kk: v.double() for kk, v in state.items()}, [u.double() for u in ups], nns, train)
            assert _close(got, want) < 1e-4
            for s, lat in enumerate(lats):
                assert _close(stages["up"][s]["latent"], lat) < 1e-4
            if train:
                _check_after(mh, after)


def test_autograd_and_unequal_clouds_run_the_reference_code():
    calls = []

    class TransitionUp(_TU):
        def forward(self, pxo1, pxo2=None):
            calls.append("original")
            return pxo1[1]

    class MultiHead(_MH):
        def forward(self, stage_list):
            calls.append("original")
            return None, stage_list

    blocks_fused.accelerate_decoder(types.SimpleNamespace(TransitionUp=TransitionUp), types.SimpleNamespace(MultiHead=MultiHead))
    p, o = _levels(2, 512, [1])[0]
    x = torch.randn(p.shape[0], 32, device="cuda")
    tu = TransitionUp(32).cuda()
    tu([p, x, o])                                              # autograd: parameters need gradients
    with torch.no_grad():
        tu([p, x, torch.tensor([300, 1024], dtype=torch.int32, device="cuda")])   # unequal packed clouds
        assert calls == ["original", "original"]
        out = tu([p, x, o])
        assert calls == ["original", "original"] and out.shape == (1024, 32)
        mh = MultiHead([32], 3).cuda()
        mh({"up": [{"p_out": p, "f_out": x, "offset": o}]})
        assert calls == ["original", "original"]
    mh({"up": [{"p_out": p, "f_out": x, "offset": o}]})
    assert calls == ["original", "original", "original"]
