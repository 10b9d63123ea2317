"""GPU: the no-grad forward of DGCNN on the tensor-core layer chain (toothgroupnetwork_b200.dgcnn.forward, csrc/pw_mlp.cu modes 0
and 2 with LeakyReLU) against the reference's own DGCnnModule (models/modules/dgcnn.py, through oracle.ref_models):

* (A) with every layer fed the neighbour indices of the reference's own fp32 run: x1|x2|x3, the conv8 activation and cls_pred
  against the float64 evaluation of the reference module, within 1e-4 element-wise or twice the reference fp32 run's distance;
* (B) BatchNorm's side effects (running statistics within the same element-wise bar) and dropout's mask;
* (C) end to end with the kernel's own neighbours: argmax(cls_pred) against the reference's;
* (D) under autograd the wrapped forward is the reference's, bitwise;
* (E) the memory one forward needs;
* mode 2 alone against a torch gather + conv on odd strides, the ReLU chains' bits with the new descriptor fields set, and the
  fallback for what ``fusable`` refuses."""
import copy
import ctypes
import importlib.util
import os

import pytest
import torch
from torch import nn

from oracle import ref_models
from toothgroupnetwork_b200 import _lib as L
from toothgroupnetwork_b200 import clouds, dgcnn, dropin
from toothgroupnetwork_b200 import pointnet2_utils as pn2

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not ref_models.available(), reason="reference snapshot not staged")]
REL_TOL, FLOOR = 1e-4, 0.05
BNS = ("bn1", "bn2", "bn3", "bn4", "bn5", "bn6", "bn7", "bn8")


def elementwise(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float(((a - b).abs() / b.abs().clamp(min=FLOOR * float(b.abs().max()))).max())


def _load(name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ref_models.reference_root(), "models", "modules", "dgcnn.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.fixture(scope="module")
def mods():
    """(unwrapped reference module, reference module with accelerate_forward)"""
    ref, fused = _load("ref_dgcnn_fwd_a"), _load("ref_dgcnn_fwd_b")
    dropin.accelerate_dgcnn_forward(fused)
    dropin.accelerate_dgcnn_forward(fused)                                  # idempotent
    return ref, fused


@pytest.fixture(autouse=True)
def fp32_settings():
    saved = torch.backends.cudnn.allow_tf32, torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = saved


def inputs(B, N, permuted):
    """(B, 6, N) [xyz; normal] of seeded arches, contiguous or the permute(0, 2, 1) view the sem pipeline passes"""
    f = torch.cat([clouds.arch_features(N, b) for b in range(B)]).cuda()
    return f.transpose(1, 2).contiguous().permute(0, 2, 1) if permuted else f.contiguous()


def build(mod, train, x, seed=0, affines=True):
    """seeded DGCnnModule, with seeded BatchNorm affines when ``affines`` (negative scales included, so the min-for-max path runs);
    in eval mode the running statistics are the batch statistics of one reference pass over x"""
    torch.manual_seed(seed)
    m = mod.DGCnnModule(None).cuda()
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for name in BNS if affines else ():
            bn = getattr(m, name)
            bn.weight.copy_(torch.rand(bn.num_features, generator=g) * 3.0 - 1.0)
            bn.bias.copy_(torch.rand(bn.num_features, generator=g) * 0.4 - 0.2)
    if not train:
        for name in BNS:
            getattr(m, name).momentum = 1.0
        m.train()
        with torch.no_grad():
            m([x])
        for name in BNS:
            getattr(m, name).momentum = 0.1
            getattr(m, name).num_batches_tracked.zero_()
        m.eval()
    return m.train() if train else m


class Taps:
    """x1|x2|x3 (conv6's input), the conv8 activation (dp1's input) and dp1's output of a reference module's forward"""

    def __init__(self, m):
        self.d = {}
        self.h = [m.conv6.register_forward_pre_hook(lambda _m, inp: self.d.__setitem__("x123", inp[0].detach().clone())),
                  m.dp1.register_forward_hook(lambda _m, inp, out: self.d.update(conv8=inp[0].detach().clone(), dp=out.detach().clone()))]

    def close(self):
        for h in self.h:
            h.remove()


def reference_run(mod, m, x, pinned=None):
    """forward of the reference module m; pinned: the indices its knn returns, in call order; returns (cls_pred, taps, indices)"""
    seen = []
    original = mod.knn

    def knn(v, k):
        idx = pinned[len(seen)] if pinned is not None else original(v, k)
        seen.append(idx)
        return idx

    taps = Taps(m)
    mod.knn = knn
    try:
        with torch.no_grad():
            torch.manual_seed(1)
            pred = m([x])["cls_pred"]
    finally:
        mod.knn = original
        taps.close()
    return pred, taps.d, seen


@pytest.mark.parametrize("permuted", [True, False])
@pytest.mark.parametrize("B,N", [(1, 4096), (2, 4096), (1, 24000), (2, 24000)])
def test_pinned_neighbours_against_float64(mods, B, N, permuted):
    """(A) and (B) with batch-statistics BatchNorm; eval mode is refused by ``fusable`` and runs the reference's forward"""
    train = True
    ref_mod, _ = mods
    x = inputs(B, N, permuted)
    m32 = build(ref_mod, train, x)
    m32.dp1.eval()                            # dropout draws differ between float32 and float64 tensors: compared in (B) instead
    m64, mnew = copy.deepcopy(m32).double(), copy.deepcopy(m32)
    torch.backends.cudnn.allow_tf32 = False
    p32, t32, idx = reference_run(ref_mod, m32, x)
    p64, t64, _ = reference_run(ref_mod, m64, x.double(), pinned=idx)
    with torch.no_grad():
        assert dgcnn.fusable(mnew, [x])
    taps, it = {}, iter(idx)
    before = L.launch_count()
    with torch.no_grad():
        torch.manual_seed(1)
        got = dgcnn.forward(mnew, [x], knn=lambda v, k: next(it), keep=taps)["cls_pred"]
    torch.cuda.synchronize()
    assert L.launch_count() - before == 8 + 22                            # 8 weight packs on first use, 22 chain launches
    for name, ours, fp32, truth in (("x123", taps["x123"], t32["x123"], t64["x123"]), ("conv8", taps["conv8"], t32["conv8"], t64["conv8"]),
                                    ("cls_pred", got, p32, p64)):
        e_ours, e_fp32 = elementwise(ours, truth), elementwise(fp32, truth)
        assert e_ours <= max(REL_TOL, 2.0 * e_fp32), (name, e_ours, e_fp32)
    # (B) BatchNorm side effects
    for name in BNS:
        new, ref64, ref32 = getattr(mnew, name), getattr(m64, name), getattr(m32, name)
        assert int(new.num_batches_tracked) == int(ref32.num_batches_tracked) == (1 if train else 0), name
        for stat in ("running_mean", "running_var"):
            e_ours, e_fp32 = elementwise(getattr(new, stat), getattr(ref64, stat)), elementwise(getattr(ref32, stat), getattr(ref64, stat))
            # the element-wise output bar: bn8's running mean, a mean of conv8 outputs whose tensor-core accumulation truncates
            # (DESIGN §3.12), measured up to 6.3e-5 from float64 where the reference's fp32 run is at 1.9e-5
            assert e_ours <= max(REL_TOL, 2.0 * e_fp32), (name, stat, e_ours, e_fp32)


def _neighbour_rows_differing(a, b):
    return int((a.sort(-1)[0] != b.sort(-1)[0]).any(-1).sum())


@pytest.mark.parametrize("B,N", [(1, 24000), (2, 4096)])
def test_end_to_end_argmax_agrees(mods, B, N):
    """(C) with each side's own neighbours, batch-statistics BatchNorm and the module's own seeded initialisation, against the
    reference's fp32 convolutions (cuDNN's default TF32 moves x1 by ~1e-3 and with it ~5 % of the layer-2 / -3 neighbour sets:
    scripts/dgcnn_bench.py records that agreement); dp1 is active and must zero the same elements (B)"""
    ref_mod, fused_mod = mods
    train = True
    torch.backends.cudnn.allow_tf32 = False
    x = inputs(B, N, True)
    mref = build(ref_mod, train, x, affines=False)
    mnew = fused_mod.DGCnnModule(None).cuda().train(train)
    mnew.load_state_dict(mref.state_dict())
    pref, tref, idx_ref = reference_run(ref_mod, mref, x)
    seen = []

    def knn(v, k):
        seen.append(dgcnn.knn_features(v, k))
        return seen[-1]

    taps = Taps(mnew)
    with torch.no_grad():
        torch.manual_seed(1)
        got = dgcnn.forward(mnew, [x], knn=knn)["cls_pred"]
    taps.close()
    agree = float((got.argmax(1) == pref.argmax(1)).float().mean())
    differ = [_neighbour_rows_differing(a, b) for a, b in zip(seen, idx_ref)]
    assert differ[0] == 0
    assert agree >= 0.999, (agree, "rows with different neighbour sets per layer", differ)
    if train:
        dropped_ref = (tref["dp"] == 0) & (tref["conv8"] != 0)
        dropped_new = (taps.d["dp"] == 0) & (taps.d["conv8"] != 0)
        assert torch.equal(dropped_ref, dropped_new)
        assert 0.4 < float(dropped_new.float().mean()) < 0.6


def test_autograd_runs_the_reference_forward_bitwise(mods):
    """(D): with gradients the wrapped class runs the reference's forward; with accelerate() too only the three kNN calls move"""
    ref_mod, fused_mod = mods
    knn_mod = _load("ref_dgcnn_fwd_c")
    dropin.accelerate_dgcnn_forward(knn_mod)
    dropin.accelerate_dgcnn(knn_mod)
    x = inputs(2, 4096, True)
    labels = torch.randint(0, 17, (2, 4096), generator=torch.Generator().manual_seed(9)).cuda()
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False
    torch.use_deterministic_algorithms(True, warn_only=True)
    results = []
    try:
        for mod in (ref_mod, fused_mod, knn_mod):
            m = build(mod, True, x)
            assert not dgcnn.fusable(m, [x])
            before = L.launch_count()
            torch.manual_seed(1)
            pred = m([x])["cls_pred"]
            torch.nn.functional.cross_entropy(pred, labels).backward()
            torch.cuda.synchronize()
            results.append((pred.detach(), [p.grad.clone() for p in m.parameters() if p.grad is not None], L.launch_count() - before,
                            {k: v.clone() for k, v in m.state_dict().items()}))
    finally:
        torch.use_deterministic_algorithms(False)
    (p0, g0, n0, s0) = results[0]
    assert n0 == 0 and results[1][2] == 0 and results[2][2] == 3
    for p1, g1, _, s1 in results[1:]:
        assert torch.equal(p0.view(torch.int32), p1.view(torch.int32))
        assert len(g0) == len(g1) and all(torch.equal(a.view(torch.int32), b.view(torch.int32)) for a, b in zip(g0, g1))
        assert all(torch.equal(s0[k], s1[k]) for k in s0)


def test_memory_of_one_forward(mods):
    """(E): the largest buffer is one EdgeConv pre-activation, 64 x 480 000 x 4 B"""
    _, fused_mod = mods
    x = inputs(1, 24000, True)
    m = build(fused_mod, True, x)
    with torch.no_grad():
        m([x])                                                             # weights packed, allocator warm
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        before = L.launch_count()
        out = m([x])["cls_pred"]
        torch.cuda.synchronize()
    grew = torch.cuda.max_memory_allocated() - base
    # 3 kNN + EdgeConv 1, 2 (2 fills, 2 layers, 1 apply) + EdgeConv 3 and conv6 (2 fills, 1 layer, 1 apply)
    # + conv7/8 (per-cloud bias, 2 layers, 1 apply)
    assert L.launch_count() - before == 3 + 5 + 5 + 4 + 4 + 4
    assert grew < 256 << 20, grew
    assert out.shape == (1, 17, 24000)


def _gather_conv_reference(x, idx, w):
    """get_graph_feature's edge tensor (models/modules/dgcnn.py:34-39) in float32, then the 1x1 conv in float64: (cout, B*N*K)"""
    B, C, N = x.shape
    xt = x.transpose(2, 1)                                                 # (B, N, C)
    safe = idx.clamp(0, N - 1).long()
    feat = torch.stack([xt[b][safe[b]] for b in range(B)])               # (B, N, K, C)
    cen = xt.unsqueeze(2).expand_as(feat)
    edge = torch.cat((feat - cen, cen), dim=3)
    edge[(idx < 0) | (idx >= N)] = 0.0
    return torch.einsum("oc,bnkc->obnk", w.double(), edge.double()).reshape(w.shape[0], -1)


@pytest.mark.parametrize("B,C,N,K,cout,view", [(2, 17, 1000, 7, 70, "strided"), (1, 6, 2048, 20, 64, "permuted"),
                                               (2, 64, 700, 20, 130, "channel_slice"), (1, 33, 300, 32, 64, "strided")])
def test_edge_mode_against_torch_gather_and_conv(B, C, N, K, cout, view):
    g = torch.Generator().manual_seed(B * 1000 + C)
    if view == "strided":                                                  # every other channel, every third point, offset
        x = (torch.randn(B, 2 * C + 1, 3 * N, generator=g).cuda())[:, 1::2, ::3]
    elif view == "permuted":
        x = torch.randn(B, N, C, generator=g).cuda().permute(0, 2, 1)
    else:                                                                  # channels 64-127 of a (B, 192, N) buffer
        x = torch.randn(B, 192, N, generator=g).cuda()[:, 64:128]
    idx = torch.randint(0, N, (B, N, K), generator=g, dtype=torch.int32)
    idx[0, 3, 1], idx[-1, N - 1, K - 1] = N, -1                           # out of range: zero rows
    idx = idx.cuda()
    w = (torch.randn(cout, 2 * C, generator=g) / (2 * C) ** 0.5).cuda()
    rows = B * N * K
    packed = torch.empty(L.load().tgn_pw_packed_bytes(cout, 2 * C), dtype=torch.uint8, device="cuda")
    L.call("tgn_pw_pack_weights", cout, 2 * C, L.ptr(w), L.ptr(packed), L.stream_ptr())
    y = torch.empty((cout, rows), dtype=torch.float32, device="cuda")
    d = L.PwLayer()
    d.rows, d.rows_per_batch, d.cin, d.cout, d.mode = rows, N * K, 2 * C, cout, 2
    d.edge_x, d.edge_C, d.gidx, d.N, d.K = L.ptr(x), C, L.ptr(idx), N, K
    d.edge_stride[0], d.edge_stride[1], d.edge_stride[2] = x.stride()
    d.w_packed, d.y = L.ptr(packed), L.ptr(y)
    L.call("tgn_pw_layer_forward", ctypes.byref(d), L.stream_ptr())
    want = _gather_conv_reference(x, idx, w)
    assert elementwise(y, want) < 5e-5
    assert float(y[:, (3 * K + 1)].abs().max()) == 0.0 and float(y[:, -1].abs().max()) == 0.0
    d.cin = 2 * C + 1
    with pytest.raises(L.TgnError, match="edge-feature"):
        L.call("tgn_pw_layer_forward", ctypes.byref(d), L.stream_ptr())


def _set_ignored_fields(monkeypatch, junk):
    """every pw_mlp launch gets nonzero values in the new fields its mode and activation kind ignore"""
    real = L.call

    def call(name, *args):
        if name == "tgn_pw_layer_forward":
            d = args[0]._obj
            assert d.in_act == 0 and d.mode in (0, 1)
            d.edge_x, d.edge_C, d.in_act_slope = L.ptr(junk), 5, 0.37
            d.edge_stride[0], d.edge_stride[1], d.edge_stride[2] = 3, 2, 1
        elif name == "tgn_pw_apply":
            a = args[0]._obj
            assert a.act == 0
            a.act_slope = 0.37
        return real(name, *args)

    monkeypatch.setattr(L, "call", call)


@pytest.mark.parametrize("train", [True, False])
def test_relu_chains_ignore_the_new_fields(monkeypatch, train):
    """a set abstraction (mode 1, last layer reduced) and a mode-0 chain: bitwise equal with the new fields zero and set"""
    torch.manual_seed(3)
    B, N, S, K, D = 2, 3000, 512, 20, 13
    xyz = torch.rand(B, N, 3).cuda()
    feats = torch.randn(B, N, D).cuda()
    new_xyz = xyz[:, :S].contiguous()
    gidx = torch.randint(0, N, (B, S, K), dtype=torch.int32).cuda()
    convs = [nn.Conv2d(D + 3, 64, 1).cuda(), nn.Conv2d(64, 96, 1).cuda()]
    bns = [nn.BatchNorm2d(64).cuda(), nn.BatchNorm2d(96).cuda()]
    seg = torch.randn(B, 40, N).cuda()
    convs0, bns0 = [nn.Conv1d(40, 128, 1).cuda(), nn.Conv1d(128, 32, 1).cuda()], [nn.BatchNorm1d(128).cuda(), nn.BatchNorm1d(32).cuda()]
    for b in bns + bns0:
        b.running_mean.uniform_(-0.1, 0.1)
        b.running_var.uniform_(0.5, 2.0)
        b.train(train)

    def run():
        cb, cb0 = copy.deepcopy(bns), copy.deepcopy(bns0)
        out = torch.empty((B, 96, S), device="cuda")
        pn2._pw_set_abstraction(pn2._PwChain(), convs, cb, xyz, feats, new_xyz, gidx, True, out, 0)
        out0 = torch.empty((B, 32, N), device="cuda")
        d = L.PwLayer()
        d.mode, d.rows_per_batch = 0, N
        d.seg_ptr[0], d.seg_channels[0] = L.ptr(seg), 40
        d.seg_batch_stride[0], d.seg_row_stride[0], d.seg_chan_stride[0] = 40 * N, 1, N
        pn2._PwChain().run(convs0, cb0, d, B * N, out0, 0, N)
        torch.cuda.synchronize()
        return [out, out0] + [t for b in cb + cb0 for t in (b.running_mean, b.running_var)]

    with torch.no_grad():
        plain = run()
        _set_ignored_fields(monkeypatch, seg)
        junk = run()
    assert all(torch.equal(a.view(torch.int32), b.view(torch.int32)) for a, b in zip(plain, junk))


def _modify(m, what):
    if what == "relu":
        m.conv2[2] = nn.ReLU()
    elif what == "bias":
        conv = m.conv4[0]
        m.conv4[0] = nn.Conv2d(conv.in_channels, conv.out_channels, 1, bias=True).cuda()
    elif what == "momentum_none":
        m.bn5.momentum = None
    elif what == "no_affine":
        m.conv7[1] = nn.BatchNorm1d(m.conv7[1].num_features, affine=False).cuda()
    elif what == "kernel_size":
        m.conv8[0] = nn.Conv1d(m.conv8[0].in_channels, m.conv8[0].out_channels, 3, padding=1, bias=False).cuda()
    elif what == "k33":
        m.k = 33
    elif what == "double":
        m.double()
    elif what == "eval":
        m.eval()
    return m


@pytest.mark.parametrize("what", ["relu", "bias", "momentum_none", "no_affine", "kernel_size", "k33", "double", "grad", "eval"])
def test_refused_calls_run_the_reference_forward(mods, what):
    ref_mod, fused_mod = mods
    x = inputs(1, 4096, True)
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False
    outs = []
    for mod in (ref_mod, fused_mod):
        m = build(mod, True, x)
        with torch.no_grad():
            assert dgcnn.fusable(m, [x])                                  # refused for the change alone
        m = _modify(m, what)
        xin = x.double() if what == "double" else x
        before = L.launch_count()
        with torch.set_grad_enabled(what == "grad"):
            assert not dgcnn.fusable(m, [xin])
            torch.manual_seed(1)
            outs.append(m([xin])["cls_pred"].detach())
        torch.cuda.synchronize()
        assert L.launch_count() == before
    assert torch.equal(outs[0], outs[1])
