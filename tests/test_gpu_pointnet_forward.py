"""GPU: the no-grad forward of PointNet on the tensor-core layer chain (toothgroupnetwork_b200.pointnet.forward, csrc/pw_mlp.cu and
csrc/pw_transform.cu) against the reference's own get_model (models/modules/pointnet.py on external_libs/pointnet2_utils/
pointnet_utils.py, through oracle.ref_models):

* (A) trans, trans_feat, g, pointfeat, the head's conv3 activation and the log-probabilities against the float64 evaluation of
  the reference module, within 1e-4 element-wise or twice the reference fp32 run's distance;
* (B) BatchNorm's side effects: the running statistics of all twelve BatchNorms within the same bar, num_batches_tracked equal;
* (C) argmax of the log-probabilities against the reference's fp32 run, through the wrapped class;
* (D) under autograd the wrapped forward is the reference's, bitwise;
* (E) the memory one forward needs, (F) the torch ops it runs;
* (G) tgn_pw_cloud_transform alone against float64, and the fallback for what ``fusable`` refuses."""
import copy
import importlib.util
import os
import sys

import pytest
import torch
import torch.nn.functional as F
from torch import nn

from oracle import ref_models
from toothgroupnetwork_b200 import _lib as L
from toothgroupnetwork_b200 import clouds, dropin, pointnet

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not ref_models.available(), reason="reference snapshot not staged")]
REL_TOL, FLOOR = 1e-4, 0.05
FORWARD_LAUNCHES = 6 + 1 + 2 + 6 + 1 + 5 + 1 + 4     # STN3d, input transform, conv1, STNkd, feature transform, encoder, cloud bias, head
WEIGHT_PACKS = 3 + 1 + 3 + 2 + 3


def elementwise(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float(((a - b).abs() / b.abs().clamp(min=FLOOR * float(b.abs().max()))).max())


def _load(name):
    """models/modules/pointnet.py of the staged reference as a fresh module, its PointNetEncoder from the staged pointnet_utils.py"""
    root = ref_models.reference_root()
    spec = importlib.util.spec_from_file_location(name + "_utils", os.path.join(root, "external_libs", "pointnet2_utils", "pointnet_utils.py"))
    utils = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(utils)
    key = "external_libs.pointnet2_utils.pointnet_utils"
    saved = sys.modules.get(key)
    sys.modules[key] = utils
    try:
        spec = importlib.util.spec_from_file_location(name, os.path.join(root, "models", "modules", "pointnet.py"))
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
    finally:
        if saved is None:
            sys.modules.pop(key, None)
        else:
            sys.modules[key] = saved
    return mod


@pytest.fixture(scope="module")
def mods():
    """(unwrapped reference module, reference module with accelerate_forward)"""
    ref, fused = _load("ref_pointnet_fwd_a"), _load("ref_pointnet_fwd_b")
    dropin.accelerate_pointnet_forward(fused)
    dropin.accelerate_pointnet_forward(fused)                              # idempotent
    return ref, fused


@pytest.fixture(autouse=True)
def fp32_settings():
    saved = torch.backends.cudnn.allow_tf32, torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = saved


def inputs(B, N, permuted):
    """(B, 6, N) [xyz; normal] of different seeded arches, contiguous or the permute(0, 2, 1) view the sem pipeline passes"""
    f = torch.cat([clouds.arch_features(N, b) for b in range(B)]).cuda()
    return f.transpose(1, 2).contiguous().permute(0, 2, 1) if permuted else f.contiguous()


def build(mod, seed=0, affines=True):
    """seeded get_model in train mode, with seeded BatchNorm affines when ``affines``: gamma in [-1, 2), so every layer has negative
    scales and the max over the points takes the min branch in both STN conv3 layers and the encoder's conv3"""
    torch.manual_seed(seed)
    m = mod.get_model().cuda().train()
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for bn in pointnet._bns(m) if affines else ():
            bn.weight.copy_(torch.rand(bn.num_features, generator=g) * 3.0 - 1.0)
            bn.bias.copy_(torch.rand(bn.num_features, generator=g) * 0.4 - 0.2)
    return m


class Taps:
    """trans, trans_feat, g, pointfeat and the head's conv3 activation of a reference module's forward"""

    def __init__(self, m):
        self.d = {}
        c3 = m.feat.conv3.out_channels

        def feat_hook(_m, inp, out):
            self.d.update(g=out[0][:, :c3, 0].detach().clone(), pointfeat=out[0][:, c3:].detach().clone(), trans=out[1].detach().clone())

        self.h = [m.feat.register_forward_hook(feat_hook),
                  m.bn3.register_forward_hook(lambda _m, inp, out: self.d.__setitem__("head3", F.relu(out).detach().clone()))]

    def close(self):
        for h in self.h:
            h.remove()


def reference_run(m, x):
    taps = Taps(m)
    try:
        with torch.no_grad():
            out, trans_feat = m([x])
    finally:
        taps.close()
    return out, trans_feat, taps.d


@pytest.mark.parametrize("permuted", [True, False])
@pytest.mark.parametrize("B,N", [(1, 4096), (2, 4096), (1, 24000), (2, 24000)])
def test_against_float64(mods, B, N, permuted):
    """(A) and (B) with batch-statistics BatchNorm, B = 2 with two different clouds so that a wrong global feature shows"""
    ref_mod, _ = mods
    x = inputs(B, N, permuted)
    m32 = build(ref_mod)
    m64, mnew = copy.deepcopy(m32).double(), copy.deepcopy(m32)
    torch.backends.cudnn.allow_tf32 = False
    o32, tf32, t32 = reference_run(m32, x)
    o64, tf64, t64 = reference_run(m64, x.double())
    with torch.no_grad():
        assert pointnet.fusable(mnew, [x])
    taps = {}
    before = L.launch_count()
    with torch.no_grad():
        got, tf_got = pointnet.forward(mnew, [x], keep=taps)
    torch.cuda.synchronize()
    assert L.launch_count() - before == WEIGHT_PACKS + FORWARD_LAUNCHES
    assert got.shape == o32.shape and tf_got.shape == tf32.shape
    for name, ours, fp32, truth in (("trans", taps["trans"], t32["trans"], t64["trans"]), ("trans_feat", tf_got, tf32, tf64),
                                    ("g", taps["g"], t32["g"], t64["g"]), ("pointfeat", taps["pointfeat"], t32["pointfeat"], t64["pointfeat"]),
                                    ("head3", taps["head3"], t32["head3"], t64["head3"]), ("log_softmax", got, o32, o64)):
        e_ours, e_fp32 = elementwise(ours, truth), elementwise(fp32, truth)
        assert e_ours <= max(REL_TOL, 2.0 * e_fp32), (name, e_ours, e_fp32)
    # (B) BatchNorm side effects
    for new, ref64, ref32 in zip(pointnet._bns(mnew), pointnet._bns(m64), pointnet._bns(m32)):
        assert int(new.num_batches_tracked) == int(ref32.num_batches_tracked) == 1
        for stat in ("running_mean", "running_var"):
            e_ours, e_fp32 = elementwise(getattr(new, stat), getattr(ref64, stat)), elementwise(getattr(ref32, stat), getattr(ref64, stat))
            assert e_ours <= max(REL_TOL, 2.0 * e_fp32), (new, stat, e_ours, e_fp32)


@pytest.mark.parametrize("B,N", [(1, 24000), (2, 24000)])
def test_argmax_agrees_with_the_reference(mods, B, N):
    """(C) through the wrapped class, with the module's own initialisation, against the reference's fp32 convolutions"""
    ref_mod, fused_mod = mods
    torch.backends.cudnn.allow_tf32 = False
    x = inputs(B, N, True)
    mref = build(ref_mod, seed=5, affines=False)
    mnew = fused_mod.get_model().cuda().train()
    mnew.load_state_dict(mref.state_dict())
    with torch.no_grad():
        pref, _ = mref([x])
        before = L.launch_count()
        pnew, _ = mnew([x])
    torch.cuda.synchronize()
    assert L.launch_count() - before == WEIGHT_PACKS + FORWARD_LAUNCHES
    agree = float((pnew.argmax(1) == pref.argmax(1)).float().mean())
    assert agree >= 0.999, agree


def test_autograd_runs_the_reference_forward_bitwise(mods):
    """(D)"""
    ref_mod, fused_mod = mods
    x = inputs(2, 4096, True)
    labels = torch.randint(0, 17, (2, 4096), generator=torch.Generator().manual_seed(9)).cuda()
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False
    torch.use_deterministic_algorithms(True, warn_only=True)
    results = []
    try:
        for mod in (ref_mod, fused_mod):
            m = build(mod)
            assert not pointnet.fusable(m, [x])
            before = L.launch_count()
            pred, trans_feat = m([x])
            (F.nll_loss(pred, labels) + 1e-3 * trans_feat.square().sum()).backward()
            torch.cuda.synchronize()
            results.append(([pred.detach(), trans_feat.detach()], [p.grad.clone() for p in m.parameters() if p.grad is not None],
                            L.launch_count() - before, {k: v.clone() for k, v in m.state_dict().items()}))
    finally:
        torch.use_deterministic_algorithms(False)
    (o0, g0, n0, s0), (o1, g1, n1, s1) = results
    assert n0 == 0 and n1 == 0
    assert all(torch.equal(a.view(torch.int32), b.view(torch.int32)) for a, b in zip(o0, o1))
    assert len(g0) == len(g1) and all(torch.equal(a.view(torch.int32), b.view(torch.int32)) for a, b in zip(g0, g1))
    assert all(torch.equal(s0[k], s1[k]) for k in s0)


def test_memory_and_ops_of_one_forward(mods):
    """(E): the largest buffer is head conv1's (1024, N) pre-activation, 98 MB; (F): no batch_norm, bmm, cat or repeat, and conv4
    is the only convolution"""
    _, fused_mod = mods
    x = inputs(1, 24000, True)
    m = build(fused_mod)
    with torch.no_grad():
        m([x])                                                             # weights packed, allocator warm
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        before = L.launch_count()
        out, trans_feat = m([x])
        torch.cuda.synchronize()
    grew = torch.cuda.max_memory_allocated() - base
    assert L.launch_count() - before == FORWARD_LAUNCHES
    assert grew <= 256 << 20, grew
    assert out.shape == (1, 17, 24000) and trans_feat.shape == (1, 128, 128)
    with torch.no_grad(), torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU]) as prof:
        m([x])
        torch.cuda.synchronize()
    names = [e.name for e in prof.events()]
    assert not [n for n in names if "batch_norm" in n or n in ("aten::bmm", "aten::cat", "aten::repeat")], sorted(set(names))
    assert names.count("aten::convolution") == 1, sorted(set(names))


def _strided(B, C, N, layout, g):
    if layout == "strided":                                                # every other channel, every third point, offset
        return torch.randn(B, 2 * C + 1, 3 * N, generator=g).cuda()[:, 1::2, ::3]
    if layout == "permuted":
        return torch.randn(B, N, C, generator=g).cuda().permute(0, 2, 1)
    return torch.randn(B, C, N, generator=g).cuda()


@pytest.mark.parametrize("ct,cpass,N,layout", [(3, 3, 1000, "permuted"), (3, 3, 129, "strided"), (64, 5, 333, "strided"),
                                               (128, 0, 4095, "strided"), (128, 0, 24000, "contiguous"), (128, 3, 200, "permuted")])
def test_cloud_transform_against_float64(ct, cpass, N, layout):
    """(G): |got - exact| <= (ct + 1) 2^-24 sum_i |x_i| |T_ij| per element, pass-through channels bitwise, output strides honoured"""
    B, C = 3, ct + cpass
    g = torch.Generator().manual_seed(ct * 1000 + N)
    x = _strided(B, C, N, layout, g)
    t = (torch.randn(B, ct, ct, generator=g) / ct ** 0.5).cuda()
    base = torch.full((B, N, C + 3), float("nan"), device="cuda")
    out = base[:, :, 1:C + 1].permute(0, 2, 1)                            # (B, C, N) with strides (N (C + 3), 1, C + 3)
    pointnet.cloud_transform(x, t, out)
    torch.cuda.synchronize()
    xd, td = x[:, :ct].double(), t.double()
    exact = torch.einsum("bin,bij->bjn", xd, td)
    bound = (ct + 1) * 2.0 ** -24 * torch.einsum("bin,bij->bjn", xd.abs(), td.abs())
    assert bool(((out[:, :ct].double() - exact).abs() <= bound).all())
    assert torch.equal(out[:, ct:].contiguous().view(torch.int32), x[:, ct:].contiguous().view(torch.int32))
    assert bool(base[:, :, 0].isnan().all()) and bool(base[:, :, C + 1:].isnan().all())
    with pytest.raises(L.TgnError):
        L.call("tgn_pw_cloud_transform", B, N, 129, 0, L.ptr(x), *x.stride(), L.ptr(t), 0, L.ptr(out), *out.stride(), L.stream_ptr())


def _modify(m, what):
    if what == "momentum_none":
        m.feat.stn.bn2.momentum = None
    elif what == "kernel_size":
        m.conv2 = nn.Conv1d(m.conv2.in_channels, m.conv2.out_channels, 3, padding=1).cuda()
    elif what == "double":
        m.double()
    elif what == "eval":
        m.eval()
    elif what == "no_fstn_bn_affine":
        m.feat.fstn.bn1 = nn.BatchNorm1d(m.feat.fstn.bn1.num_features, affine=False).cuda()
    return m


@pytest.mark.parametrize("what", ["momentum_none", "kernel_size", "double", "grad", "eval", "no_fstn_bn_affine"])
def test_refused_calls_run_the_reference_forward(mods, what):
    ref_mod, fused_mod = mods
    x = inputs(2, 4096, True)
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False
    outs = []
    for mod in (ref_mod, fused_mod):
        m = build(mod)
        with torch.no_grad():
            assert pointnet.fusable(m, [x])                               # refused for the change alone
        m = _modify(m, what)
        xin = x.double() if what == "double" else x
        before = L.launch_count()
        with torch.set_grad_enabled(what == "grad"):
            assert not pointnet.fusable(m, [xin])
            pred, trans_feat = m([xin])
            outs.append((pred.detach(), trans_feat.detach()))
        torch.cuda.synchronize()
        assert L.launch_count() == before
    assert all(torch.equal(a, b) for a, b in zip(outs[0], outs[1]))
