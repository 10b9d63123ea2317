"""GPU: the eval-mode (running-statistics BatchNorm) no-grad forwards of DGCNN and PointNet on the layer chain with promoted
accumulation (``dgcnn.forward`` / ``pointnet.forward`` with ``promote=True``, reached through ``accelerate_forward(...,
running_stats=True)``), against the reference's own modules (models/modules/dgcnn.py, models/modules/pointnet.py through
oracle.ref_models).

Running statistics come (i) from one reference pass over the same batch, or (ii) from a pass over different seeded clouds, so
that per-cloud offsets survive the running-mean subtraction (what moved DGCNN's conv8 2-3x past the reference's own distance
with a single accumulator, DESIGN §3.12).  BatchNorm affines are seeded, with negative scales.

* (A) against float64 (DGCNN with the reference fp32 run's neighbours): DGCNN x1|x2|x3, conv8's activation and cls_pred; PointNet
  trans, trans_feat, g, pointfeat, head conv3 and the log-probabilities -- within 1e-4 element-wise or twice the reference fp32
  run's distance (cuDNN TF32 off);
* (B) the running statistics and num_batches_tracked bitwise unchanged;
* (C) one train-mode BatchNorm among eval ones: its running statistics updated within the same bar, the others untouched;
* (D) with each side's own neighbours, argmax: PointNet against the reference's fp32 run on >= 99.9 % of the points; DGCNN
  against float64, no more than 1.25x as many points off as the reference's fp32 run (which itself is 0.3-0.7 % off);
* (E) autograd, and eval mode on a class wrapped without running_stats, run the reference's forward bitwise; all-train calls
  are bitwise the same with and without running_stats;
* (F) the peak memory of one (1, 24 000) forward; (G) the torch ops it runs."""
import copy
import importlib.util
import os
import sys

import pytest
import torch
import torch.nn.functional as F

from oracle import ref_models
from toothgroupnetwork_b200 import _lib as L
from toothgroupnetwork_b200 import clouds, dgcnn, dropin, pointnet

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not ref_models.available(), reason="reference snapshot not staged")]
REL_TOL, FLOOR = 1e-4, 0.05
DGCNN_BNS = ("bn1", "bn2", "bn3", "bn4", "bn5", "bn6", "bn7", "bn8")


def elementwise(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float(((a - b).abs() / b.abs().clamp(min=FLOOR * float(b.abs().max()))).max())


def _load_dgcnn(name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ref_models.reference_root(), "models", "modules", "dgcnn.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _load_pointnet(name):
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
    """{model: (unwrapped reference module, wrapped with running_stats=True, wrapped with the default)}"""
    out = {}
    for model, load, wrap in (("dgcnn", _load_dgcnn, dropin.accelerate_dgcnn_forward), ("pointnet", _load_pointnet, dropin.accelerate_pointnet_forward)):
        ref, on, off = load(f"ref_{model}_eval_a"), load(f"ref_{model}_eval_b"), load(f"ref_{model}_eval_c")
        wrap(on)
        wrap(on, running_stats=True)                                        # a later call turns the eval-mode routing on
        wrap(off)
        out[model] = (ref, on, off)
    return out


@pytest.fixture(autouse=True)
def fp32_settings():
    saved = torch.backends.cudnn.allow_tf32, torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = saved


def inputs(B, N, permuted, seed=0):
    f = torch.cat([clouds.arch_features(N, seed + b) for b in range(B)]).cuda()
    return f.transpose(1, 2).contiguous().permute(0, 2, 1) if permuted else f.contiguous()


def _bns(model, m):
    return [getattr(m, n) for n in DGCNN_BNS] if model == "dgcnn" else pointnet._bns(m)


def build(model, mod, x, stats="same", seed=0, affines=True):
    """seeded module in eval mode, seeded BatchNorm affines (gamma in [-1, 2): negative scales) when ``affines``; running statistics
    of one train-mode reference pass (momentum 1) over x ("same") or over different seeded clouds of the same shape ("other")"""
    torch.manual_seed(seed)
    m = (mod.DGCnnModule(None) if model == "dgcnn" else mod.get_model()).cuda()
    g = torch.Generator().manual_seed(seed + 1)
    bns = _bns(model, m)
    with torch.no_grad():
        for bn in bns if affines else ():
            bn.weight.copy_(torch.rand(bn.num_features, generator=g) * 3.0 - 1.0)
            bn.bias.copy_(torch.rand(bn.num_features, generator=g) * 0.4 - 0.2)
    src = x if stats == "same" else inputs(x.shape[0], x.shape[2], False, seed=100)
    for bn in bns:
        bn.momentum = 1.0
    m.train()
    with torch.enable_grad():                 # the reference's forward, also on a wrapped class
        m([src])
    for bn in bns:
        bn.momentum = 0.1
        bn.num_batches_tracked.zero_()
    return m.eval()


def _state(m):
    return {k: v.clone() for k, v in m.state_dict().items()}


class DgcnnTaps:
    def __init__(self, m):
        self.d = {}
        self.h = [m.conv6.register_forward_pre_hook(lambda _m, inp: self.d.__setitem__("x123", inp[0].detach().clone())),
                  m.dp1.register_forward_hook(lambda _m, inp, out: self.d.__setitem__("conv8", inp[0].detach().clone()))]

    def close(self):
        for h in self.h:
            h.remove()


class PointnetTaps:
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


def reference_run(model, mod, m, x, pinned=None):
    """-> ({name: tensor} of the compared quantities, the kNN indices in call order)"""
    seen = []
    if model == "dgcnn":
        original = mod.knn

        def knn(v, k):
            idx = pinned[len(seen)] if pinned is not None else original(v, k)
            seen.append(idx)
            return idx

        taps = DgcnnTaps(m)
        mod.knn = knn
        try:
            with torch.no_grad():
                out = {"cls_pred": m([x])["cls_pred"]}
        finally:
            mod.knn = original
            taps.close()
        out.update(x123=taps.d["x123"], conv8=taps.d["conv8"])
        return out, seen
    taps = PointnetTaps(m)
    try:
        with torch.no_grad():
            logp, trans_feat = m([x])
    finally:
        taps.close()
    return dict(taps.d, trans_feat=trans_feat, log_softmax=logp), seen


def fused_run(model, m, x, pinned=None):
    keep = {}
    with torch.no_grad():
        if model == "dgcnn":
            it = iter(pinned) if pinned is not None else None
            out = {"cls_pred": dgcnn.forward(m, [x], knn=(lambda v, k: next(it)) if it is not None else None, keep=keep, promote=True)["cls_pred"]}
            out.update(x123=keep["x123"], conv8=keep["conv8"])
            return out
        logp, trans_feat = pointnet.forward(m, [x], keep=keep, promote=True)
    return {"trans": keep["trans"], "trans_feat": trans_feat, "g": keep["g"], "pointfeat": keep["pointfeat"], "head3": keep["head3"],
            "log_softmax": logp}


def _against_float64(model, mods, x, stats, train_bn=None):
    """(A) and (B) / (C): returns nothing, asserts"""
    ref_mod = mods[model][0]
    m32 = build(model, ref_mod, x, stats)
    if train_bn is not None:
        _bns(model, m32)[train_bn].train()
    m64, mnew, m_before = copy.deepcopy(m32).double(), copy.deepcopy(m32), copy.deepcopy(m32)
    before = _state(mnew)
    with torch.no_grad():
        assert not (model == "dgcnn" and dgcnn.fusable(mnew, [x])) and not (model == "pointnet" and pointnet.fusable(mnew, [x]))
        assert (dgcnn if model == "dgcnn" else pointnet).eval_fusable(mnew, [x])
    r32, idx = reference_run(model, ref_mod, m32, x)
    r64, _ = reference_run(model, ref_mod, m64, x.double(), pinned=idx if model == "dgcnn" else None)
    got = fused_run(model, mnew, x, pinned=idx if model == "dgcnn" else None)
    torch.cuda.synchronize()
    report = {}
    for name in r32:
        e_ours, e_fp32 = elementwise(got[name], r64[name]), elementwise(r32[name], r64[name])
        report[name] = (e_ours, e_fp32)
    print(model, tuple(x.shape), stats, train_bn, {k: f"{a:.2e} (fp32 {b:.2e})" for k, (a, b) in report.items()})
    for name, (e_ours, e_fp32) in report.items():
        assert e_ours <= max(REL_TOL, 2.0 * e_fp32), (name, e_ours, e_fp32)
    after = _state(mnew)
    names = [n for n in after if n.endswith(("running_mean", "running_var", "num_batches_tracked"))]
    if train_bn is None:
        assert all(torch.equal(before[k], after[k]) for k in names)                                    # (B)
        return
    # (C) the train-mode BatchNorm's running statistics move as the reference's do; every other one stays as it was
    for i, (bn, bn_before) in enumerate(zip(_bns(model, mnew), _bns(model, m_before))):
        if i != train_bn:
            for stat in ("running_mean", "running_var", "num_batches_tracked"):
                assert torch.equal(getattr(bn, stat), getattr(bn_before, stat)), (i, stat)
    bn_new, bn32, bn64 = (_bns(model, mm)[train_bn] for mm in (mnew, m32, m64))
    assert int(bn_new.num_batches_tracked) == int(bn32.num_batches_tracked) == 1
    for stat in ("running_mean", "running_var"):
        e_ours, e_fp32 = elementwise(getattr(bn_new, stat), getattr(bn64, stat)), elementwise(getattr(bn32, stat), getattr(bn64, stat))
        assert e_ours <= max(REL_TOL, 2.0 * e_fp32), (stat, e_ours, e_fp32)


@pytest.mark.parametrize("stats", ["same", "other"])
@pytest.mark.parametrize("B,N,permuted", [(1, 4096, False), (2, 4096, True), (1, 24000, True), (2, 24000, False)])
@pytest.mark.parametrize("model", ["dgcnn", "pointnet"])
def test_eval_against_float64(mods, model, B, N, permuted, stats):
    """(A) and (B)"""
    _against_float64(model, mods, inputs(B, N, permuted), stats)


@pytest.mark.parametrize("model,train_bn", [("dgcnn", 5), ("dgcnn", 7), ("pointnet", 7), ("pointnet", 10)])
def test_mixed_modes(mods, model, train_bn):
    """(C): DGCNN bn6 (conv6, the global max) or bn8; PointNet's encoder bn2 or head bn2, in train mode among eval ones"""
    _against_float64(model, mods, inputs(2, 4096, True), "other", train_bn=train_bn)


@pytest.mark.parametrize("model", ["dgcnn", "pointnet"])
@pytest.mark.parametrize("B,N", [(1, 24000), (2, 4096)])
def test_argmax_agrees(mods, model, B, N):
    """(D) through the wrapped class, each side with its own neighbours, running statistics of other clouds.

    PointNet: argmax agrees with the reference's fp32 run on >= 99.9 % of the points.  DGCNN in eval mode: the reference's own
    fp32 run agrees with its float64 evaluation (its own neighbours too) on only 99.35-99.74 % of the points at these shapes on an
    H100 -- the layer-2 / -3 neighbour sets follow features that fp32 rounding moves by ~1e-5 -- so a 99.9 % bar against the fp32
    run is below what the exact answer meets (the fused forward: 99.69-100 % against fp32).  The bar is instead the float64
    evaluation: the fused argmax disagrees with it on at most 1.25x the share of points the reference's fp32 run does (measured
    0.99-1.01x)."""
    ref_mod, on_mod, _ = mods[model]
    x = inputs(B, N, True)
    mref = build(model, ref_mod, x, "other", affines=False)
    mnew = build(model, on_mod, x, "other", affines=False)
    mnew.load_state_dict(mref.state_dict())
    with torch.no_grad():
        pref = mref([x])
        before = L.launch_count()
        pnew = mnew([x])
    torch.cuda.synchronize()
    assert L.launch_count() > before                                                      # the fused forward ran
    pref, pnew = (pref["cls_pred"], pnew["cls_pred"]) if model == "dgcnn" else (pref[0], pnew[0])
    agree = float((pnew.argmax(1) == pref.argmax(1)).float().mean())
    if model == "pointnet":
        assert agree >= 0.999, agree
        return
    with torch.no_grad():
        p64 = copy.deepcopy(mref).double()([x.double()])["cls_pred"]
    off_new = float((pnew.argmax(1) != p64.argmax(1)).float().mean())
    off_fp32 = float((pref.argmax(1) != p64.argmax(1)).float().mean())
    print(model, B, N, f"agree with fp32 {agree:.5f}, off float64: fused {off_new:.5f}, fp32 {off_fp32:.5f}")
    assert off_new <= 1.25 * off_fp32, (off_new, off_fp32, agree)


def _outputs(model, m, x):
    torch.manual_seed(1)
    out = m([x])
    return [out["cls_pred"]] if model == "dgcnn" else list(out)


@pytest.mark.parametrize("model", ["dgcnn", "pointnet"])
def test_autograd_runs_the_reference_forward_bitwise(mods, model):
    """(E) eval mode with gradients: the running_stats wrapper runs the reference's forward"""
    ref_mod, on_mod, _ = mods[model]
    x = inputs(2, 4096, True)
    labels = torch.randint(0, 17, (2, 4096), generator=torch.Generator().manual_seed(9)).cuda()
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False
    torch.use_deterministic_algorithms(True, warn_only=True)
    results = []
    try:
        for mod in (ref_mod, on_mod):
            m = build(model, mod, x, "other")
            assert not (dgcnn if model == "dgcnn" else pointnet).eval_fusable(m, [x])
            before = L.launch_count()
            outs = _outputs(model, m, x)
            loss = F.cross_entropy(outs[0], labels) if model == "dgcnn" else F.nll_loss(outs[0], labels) + 1e-3 * outs[1].square().sum()
            loss.backward()
            torch.cuda.synchronize()
            results.append(([o.detach() for o in outs], [p.grad.clone() for p in m.parameters() if p.grad is not None],
                            L.launch_count() - before, _state(m)))
    finally:
        torch.use_deterministic_algorithms(False)
    (o0, g0, n0, s0), (o1, g1, n1, s1) = results
    assert n0 == 0 and n1 == 0
    assert all(torch.equal(a.view(torch.int32), b.view(torch.int32)) for a, b in zip(o0, o1))
    assert len(g0) == len(g1) and all(torch.equal(a.view(torch.int32), b.view(torch.int32)) for a, b in zip(g0, g1))
    assert all(torch.equal(s0[k], s1[k]) for k in s0)


@pytest.mark.parametrize("model", ["dgcnn", "pointnet"])
def test_opt_in(mods, model):
    """(E) eval mode on the class wrapped without running_stats runs the reference's forward bitwise (no launch); all-train calls
    are bitwise the same on the classes wrapped with and without it"""
    ref_mod, on_mod, off_mod = mods[model]
    x = inputs(1, 4096, True)
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False
    outs = []
    for mod in (ref_mod, off_mod):
        m = build(model, mod, x, "other")
        before = L.launch_count()
        with torch.no_grad():
            outs.append((_outputs(model, m, x), _state(m)))
        torch.cuda.synchronize()
        assert L.launch_count() == before
    assert all(torch.equal(a.view(torch.int32), b.view(torch.int32)) for a, b in zip(outs[0][0], outs[1][0]))
    assert all(torch.equal(outs[0][1][k], outs[1][1][k]) for k in outs[0][1])
    outs = []
    for mod in (off_mod, on_mod):
        m = build(model, mod, x, "other").train()
        before = L.launch_count()
        with torch.no_grad():
            outs.append((_outputs(model, m, x), _state(m)))
        torch.cuda.synchronize()
        assert L.launch_count() > before
    assert all(torch.equal(a.view(torch.int32), b.view(torch.int32)) for a, b in zip(outs[0][0], outs[1][0]))
    assert all(torch.equal(outs[0][1][k], outs[1][1][k]) for k in outs[0][1])


@pytest.mark.parametrize("model", ["dgcnn", "pointnet"])
def test_memory_and_ops(mods, model):
    """(F) peak growth of one (1, 24 000) eval forward under 256 MB; (G) no batch_norm, cat or repeat, and only the module's own
    last convolution (DGCNN cls_conv, PointNet conv4)"""
    _, on_mod, _ = mods[model]
    x = inputs(1, 24000, True)
    m = build(model, on_mod, x, "other")
    with torch.no_grad():
        m([x])                                                             # weights packed, allocator warm
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        m([x])
        torch.cuda.synchronize()
    grew = torch.cuda.max_memory_allocated() - base
    print(model, "peak growth", grew)
    assert grew < 256 << 20, grew
    with torch.no_grad(), torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU]) as prof:
        m([x])
        torch.cuda.synchronize()
    names = [e.name for e in prof.events()]
    assert not [n for n in names if "batch_norm" in n or n in ("aten::cat", "aten::repeat")], sorted(set(names))
    assert names.count("aten::convolution") == 1, sorted(set(names))
