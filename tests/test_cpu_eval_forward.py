"""CPU: the host side of the eval-mode forwards of DGCNN and PointNet -- what ``eval_fusable`` accepts and refuses from attributes
alone, the opt-in routing of ``accelerate_forward(..., running_stats=True)`` and its drop-ins, the ``accum`` descriptor field, and
the compiler's report for both instantiations of the layer kernel (csrc/pw_mlp.cu: one accumulator over K, unchanged at 227
registers; csrc/pw_mlp_promoted.cu: promoted accumulation)."""
import copy
import ctypes
import os
import re
import shutil
import subprocess
import sys
import types

import pytest
import torch
from torch import nn

from oracle import ref_models
from toothgroupnetwork_b200 import _lib as L
from toothgroupnetwork_b200 import build, dgcnn, dropin, pointnet
from toothgroupnetwork_b200 import pointnet2_utils as pn2

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KERNEL = "pw_layer_kernel"


def _layer(cin, cout, two_d):
    conv, bn = (nn.Conv2d, nn.BatchNorm2d) if two_d else (nn.Conv1d, nn.BatchNorm1d)
    return nn.Sequential(conv(cin, cout, kernel_size=1, bias=False), bn(cout), nn.LeakyReLU(negative_slope=0.2))


class FakeDGCnn(nn.Module):
    """the attribute layout of the DGCNN model at small widths"""

    def __init__(self, c_in=6, w=(8, 8, 8), emb=16, k=4):
        super().__init__()
        self.k = k
        self.conv1, self.conv2 = _layer(2 * c_in, 8, True), _layer(8, w[0], True)
        self.conv3, self.conv4 = _layer(2 * w[0], 8, True), _layer(8, w[1], True)
        self.conv5 = _layer(2 * w[1], w[2], True)
        self.conv6 = _layer(sum(w), emb, False)
        self.conv7, self.conv8 = _layer(emb + sum(w), 12, False), _layer(12, 10, False)
        self.dp1 = nn.Dropout(0.5)
        self.cls_conv = nn.Conv1d(10, 5, kernel_size=1, bias=False)

    def forward(self, x_in):
        return "original"


def _load_pointnet(name):
    import importlib.util
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


needs_reference = pytest.mark.skipif(not ref_models.available(), reason="reference snapshot not staged")


@pytest.fixture(scope="module")
def pn_model():
    torch.manual_seed(0)
    return _load_pointnet("ref_pointnet_eval_cpu").get_model()


def _cases(model, lib):
    """(name, module, x, expected eval_fusable, expected fusable) for one model whose BatchNorms are ``bns``"""
    x = torch.zeros(1, 6, 100)
    yield "train", model, x, True, True
    m = copy.deepcopy(model).eval()
    yield "eval", m, x, True, False
    m = copy.deepcopy(model)
    lib(m)[3].eval()
    yield "mixed", m, x, True, False
    m = copy.deepcopy(model).eval()
    lib(m)[0].momentum = None
    yield "eval_momentum_none", m, x, False, False
    m = copy.deepcopy(model).eval().double()
    yield "eval_float64", m, x.double(), False, False


def _dgcnn_bns(m):
    return [getattr(m, n)[1] for n in dgcnn._LAYERS]


def _check(mod, model, lib, monkeypatch):
    monkeypatch.setattr(mod, "input_ok", lambda *a: a[1] == torch.float32)             # as if the input were on the GPU
    with torch.no_grad():
        for name, m, x, want_eval, want in _cases(model, lib):
            assert mod.eval_fusable(m, [x]) == want_eval, name
            assert mod.fusable(m, [x]) == want, name
    for name, m, x, _, _ in _cases(model, lib):
        assert not mod.eval_fusable(m, [x]), name                                       # parameters require grad
    m = copy.deepcopy(model).eval().requires_grad_(False)
    assert mod.eval_fusable(m, [torch.zeros(1, 6, 100)])
    assert not mod.eval_fusable(m, [torch.zeros(1, 6, 100).requires_grad_(True)])       # the input requires grad
    monkeypatch.undo()
    with torch.no_grad():
        assert not mod.eval_fusable(m, [torch.zeros(1, 6, 100)])                         # a CPU tensor
        assert not mod.eval_fusable(m, [])
        assert not mod.eval_fusable(m, None)
        assert not mod.eval_fusable(m, ["not a tensor"])
        assert not mod.eval_fusable(types.SimpleNamespace(k=4), [torch.zeros(1, 6, 100)])  # wrong structure


def test_dgcnn_eval_fusable_from_attributes(monkeypatch):
    monkeypatch.setattr(L, "call", lambda *a, **kw: (_ for _ in ()).throw(AssertionError("touched the library")))
    _check(dgcnn, FakeDGCnn(), _dgcnn_bns, monkeypatch)


@needs_reference
def test_pointnet_eval_fusable_from_attributes(pn_model, monkeypatch):
    monkeypatch.setattr(L, "call", lambda *a, **kw: (_ for _ in ()).throw(AssertionError("touched the library")))
    _check(pointnet, pn_model, pointnet._bns, monkeypatch)


def test_dgcnn_eval_needs_no_second_value():
    """eval mode normalises with running statistics: one point is enough, as in torch; any train-mode BatchNorm needs two values"""
    assert dgcnn.input_ok(True, torch.float32, (1, 6, 1), 1, 6, False)
    assert not dgcnn.input_ok(True, torch.float32, (1, 6, 1), 1, 6, True)


def _route(mod, cls_name, base, monkeypatch, wrap):
    """wrapped class with forward / fusable stubs: which path each call takes"""
    holder = types.SimpleNamespace(**{cls_name: type(cls_name, (base,), {"forward": lambda self, x_in: "original"})})
    wrap(holder)
    cls = getattr(holder, cls_name)
    monkeypatch.setattr(mod, "forward", lambda module, x_in, promote=False: "promoted" if promote else "fused")
    monkeypatch.setattr(mod, "fusable", lambda module, x_in: module.kind == "train")
    monkeypatch.setattr(mod, "eval_fusable", lambda module, x_in: module.kind in ("train", "eval"))
    return holder, cls


@pytest.mark.parametrize("model", ["dgcnn", "pointnet"])
def test_running_stats_is_opt_in(model, monkeypatch):
    mod, cls_name, key = (dgcnn, "DGCnnModule", "models.modules.dgcnn") if model == "dgcnn" else (pointnet, "get_model", "models.modules.pointnet")
    drop = dropin.accelerate_dgcnn_forward if model == "dgcnn" else dropin.accelerate_pointnet_forward

    class Base:
        def __init__(self, kind):
            self.kind = kind

        def __call__(self, x_in):
            return type(self).forward(self, x_in)

    holder, cls = _route(mod, cls_name, Base, monkeypatch, mod.accelerate_forward)
    wrapped = cls.forward
    x = [torch.zeros(1)]
    assert [cls(k)(x) for k in ("train", "eval", "grad")] == ["fused", "original", "original"]     # the default: as before
    mod.accelerate_forward(holder)
    assert cls.forward is wrapped and cls("eval")(x) == "original"                                 # a plain second call
    monkeypatch.setitem(sys.modules, key, holder)
    drop(running_stats=True)                                                                       # a later call turns it on
    assert cls.forward is wrapped
    assert [cls(k)(x) for k in ("train", "eval", "grad")] == ["fused", "promoted", "original"]
    drop()                                                                                         # ... and the default keeps it
    assert cls.forward is wrapped and cls("eval")(x) == "promoted"
    fresh, fcls = _route(mod, cls_name, Base, monkeypatch, lambda h: drop(h, running_stats=True))   # on from the first call
    assert [fcls(k)(x) for k in ("train", "eval", "grad")] == ["fused", "promoted", "original"]


def test_chain_promotes_exactly_the_running_statistics_layers(monkeypatch):
    """_PwChain.run: accum = 1 on the layers whose own BatchNorm uses running statistics, and only with promote=True; the
    extrema of a promoted last layer merge with atomics when the group does not divide its 64-row half tile"""
    seen = []

    def call(name, *args):
        if name == "tgn_pw_layer_forward":
            d = args[0]._obj
            seen.append((d.accum, d.in_affine, d.extrema_atomic))
        elif name == "tgn_pw_packed_bytes":
            return 0

    class FakeLib:
        def tgn_pw_packed_bytes(self, cout, cin):
            return 16

    monkeypatch.setattr(L, "call", call)
    monkeypatch.setattr(L, "load", lambda: FakeLib())
    monkeypatch.setattr(L, "stream_ptr", lambda: None)
    monkeypatch.setattr(L, "ptr", lambda t: None)
    monkeypatch.setattr(torch.cuda, "Event", lambda: types.SimpleNamespace(record=lambda: None))
    monkeypatch.setattr(torch.cuda, "current_stream", lambda: None)
    convs = [nn.Conv1d(4, 8, 1), nn.Conv1d(8, 8, 1), nn.Conv1d(8, 6, 1)]
    bns = [nn.BatchNorm1d(8), nn.BatchNorm1d(8).eval(), nn.BatchNorm1d(6).eval()]
    out = torch.empty(2, 6, 1)
    for promote, want in ((False, [0, 0, 0]), (True, [0, 1, 1])):
        seen.clear()
        pn2._PwChain().run(convs, bns, L.PwLayer(), 2 * 128, out, 0, 1, group=128, promote=promote)
        assert [s[0] for s in seen] == want, (promote, seen)
        assert seen[-1][2] == (1 if promote else 0)           # 128 fills a 256-row tile's half but not a 128-row tile's
    for b in bns:
        b.train()
    seen.clear()
    pn2._PwChain().run(convs, bns, L.PwLayer(), 2 * 128, out, 0, 1, group=128, promote=True)
    assert [s[0] for s in seen] == [0, 0, 0]


def test_descriptor_field():
    lib = L.load()
    assert lib.tgn_pw_struct_size(0) == ctypes.sizeof(L.PwLayer) == 328       # the field sits in what was padding after `mode`
    assert L.PwLayer.accum.offset == L.PwLayer.mode.offset + 4 and L.PwLayer.seg_ptr.offset == 24
    with open(os.path.join(ROOT, "include", "tgn_b200.h")) as f:
        header = " ".join(f.read().split())
    assert "int mode; int accum;" in header
    assert "pw_mlp_promoted.cu" in build.SOURCES


def _ptxas(src, tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    res = subprocess.run([nvcc] + build.NVCC_FLAGS + ["-Xptxas", "-v", "-c", os.path.join(build.CSRC, src), "-o", str(tmp_path / "k.o")],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    out, current = {}, None
    for line in (res.stdout + res.stderr).splitlines():
        m = re.search(r"Compiling entry function '(\w+)'", line)
        if m:
            current = m.group(1) if KERNEL in m.group(1) else None
            if current:
                out.setdefault(current, [])
            continue
        m = re.search(r"in (?:the )?function '(\w+)", line)
        if m and KERNEL in m.group(1):
            out.setdefault(m.group(1), []).append(line)
        elif current:
            out[current].append(line)
    return out


@pytest.mark.parametrize("src,regs", [("pw_mlp.cu", 227), ("pw_mlp_promoted.cu", None)])
def test_layer_kernel_codegen(src, regs, tmp_path):
    """one instantiation per file; no spills; at most 255 registers (227 exactly for the existing one); no serialised wgmma"""
    kernels = _ptxas(src, tmp_path)
    assert len(kernels) == 1, sorted(kernels)
    name, lines = next(iter(kernels.items()))
    assert ("ILi256ELi0E" if regs else "ILi128ELi1E") in name, name
    spills = [re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", l) for l in lines]
    spills = [m for m in spills if m]
    assert spills and all(m.group(1) == "0" and m.group(2) == "0" for m in spills), lines
    used = [int(m.group(1)) for m in (re.search(r"Used (\d+) registers", l) for l in lines) if m]
    assert len(used) == 1 and (used[0] == regs if regs else used[0] <= 255), used
    bad = [l.strip() for l in lines if re.search(r"\(C75(1[4-8]|20)\)", l) or "mma_async instructions are serialized" in l
           or "warpgroup.wait is injected" in l]
    assert not bad, bad
