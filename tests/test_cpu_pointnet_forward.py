"""CPU: the host side of PointNet's fused no-grad forward (toothgroupnetwork_b200.pointnet.forward) -- what ``fusable`` accepts
and refuses before any device work, on the reference's own get_model built on the CPU, ``accelerate_forward``'s wrapping, its
idempotence and its stepping aside under autograd, the ctypes signature of tgn_pw_cloud_transform, the imports, and the code
generation of csrc/pw_transform.cu and csrc/pw_mlp.cu."""
import copy
import importlib.util
import os
import re
import shutil
import subprocess
import sys
import tempfile
import types

import pytest
import torch
from torch import nn

from oracle import ref_models
from toothgroupnetwork_b200 import _lib as L
from toothgroupnetwork_b200 import build, dropin, pointnet

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
needs_reference = pytest.mark.skipif(not ref_models.available(), reason="reference snapshot not staged")


def load_reference_pointnet(name):
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
def model():
    torch.manual_seed(0)
    return load_reference_pointnet("ref_pointnet_cpu").get_model()


@needs_reference
def test_reference_model_is_accepted(model):
    assert pointnet.structure_ok(model)
    assert len(pointnet._bns(model)) == 12 and all(isinstance(b, nn.BatchNorm1d) for b in pointnet._bns(model))


def _modify(m, what):
    f = m.feat
    if what == "momentum_none":
        f.fstn.bn2.momentum = None
    elif what == "channels":
        f.conv1 = nn.Conv1d(9, f.conv1.out_channels, 1)
        f.stn.conv1 = nn.Conv1d(9, 64, 1)
    elif what == "kernel_size":
        m.conv2 = nn.Conv1d(m.conv2.in_channels, m.conv2.out_channels, 3, padding=1)
    elif what == "missing_fstn":
        del f.fstn
    elif what == "no_feature_transform":
        f.feature_transform = False
    elif what == "global_feat":
        f.global_feat = True
    elif what == "stride":
        f.conv2 = nn.Conv1d(f.conv2.in_channels, f.conv2.out_channels, 1, stride=2)
    elif what == "no_affine":
        m.bn3 = nn.BatchNorm1d(m.bn3.num_features, affine=False)
    elif what == "layer_norm":
        f.stn.bn4 = nn.BatchNorm1d(f.stn.bn4.normalized_shape[0])
    elif what == "head_width":
        m.conv4 = nn.Conv1d(m.conv4.in_channels, m.k + 1, 1)
    elif what == "float64":
        f.conv3.double()
    return m


@needs_reference
@pytest.mark.parametrize("what", ["momentum_none", "channels", "kernel_size", "missing_fstn", "no_feature_transform", "global_feat",
                                  "stride", "no_affine", "layer_norm", "head_width", "float64"])
def test_structure_refusals(model, what):
    assert not pointnet.structure_ok(_modify(copy.deepcopy(model), what)), what


def test_input_checks():
    ok = dict(is_cuda=True, dtype=torch.float32, shape=(2, 6, 24000), training=True)
    assert pointnet.input_ok(**ok)
    assert pointnet.input_ok(**{**ok, "shape": (1, 6, 2)})
    for change in ({"is_cuda": False}, {"dtype": torch.float64}, {"dtype": torch.float16}, {"shape": (2, 6)}, {"shape": (2, 3, 100)},
                   {"shape": (2, 9, 100)}, {"shape": (1, 6, 1)}, {"shape": (0, 6, 100)}, {"shape": (65536, 6, 2)}):
        assert not pointnet.input_ok(**{**ok, **change}), change
    assert pointnet.input_ok(**{**ok, "shape": (1, 6, 1), "training": False})


@needs_reference
def test_fusable_refuses_before_device_work(model, monkeypatch):
    def no_device_work(*a, **kw):
        raise AssertionError("fusable touched the library")

    monkeypatch.setattr(L, "call", no_device_work)
    x = torch.zeros(1, 6, 100)
    with torch.no_grad():
        assert not pointnet.fusable(model, [x])                             # CPU tensor
        assert not pointnet.fusable(model, [])
        assert not pointnet.fusable(model, None)
        assert not pointnet.fusable(model, ["not a tensor"])
        assert not pointnet.fusable(types.SimpleNamespace(k=17), [x])


@needs_reference
def test_fusable_steps_aside_under_autograd_and_eval_mode(model, monkeypatch):
    monkeypatch.setattr(pointnet, "input_ok", lambda *a: True)              # as if the input were on the GPU
    m = copy.deepcopy(model)
    x = torch.zeros(1, 6, 100)
    assert not pointnet.fusable(m, [x])                                     # parameters require grad
    with torch.no_grad():
        assert pointnet.fusable(m, [x])
    m.requires_grad_(False)
    assert pointnet.fusable(m, [x])
    assert not pointnet.fusable(m, [x.clone().requires_grad_(True)])
    for bn in pointnet._bns(m):
        bn.eval()                                                           # running statistics: the reference's forward
        assert not pointnet.fusable(m, [x])
        bn.train()
    m.eval()
    assert not pointnet.fusable(m, [x])


@needs_reference
def test_accelerate_forward_wraps_once_and_routes(model, monkeypatch):
    mod = types.SimpleNamespace(get_model=type("get_model", (nn.Module,), {"forward": lambda self, x_in: "original"}))
    pointnet.accelerate_forward(mod)
    wrapped = mod.get_model.forward
    pointnet.accelerate_forward(mod)
    pointnet.accelerate_forward(mod.get_model)
    assert mod.get_model.forward is wrapped
    m = mod.get_model()
    for name, child in model.named_children():
        m.add_module(name, copy.deepcopy(child))
    m.k = model.k
    x = torch.zeros(1, 6, 100)
    monkeypatch.setattr(pointnet, "forward", lambda module, x_in: "fused")
    with torch.no_grad():
        assert m([x]) == "original"                                         # CPU input
    monkeypatch.setattr(pointnet, "input_ok", lambda *a: True)
    assert m([x]) == "original"                                             # autograd
    with torch.no_grad():
        assert m([x]) == "fused"
    monkeypatch.setitem(sys.modules, "models.modules.pointnet", mod)
    dropin.accelerate_pointnet_forward()
    assert mod.get_model.forward is wrapped


_CTYPES = {"int": L._i, "long long": L.ctypes.c_longlong, "const float *": L._vp, "float *": L._vp, "void *": L._vp}


def test_cloud_transform_signature_matches_the_header():
    with open(os.path.join(ROOT, "include", "tgn_b200.h")) as f:
        header = " ".join(f.read().split())
    m = re.search(r"int tgn_pw_cloud_transform\(([^)]*)\);", header)
    assert m, "tgn_pw_cloud_transform is not declared"
    args = [re.sub(r"\s*\w+$", "", a.strip()).replace("*", " *").replace("  ", " ").strip() for a in m.group(1).split(",")]
    assert [_CTYPES[a] for a in args] == L._SIGS["tgn_pw_cloud_transform"]
    assert "tgn_pw_cloud_transform" in L.EXPORTS
    assert "pw_transform.cu" in build.SOURCES


def _ptxas_report(src):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    out = os.path.join(tempfile.gettempdir(), f"ptxas_{os.getpid()}_{os.path.basename(src)}.o")
    res = subprocess.run([nvcc] + build.NVCC_FLAGS + ["-Xptxas", "-v", "-c", os.path.join(build.CSRC, src), "-o", out],
                         capture_output=True, text=True)
    if os.path.exists(out):
        os.remove(out)
    assert res.returncode == 0, res.stdout + res.stderr
    current, seen = None, {}
    for line in (res.stdout + res.stderr).splitlines():
        m = re.search(r"Compiling entry function '(\w+)'", line)
        if m:
            current = m.group(1)
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and current:
            seen.setdefault(current, {})["spill"] = (int(m.group(1)), int(m.group(2)))
        m = re.search(r"Used (\d+) registers", line)
        if m and current:
            seen.setdefault(current, {})["regs"] = int(m.group(1))
    return seen


def test_cloud_transform_kernel_does_not_spill_and_the_chain_is_unchanged():
    new = _ptxas_report("pw_transform.cu")
    assert len(new) == 1 and "pw_cloud_transform_kernel" in next(iter(new)), new
    assert all(v["spill"] == (0, 0) for v in new.values()), new
    chain = _ptxas_report("pw_mlp.cu")
    regs = {name: v["regs"] for name, v in chain.items()}
    assert all(v["spill"] == (0, 0) for v in chain.values()), chain
    assert [r for n, r in regs.items() if "pw_layer_kernel" in n] == [227], regs
    assert [r for n, r in regs.items() if "pw_apply_kernel" in n] == [38], regs


def test_pointnet_imports_neither_the_checkers_nor_the_reference():
    code = ("import sys; import toothgroupnetwork_b200.pointnet, toothgroupnetwork_b200.dropin; "
            "bad = sorted(m for m in sys.modules if m.split('.')[0] in ('oracle', 'oracle_dgcnn', 'models', 'external_libs')); "
            "assert not bad, bad")
    res = subprocess.run([sys.executable, "-c", code], cwd=ROOT, capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
