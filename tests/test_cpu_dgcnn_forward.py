"""CPU: the host side of DGCNN's fused no-grad forward (toothgroupnetwork_b200.dgcnn.forward) -- what ``fusable`` accepts and
refuses before any device work, ``accelerate_forward``'s wrapping, its idempotence and its stepping aside under autograd, the
ctypes mirror of the pw_mlp descriptors, the imports, and the code generation of csrc/pw_mlp.cu."""
import ctypes
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

from toothgroupnetwork_b200 import _lib as L
from toothgroupnetwork_b200 import build, dgcnn, dropin

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _layer(cin, cout, two_d):
    conv, bn = (nn.Conv2d, nn.BatchNorm2d) if two_d else (nn.Conv1d, nn.BatchNorm1d)
    return nn.Sequential(conv(cin, cout, kernel_size=1, bias=False), bn(cout), nn.LeakyReLU(negative_slope=0.2))


class FakeDGCnn(nn.Module):
    """the attribute layout of the DGCNN model (three EdgeConvs, conv6-8, dp1, cls_conv) at small widths, built on the CPU"""

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


def test_structure_of_the_model_is_accepted():
    m = FakeDGCnn()
    assert dgcnn.structure_ok(m)
    assert dgcnn.structure_ok(FakeDGCnn(c_in=3, w=(64, 32, 16), emb=40, k=20))


@pytest.mark.parametrize("change", ["relu", "bias", "kernel_size", "groups", "stride", "momentum_none", "no_affine", "float64",
                                    "missing_conv6", "short_sequential", "cls_width", "edge_width_65", "conv7_width"])
def test_structure_refusals(change):
    m = FakeDGCnn()
    if change == "relu":
        m.conv3[2] = nn.ReLU()
    elif change == "bias":
        m.conv2[0] = nn.Conv2d(8, 8, 1, bias=True)
    elif change == "kernel_size":
        m.conv8[0] = nn.Conv1d(12, 10, 3, padding=1, bias=False)
    elif change == "groups":
        m.conv4[0] = nn.Conv2d(8, 8, 1, groups=2, bias=False)
    elif change == "stride":
        m.conv7[0] = nn.Conv1d(40, 12, 1, stride=2, bias=False)
    elif change == "momentum_none":
        m.conv5[1].momentum = None
    elif change == "no_affine":
        m.conv6[1] = nn.BatchNorm1d(16, affine=False)
    elif change == "float64":
        m.conv1.double()
    elif change == "missing_conv6":
        del m.conv6
    elif change == "short_sequential":
        m.conv2 = nn.Sequential(m.conv2[0], m.conv2[1])
    elif change == "cls_width":
        m.cls_conv = nn.Conv1d(11, 5, 1, bias=False)
    elif change == "edge_width_65":
        m = FakeDGCnn(w=(65, 8, 8))
    elif change == "conv7_width":
        m.conv7 = _layer(41, 12, False)
    assert not dgcnn.structure_ok(m), change


def test_input_checks():
    ok = dict(is_cuda=True, dtype=torch.float32, shape=(2, 6, 4096), k=20, c_in=6, training=True)
    assert dgcnn.input_ok(**ok)
    assert dgcnn.input_ok(**{**ok, "shape": (1, 6, 20)})
    assert dgcnn.input_ok(**{**ok, "k": 32})
    for change in ({"is_cuda": False}, {"dtype": torch.float64}, {"dtype": torch.float16}, {"shape": (2, 6)}, {"shape": (2, 7, 4096)},
                   {"shape": (2, 65, 4096), "c_in": 65}, {"shape": (1, 6, 19)}, {"k": 33}, {"k": 0}, {"k": 20.0},
                   {"shape": (1, 6, 1), "k": 1}):
        assert not dgcnn.input_ok(**{**ok, **change}), change
    assert dgcnn.input_ok(**{**ok, "shape": (1, 6, 1), "k": 1, "training": False})


def test_fusable_refuses_before_device_work(monkeypatch):
    def no_device_work(*a, **kw):
        raise AssertionError("fusable touched the library")

    monkeypatch.setattr(L, "call", no_device_work)
    m = FakeDGCnn()
    x = torch.zeros(1, 6, 100)
    assert not dgcnn.fusable(m, [x])                                    # CPU tensor
    assert not dgcnn.fusable(m, [])
    assert not dgcnn.fusable(m, None)
    assert not dgcnn.fusable(m, ["not a tensor"])
    assert not dgcnn.fusable(types.SimpleNamespace(k=20), [x])


def test_fusable_steps_aside_under_autograd(monkeypatch):
    monkeypatch.setattr(dgcnn, "input_ok", lambda *a: True)             # as if the input were on the GPU
    m = FakeDGCnn()
    x = torch.zeros(1, 6, 100)
    assert not dgcnn.fusable(m, [x])                                    # parameters require grad
    with torch.no_grad():
        assert dgcnn.fusable(m, [x])
    m.requires_grad_(False)
    assert dgcnn.fusable(m, [x])
    assert not dgcnn.fusable(m, [x.clone().requires_grad_(True)])
    m.conv6[1].eval()                                                   # running statistics: the reference's forward
    assert not dgcnn.fusable(m, [x])
    m.conv6[1].track_running_stats, m.conv6[1].running_mean, m.conv6[1].running_var = False, None, None
    assert dgcnn.fusable(m, [x])                                        # eval mode without running statistics: batch statistics


def test_accelerate_forward_wraps_once_and_routes(monkeypatch):
    mod = types.SimpleNamespace(DGCnnModule=type("DGCnnModule", (FakeDGCnn,), {"forward": lambda self, x_in: "original"}))
    dgcnn.accelerate_forward(mod)
    wrapped = mod.DGCnnModule.forward
    dgcnn.accelerate_forward(mod)
    dgcnn.accelerate_forward(mod.DGCnnModule)
    assert mod.DGCnnModule.forward is wrapped
    m = mod.DGCnnModule()
    x = torch.zeros(1, 6, 100)
    monkeypatch.setattr(dgcnn, "forward", lambda module, x_in: "fused")
    with torch.no_grad():
        assert m([x]) == "original"                                     # CPU input
    monkeypatch.setattr(dgcnn, "input_ok", lambda *a: True)
    assert m([x]) == "original"                                         # autograd
    with torch.no_grad():
        assert m([x]) == "fused"
    monkeypatch.setitem(sys.modules, "models.modules.dgcnn", mod)
    dropin.accelerate_dgcnn_forward()
    assert mod.DGCnnModule.forward is wrapped


def test_descriptor_mirror_matches_the_library():
    lib = L.load()                                                      # raises when the ctypes mirror is out of date
    assert lib.tgn_pw_struct_size(0) == ctypes.sizeof(L.PwLayer) and lib.tgn_pw_struct_size(1) == ctypes.sizeof(L.PwApply)
    names = [f[0] for f in L.PwLayer._fields_]
    assert names[-6:] == ["edge_x", "edge_stride", "edge_C", "in_act", "in_act_slope", "cloud_bias"]
    assert [f[0] for f in L.PwApply._fields_][-2:] == ["act", "act_slope"]
    with open(os.path.join(ROOT, "include", "tgn_b200.h")) as f:
        header = " ".join(f.read().split())
    assert ("int precision; /* 0 / 3: three bf16 parts per operand, six MMAs per K step (fp32-grade); 2: two parts, three MMAs (~1e-5) */ "
            "const float *edge_x; /* mode 2 */ long long edge_stride[3]; int edge_C; int in_act; float in_act_slope; const float *cloud_bias; "
            "} tgn_pw_layer_t;") in header
    assert "tgn_pw_cloud_bias" in L._SIGS and "tgn_pw_cloud_bias" in L.EXPORTS
    assert "float eps, momentum; int act; float act_slope; } tgn_pw_apply_t;" in header


def test_dgcnn_imports_neither_the_checkers_nor_the_reference():
    code = ("import sys; import toothgroupnetwork_b200.dgcnn, toothgroupnetwork_b200.dropin; "
            "bad = sorted(m for m in sys.modules if m.split('.')[0] in ('oracle', 'oracle_dgcnn', 'models')); assert not bad, bad")
    res = subprocess.run([sys.executable, "-c", code], cwd=ROOT, capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr


def test_pw_mlp_kernels_do_not_spill():
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    out = os.path.join(tempfile.gettempdir(), f"pw_mlp_{os.getpid()}.o")
    cmd = [nvcc] + build.NVCC_FLAGS + ["-Xptxas", "-v", "-c", os.path.join(build.CSRC, "pw_mlp.cu"), "-o", out]
    res = subprocess.run(cmd, capture_output=True, text=True)
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
            seen[current] = (m.group(1), m.group(2))
    assert len(seen) == 5 and any("pw_layer_kernel" in k for k in seen), seen      # layer, apply, pack, fill, cloud bias
    assert all(v == ("0", "0") for v in seen.values()), seen
