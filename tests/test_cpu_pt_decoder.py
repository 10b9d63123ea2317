"""oracle/pt_decoder.py against the reference's own TransitionUp / MultiHead (tests/golden/ref_torch_decoder.npz), the fused
decoder's dispatch decisions from module attributes, and the ptxas report of csrc/pt_head.cu."""
import os
import re
import shutil
import subprocess
import tempfile

import numpy as np
import pytest
import torch
import torch.nn as nn

from oracle import pt_decoder as D
from toothgroupnetwork_b200 import blocks_fused, build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIX = os.path.join(ROOT, "tests", "golden", "ref_torch_decoder.npz")


def _state(fix, tag):
    pre = tag + "_state_"
    return {k[len(pre):]: torch.from_numpy(fix[k]) for k in fix.files if k.startswith(pre)}


def _within(got, err, want):
    """the float32 reference run lies within the oracle's bound (plus one rounding of the value itself)"""
    gap = (torch.from_numpy(want).double() - got).abs()
    assert bool((gap <= err + 2.0 ** -23 * got.abs() + 1e-30).all()), float((gap - err).max())


def _after(fix, tag, after):
    for k, v in after.items():
        want = torch.from_numpy(fix[f"{tag}_after_{k}"])
        if "num_batches" in k:
            assert int(v) == int(want)
        else:
            assert torch.allclose(v, want.double(), rtol=1e-5, atol=1e-6), k


@pytest.mark.parametrize("train", [True, False])
def test_transition_up_oracle_matches_reference(train):
    fix = np.load(FIX)
    mode = "train" if train else "eval"
    got, err, after = D.transition_up(_state(fix, "tu"), fix["tu_x1"], list(fix["o1"]), train, x2=fix["tu_x2"],
                                      idx=fix["interp_idx"], w=fix["interp_w"])
    _within(got, err, fix["tu_out_" + mode])
    if train:
        _after(fix, "tu", after)
    got, err, after = D.transition_up(_state(fix, "th"), fix["th_x"], list(fix["o1"]), train)
    _within(got, err, fix["th_out_" + mode])
    if train:
        _after(fix, "th", after)


@pytest.mark.parametrize("train", [True, False])
def test_multi_head_oracle_matches_reference(train):
    fix = np.load(FIX)
    mode = "train" if train else "eval"
    got, err, lats, after = D.multi_head(_state(fix, "mh"), [fix["mh_f0"], fix["mh_f1"]], [None, fix["nn1"]], train)
    _within(got, err, fix["mh_out_" + mode])
    for s, lat in enumerate(lats):
        assert torch.allclose(lat, torch.from_numpy(fix[f"mh_extra{s}_{mode}"]).double(), rtol=1e-5, atol=1e-6)
    if train:
        _after(fix, "mh", after)


class _TU(nn.Module):
    """blocks.TransitionUp's layers (blocks.py:84-90)"""

    def __init__(self, cin, cout=None):
        super().__init__()
        if cout is None:
            self.linear1 = nn.Sequential(nn.Linear(2 * cin, cin), nn.BatchNorm1d(cin), nn.ReLU(inplace=True))
            self.linear2 = nn.Sequential(nn.Linear(cin, cin), nn.ReLU(inplace=True))
        else:
            self.linear1 = nn.Sequential(nn.Linear(cout, cout), nn.BatchNorm1d(cout), nn.ReLU(inplace=True))
            self.linear2 = nn.Sequential(nn.Linear(cin, cout), nn.BatchNorm1d(cout), nn.ReLU(inplace=True))


class _MLP(nn.Module):
    def __init__(self, fdim, extra=()):
        super().__init__()
        self.infer = nn.Sequential(nn.Linear(fdim, 32), nn.BatchNorm1d(32), nn.ReLU(inplace=True), *extra)


class _MH(nn.Module):
    """heads.MultiHead with combine = concat (heads.py:14-42)"""

    def __init__(self, fdims, k, d=32):
        super().__init__()
        self.ftype = "latent"
        self.ni_list = [("up", i) for i in range(len(fdims))]
        self.infer_list = nn.ModuleList([_MLP(f) for f in fdims])
        self.cls = nn.Linear(d * len(fdims), k)


def test_fusable_decisions_from_attributes():
    ok = blocks_fused.transition_up_structure_ok
    assert ok(_TU(64, 32), False, 64, 32) and ok(_TU(512), True, 512)
    assert not ok(_TU(64, 32), False, 32, 32) and not ok(_TU(64, 32), False, 64, 64)
    assert not ok(_TU(64, 32), True, 64)                                # the head form's layers differ
    assert not ok(_TU(512), False, 512, 512)
    tu = _TU(64, 32)
    tu.linear1[1] = nn.BatchNorm1d(32, momentum=None)                   # cumulative average: torch's own
    assert not ok(tu, False, 64, 32)
    tu = _TU(64, 32)
    tu.linear2[1] = nn.BatchNorm1d(32, affine=False)
    assert not ok(tu, False, 64, 32)
    assert not ok(_TU(64, 32).double(), False, 64, 32)
    tu = _TU(64, 32)
    tu.linear1 = nn.Sequential(*list(tu.linear1)[:2])                   # no ReLU
    assert not ok(tu, False, 64, 32)

    mh_ok = blocks_fused.multi_head_structure_ok
    assert mh_ok(_MH([32, 64, 128, 256, 512], 17)) and mh_ok(_MH([16, 32], 3)) and mh_ok(_MH([32] * 8, 32))
    assert not mh_ok(_MH([32] * 9, 2)) and not mh_ok(_MH([32], 33))
    mh = _MH([32, 64], 3)
    mh.cls = nn.Sequential(nn.Linear(64, 32), nn.BatchNorm1d(32), nn.ReLU(), nn.Linear(32, 3))    # combine = concat...mlp
    assert not mh_ok(mh)
    mh = _MH([32, 64], 3)
    mh.infer_list[1] = _MLP(64, extra=(nn.Linear(32, 5),))              # ftype logits
    assert not mh_ok(mh)
    # CPU tensors never take the fused paths
    x = torch.zeros(8, 32)
    o = torch.tensor([8], dtype=torch.int32)
    assert not blocks_fused.transition_up_fusable(_TU(32), [torch.zeros(8, 3), x, o])
    assert not blocks_fused.transition_up_fusable(_TU(64, 32), [torch.zeros(8, 3), x, o], [torch.zeros(2, 3), torch.zeros(2, 64), o])


def _ptxas(src):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    out = os.path.join(tempfile.gettempdir(), f"pt_head_{os.getpid()}.o")
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


def test_pt_head_kernels_do_not_spill_and_match_the_stated_registers():
    """DESIGN §3.7 states these counts; pw_mlp.cu's own kernels are pinned by the PointNet and DGCNN tests and compile to the
    same SASS with the BatchNorm epilogue moved to pw_bn.cuh"""
    seen = _ptxas("pt_head.cu")
    assert all(v["spill"] == (0, 0) for v in seen.values()), seen
    regs = {}
    for name, v in seen.items():
        key = "pt_up_apply" if "pt_up_apply_kernel" in name else "head_classify_" + re.search(r"ILi(\d+)E", name).group(1)
        regs[key] = v["regs"]
    assert regs == {"pt_up_apply": 32, "head_classify_4": 32, "head_classify_8": 32, "head_classify_16": 44,
                    "head_classify_32": 80}, regs
