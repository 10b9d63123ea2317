"""CPU: the host side of the boundary resampling (toothgroupnetwork_b200.boundary) -- the method swap, argument checks that run
before any device work, its imports -- and the code generation of the float64 kNN query kernel (csrc/knn_f64.cu)."""
import os
import re
import shutil
import subprocess
import sys
import types

import numpy as np
import pytest
import torch

from toothgroupnetwork_b200 import _lib as L
from toothgroupnetwork_b200 import boundary, build, clouds, dropin

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _fake_module():
    calls = []

    class InferencePipeLine:
        def __init__(self):
            self.config = {"boundary_sampling_info": {"bdl_ratio": 0.7, "num_of_bdl_points": 20000, "num_of_all_points": 24000}}

        def get_boundary_sampled_feats(self, point_labels, org_feats, sampled_feats, sample_output_features):
            calls.append(sample_output_features)
            return "original"

    return types.SimpleNamespace(InferencePipeLine=InferencePipeLine), calls


def test_accelerate_swaps_the_method_and_keeps_the_original_for_sample_output_features():
    mod, calls = _fake_module()
    dropin.accelerate_inference_pipeline(mod)
    assert mod.InferencePipeLine.get_boundary_sampled_feats is boundary.get_boundary_sampled_feats
    boundary.accelerate(mod)                      # idempotent: the original stays the reference's
    feats = np.zeros((10, 6))
    assert mod.InferencePipeLine().get_boundary_sampled_feats(np.zeros(5), feats, feats, "features") == "original"
    assert calls == ["features"]


def test_without_cuda_the_accelerated_method_raises(monkeypatch):
    mod, calls = _fake_module()
    boundary.accelerate(mod)
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    org, sampled, labels = clouds.boundary_inputs(3000, 1, n_sampled=500)
    with pytest.raises(L.TgnError, match="CUDA"):
        mod.InferencePipeLine().get_boundary_sampled_feats(labels, org, sampled, None)
    assert calls == []


def test_nan_coordinates_and_labels_are_refused():
    mod, _ = _fake_module()
    boundary.accelerate(mod)
    org, sampled, labels = clouds.boundary_inputs(3000, 2, n_sampled=500)
    pipe = mod.InferencePipeLine()
    for which in ("org", "sampled"):
        o, s = org.copy(), sampled.copy()
        (o if which == "org" else s)[7, 1] = np.nan
        with pytest.raises(L.TgnError, match="non-finite"):
            pipe.get_boundary_sampled_feats(labels, o, s, None)
    lab = labels.copy()
    lab[3] = np.nan
    with pytest.raises(L.TgnError, match="NaN labels"):
        pipe.get_boundary_sampled_feats(lab, org, sampled, None)
    with pytest.raises(L.TgnError, match="NaN labels"):
        boundary.label_codes(torch.from_numpy(lab))


def test_knn_arguments_are_checked_before_device_work():
    pts, q = torch.zeros(50, 3, dtype=torch.float64), torch.zeros(10, 3, dtype=torch.float64)
    for k in (0, 51, 65):
        with pytest.raises(L.TgnError, match="k <="):
            boundary.knn_f64(pts, q, k)
    with pytest.raises(L.TgnError, match="float64"):
        boundary.knn_f64(pts.float(), q, 4)
    with pytest.raises(L.TgnError, match="float64"):
        boundary.knn_f64(pts, torch.zeros(10, 2, dtype=torch.float64), 4)
    with pytest.raises(L.TgnError, match="CUDA"):
        boundary.knn_f64(pts, q, 4)                # no CPU path


def test_boundary_imports_neither_the_checker_nor_scikit_learn():
    code = ("import sys; import toothgroupnetwork_b200.boundary; "
            "bad = sorted(m for m in sys.modules if m.split('.')[0] in ('oracle', 'sklearn')); assert not bad, bad")
    res = subprocess.run([sys.executable, "-c", code], cwd=ROOT, capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr


def test_query_kernel_does_not_spill():
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    out = os.path.join(os.environ.get("TMPDIR", "/tmp"), f"knn_f64_{os.getpid()}.o")
    cmd = [nvcc] + build.NVCC_FLAGS + ["-Xptxas", "-v", "-c", os.path.join(build.CSRC, "knn_f64.cu"), "-o", out]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if os.path.exists(out):
        os.remove(out)
    assert res.returncode == 0, res.stdout + res.stderr
    report, current, seen = res.stdout + res.stderr, None, {}
    for line in report.splitlines():
        m = re.search(r"Compiling entry function '(\w+)'", line)
        if m:
            current = m.group(1) if "knn_f64_query_kernel" in m.group(1) else None
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and current:
            seen[current] = (m.group(1), m.group(2))
    assert len(seen) == 2, seen                   # one list entry per lane (k <= 32) and two (k <= 64)
    assert all(v == ("0", "0") for v in seen.values()), seen
