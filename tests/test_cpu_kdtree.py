"""CPU: the host side of the KDTree drop-in of the label transfers (toothgroupnetwork_b200.neighbors) -- the name swaps, the
refusals that come before any device work, its imports, the C declarations of the build / query split -- and the code generation
of the tie-flag query kernel (csrc/knn_f64.cu)."""
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
from toothgroupnetwork_b200 import build, dropin, neighbors

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TGN = "inference_pipelines.inference_pipeline_tgn"
OTHERS = ("inference_pipelines.inference_pipeline_tsegnet", "inference_pipelines.inference_pipeline_sem")


def test_accelerate_label_transfer_swaps_kdtree_in_the_pipelines(monkeypatch):
    sk = object()                                 # stands for sklearn.neighbors.KDTree
    tgn = types.SimpleNamespace(KDTree=sk)
    others = {name: types.SimpleNamespace(KDTree=sk) for name in OTHERS}
    ops_utils = types.SimpleNamespace(KDTree=sk)
    for name, mod in others.items():
        monkeypatch.setitem(sys.modules, name, mod)
    monkeypatch.setitem(sys.modules, "ops_utils", ops_utils)
    dropin.accelerate_label_transfer(tgn)
    assert tgn.KDTree is neighbors.KDTree
    assert all(m.KDTree is neighbors.KDTree for m in others.values())
    assert ops_utils.KDTree is sk                 # its k = 10 vote and k = 3072 crops are accelerate_ops_utils' business


def test_accelerate_label_transfer_imports_tgn_and_leaves_absent_pipelines_alone(monkeypatch):
    tgn = types.ModuleType(TGN)
    tgn.KDTree = object()
    monkeypatch.setitem(sys.modules, TGN, tgn)    # what importlib.import_module returns
    for name in OTHERS:
        monkeypatch.delitem(sys.modules, name, raising=False)
    dropin.accelerate_label_transfer()
    assert tgn.KDTree is neighbors.KDTree
    assert not any(name in sys.modules for name in OTHERS)
    bare = types.SimpleNamespace()
    neighbors.accelerate(bare)                    # a module without the name is left without it
    assert not hasattr(bare, "KDTree")


def test_without_cuda_the_tree_is_refused(monkeypatch):
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    with pytest.raises(L.TgnError, match="CUDA"):
        neighbors.KDTree(np.random.default_rng(0).random((100, 3)), leaf_size=2)


def test_constructor_refusals_before_device_work():
    pts = np.random.default_rng(1).random((50, 3))
    for kwargs in ({"metric": "euclidean"}, {"metric": "manhattan"}, {"p": 1}):
        with pytest.raises(L.TgnError, match="metric"):
            neighbors.KDTree(pts, **kwargs)
    with pytest.raises(L.TgnError, match=r"\(n, 3\)"):
        neighbors.KDTree(np.zeros((50, 2)))
    bad = pts.copy()
    bad[4, 2] = np.nan
    with pytest.raises(ValueError):               # scikit-learn's type for NaN, inf, not 2-D, empty, leaf_size < 1
        neighbors.KDTree(bad)
    bad[4, 2] = np.inf
    for X in (bad, np.zeros(3), np.zeros((0, 3))):
        with pytest.raises(ValueError):
            neighbors.KDTree(X)
    with pytest.raises(ValueError):
        neighbors.KDTree(pts, leaf_size=0)


def test_neighbors_imports_neither_the_checker_nor_scikit_learn():
    code = ("import sys; import toothgroupnetwork_b200.neighbors, toothgroupnetwork_b200.dropin; "
            "bad = sorted(m for m in sys.modules if m.split('.')[0] in ('oracle', 'sklearn')); assert not bad, bad")
    res = subprocess.run([sys.executable, "-c", code], cwd=ROOT, capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr


def test_build_and_query_are_declared():
    with open(os.path.join(ROOT, "include", "tgn_b200.h")) as f:
        header = " ".join(f.read().split())
    assert "int tgn_knn_f64_build(int n, const double *xyz, void *workspace, void *stream);" in header
    assert ("int tgn_knn_f64_query(int n, int m, int k, const double *xyz, const double *queries, const void *workspace, "
            "const int *labels, long long *idx, double *dist, int *nn0, int *agree, unsigned char *tie, void *stream);") in header
    assert len(L._SIGS["tgn_knn_f64_build"]) == 4 and len(L._SIGS["tgn_knn_f64_query"]) == 13
    assert {"tgn_knn_f64_build", "tgn_knn_f64_query"} <= set(L.EXPORTS)


def test_tie_query_kernel_does_not_spill():
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    out = os.path.join(os.environ.get("TMPDIR", "/tmp"), f"knn_f64_tie_{os.getpid()}.o")
    cmd = [nvcc] + build.NVCC_FLAGS + ["-Xptxas", "-v", "-c", os.path.join(build.CSRC, "knn_f64.cu"), "-o", out]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if os.path.exists(out):
        os.remove(out)
    assert res.returncode == 0, res.stdout + res.stderr
    current, seen = None, {}
    for line in (res.stdout + res.stderr).splitlines():
        m = re.search(r"Compiling entry function '(\w+)'", line)
        if m:
            current = m.group(1) if "knn_f64_tie_query_kernel" in m.group(1) else None
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and current:
            seen[current] = (m.group(1), m.group(2))
    assert len(seen) == 2, seen                   # k + 1 <= 32 entries (one per lane) and k + 1 <= 64 (two per lane)
    assert all(v == ("0", "0") for v in seen.values()), seen
