"""CPU: the host side of DGCNN's exact feature-space kNN (toothgroupnetwork_b200.dgcnn) -- the swap and its idempotence, the
routing decision, the refusals that come before any device work, its imports, the C declaration -- the selection of the C
restatement (oracle_dgcnn) against a numpy ordering of its own values, and the code generation of csrc/knn_feat.cu."""
import functools
import os
import re
import shutil
import subprocess
import sys
import tempfile
import types

import numpy as np
import pytest
import torch

from oracle_dgcnn import oracle as O
from toothgroupnetwork_b200 import _lib as L
from toothgroupnetwork_b200 import build, dgcnn, dropin

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_accelerate_swaps_knn_once_and_keeps_the_original_as_the_fallback(monkeypatch):
    def original(x, k):
        return ("reference", k)

    mod = types.SimpleNamespace(knn=original)
    dgcnn.accelerate(mod)
    swapped = mod.knn
    assert isinstance(swapped, functools.partial) and swapped.func is dgcnn.knn and swapped.keywords == {"reference": original}
    dgcnn.accelerate(mod)
    assert mod.knn is swapped
    assert mod.knn(torch.zeros(1, 6, 100), 20) == ("reference", 20)       # a CPU tensor never reaches the kernel
    monkeypatch.setitem(sys.modules, "models.modules.dgcnn", types.SimpleNamespace(knn=original))
    dropin.accelerate_dgcnn()
    assert sys.modules["models.modules.dgcnn"].knn.keywords == {"reference": original}


@pytest.mark.parametrize("B,C,N,permuted", [(1, 6, 24000, True), (1, 64, 24000, False), (2, 6, 4096, True), (2, 64, 4096, False),
                                            (2, 64, 4096, True), (1, 6, 10000, False)])
def test_route_accepts_the_pinned_shapes_and_layouts(B, C, N, permuted):
    strides = (N * C, 1, C) if permuted else (C * N, N, 1)
    assert dgcnn.kernel_route(True, torch.float32, (B, C, N), strides, 20, False)


def test_route_refuses_everything_else():
    ok = dict(is_cuda=True, dtype=torch.float32, shape=(1, 64, 24000), strides=(64 * 24000, 24000, 1), k=20, tf32_matmul=False)
    assert dgcnn.kernel_route(**ok)
    for change in ({"is_cuda": False}, {"dtype": torch.float64}, {"dtype": torch.float16}, {"tf32_matmul": True}, {"k": 33},
                   {"k": 0}, {"shape": (1, 32, 24000), "strides": (32 * 24000, 24000, 1)},
                   {"shape": (1, 64, 4095), "strides": (64 * 4095, 4095, 1)}, {"shape": (1, 64, 24001), "strides": (64 * 24001, 24001, 1)},
                   {"shape": (3, 64, 24000), "strides": (64 * 24000, 24000, 1)}, {"strides": (64 * 24000 * 2, 2 * 24000, 2)},
                   {"strides": (64 * 24000, 1, 128)}, {"shape": (1, 64), "strides": (1, 64)}):
        assert not dgcnn.kernel_route(**{**ok, **change}), change


def test_tf32_setting_is_seen(monkeypatch):
    assert not dgcnn.tf32_matmul()
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", True)
    assert dgcnn.tf32_matmul()
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    monkeypatch.setattr(torch, "get_float32_matmul_precision", lambda: "high")
    assert dgcnn.tf32_matmul()


def test_refusals_before_device_work():
    x = torch.zeros(1, 64, 100)
    with pytest.raises(L.TgnError, match="CUDA"):
        dgcnn.knn_features(x, 20)
    for bad, match in ((x.double(), "float32"), (torch.zeros(1, 65, 100), "C"), (torch.zeros(1, 0, 100), "C"),
                       (torch.zeros(64, 100), r"\(B, C, N\)")):
        with pytest.raises(L.TgnError, match=match):
            dgcnn.knn_features(bad, 20)
    for k in (0, 33, 101):
        with pytest.raises(L.TgnError, match="k"):
            dgcnn.knn_features(torch.zeros(1, 64, 100), k)


def test_dgcnn_imports_neither_the_checkers_nor_the_reference():
    code = ("import sys; import toothgroupnetwork_b200.dgcnn, toothgroupnetwork_b200.dropin; "
            "bad = sorted(m for m in sys.modules if m.split('.')[0] in ('oracle', 'oracle_dgcnn', 'models')); assert not bad, bad")
    res = subprocess.run([sys.executable, "-c", code], cwd=ROOT, capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr


def test_entry_point_is_declared():
    with open(os.path.join(ROOT, "include", "tgn_b200.h")) as f:
        header = " ".join(f.read().split())
    assert ("int tgn_knn_feat(int b, int n, int c, int k, const float *x, long long stride_b, long long stride_c, "
            "long long stride_n, const float *xx, long long *idx, float *val, void *stream);") in header
    assert len(L._SIGS["tgn_knn_feat"]) == 12 and "tgn_knn_feat" in L.EXPORTS
    assert "knn_feat.cu" in build.SOURCES


def _radix_key(v):
    bits = v.view(np.uint32).astype(np.int64)
    key = np.where(bits >= 0x80000000, bits ^ 0xFFFFFFFF, bits ^ 0x80000000)
    return np.where(np.isnan(v), 0xFFFFFFFF, key)


@pytest.mark.parametrize("k", [1, 5, 20, 32])
@pytest.mark.parametrize("name", ["lattice", "duplicates", "zero_vectors"])
def test_oracle_selection_is_the_k_largest_keys_lower_index_first(name, k):
    """small-integer inputs make every product and sum exact, so v is the same in any order and numpy can rank it"""
    g = np.random.default_rng(7)
    if name == "lattice":
        x = g.integers(-3, 4, (2, 16, 300)).astype(np.float32)
    elif name == "duplicates":
        pts = g.integers(-4, 5, (150, 6)).astype(np.float32)
        x = np.concatenate([pts, pts])[g.permutation(300)].T[None].copy()
    else:
        x = g.integers(-2, 3, (1, 6, 300)).astype(np.float32)
        x[:, :, g.permutation(300)[:120]] = 0.0
    xt = torch.from_numpy(x)
    xx = torch.sum(xt ** 2, dim=1, keepdim=True)
    idx, val = O.dgcnn_knn(xt, xx, k)
    x64 = x.astype(np.float64)
    xx64 = (x64 ** 2).sum(1)
    v = (2.0 * np.einsum("bci,bcj->bij", x64, x64) - xx64[:, None, :] - xx64[:, :, None]).astype(np.float32)
    key = _radix_key(v)
    n = v.shape[-1]
    for b in range(v.shape[0]):
        for i in range(n):
            order = np.lexsort((np.arange(n), -key[b, i]))[:k]        # key descending, index ascending
            assert set(idx[b, i].tolist()) == set(order.tolist())
            assert np.array_equal(val[b, i], v[b, i, idx[b, i]])
            assert np.all(np.diff(val[b, i].astype(np.float64)) <= 0)
    if k > 1:
        assert any(len(set(val[b, i].tolist())) < k for b in range(v.shape[0]) for i in range(n))   # ties inside the top k


def test_knn_feat_kernels_do_not_spill():
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    out = os.path.join(tempfile.gettempdir(), f"knn_feat_{os.getpid()}.o")
    cmd = [nvcc] + build.NVCC_FLAGS + ["-Xptxas", "-v", "-c", os.path.join(build.CSRC, "knn_feat.cu"), "-o", out]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if os.path.exists(out):
        os.remove(out)
    assert res.returncode == 0, res.stdout + res.stderr
    current, seen = None, {}
    for line in (res.stdout + res.stderr).splitlines():
        m = re.search(r"Compiling entry function '(\w+)'", line)
        if m:
            current = m.group(1) if "knn_feat_kernel" in m.group(1) else None
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and current:
            seen[current] = (m.group(1), m.group(2))
    assert len(seen) == 2, seen                   # C <= 8 and C <= 64
    assert all(v == ("0", "0") for v in seen.values()), seen
