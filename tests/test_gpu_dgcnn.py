"""GPU: the exact feature-space kNN of DGCNN (csrc/knn_feat.cu, toothgroupnetwork_b200.dgcnn) against the reference's expression
evaluated by torch on the same tensor -- values bitwise and indices equal to ``pairwise_distance.topk(k)`` -- at the model's
shapes and layouts and on tie-heavy inputs; against the C restatement (oracle_dgcnn) on other shapes and strides; the reference's
own DGCnnModule forward and backward with and without ``accelerate``; the routing; and the memory the kernel needs."""
import importlib.util
import os

import numpy as np
import pytest
import torch

from oracle import ref_models
from oracle_dgcnn import oracle as O
from toothgroupnetwork_b200 import _lib as L
from toothgroupnetwork_b200 import clouds, dgcnn, dropin

pytestmark = pytest.mark.gpu


def reference_topk(x, k):
    """models/modules/dgcnn.py:4-10 with the values kept"""
    inner = -2 * torch.matmul(x.transpose(2, 1), x)
    xx = torch.sum(x ** 2, dim=1, keepdim=True)
    return (-xx - inner - xx.transpose(2, 1)).topk(k=k, dim=-1)


def features(B, N, C, permuted, seed=0):
    """(B, C, N) cuda float32: [xyz; normal] of arches for C = 6, a seeded LeakyReLU projection of them for larger C; either a
    contiguous tensor or the permute(0, 2, 1) view of a contiguous (B, N, C) one (inference_pipeline_sem.py:30)"""
    f6 = torch.cat([clouds.arch_features(N, seed + b) for b in range(B)])
    if C == 6:
        x = f6
    else:
        g = torch.Generator().manual_seed(seed + 17)
        x = torch.nn.functional.leaky_relu(torch.einsum("oc,bcn->bon", torch.randn(C, 6, generator=g) * 2.0, f6)
                                           + 0.1 * torch.randn(B, C, N, generator=g), 0.2)
    x = x.cuda()
    return x.transpose(1, 2).contiguous().permute(0, 2, 1) if permuted else x.contiguous()


def tie_inputs():
    g = torch.Generator().manual_seed(3)
    dup = clouds.with_duplicates(clouds.dental_arch(2048, 3)[0], 3)                       # (4096, 3), every point twice
    lattice = torch.randint(-3, 4, (1, 64, 4096), generator=g).float()                    # every product exact
    zeros = torch.randn(1, 6, 4096, generator=g)
    zeros[:, :, torch.randperm(4096, generator=g)[:1500]] = 0.0
    negz = zeros.clone()
    negz[:, :, :64] = -0.0
    return {
        "duplicates_C6_permuted": torch.cat([dup, dup], 1).unsqueeze(0).cuda().permute(0, 2, 1),
        "lattice_C64": lattice.cuda(),
        "lattice_C6": lattice[:, :6].contiguous().cuda(),
        "zero_vectors_C6": zeros.cuda(),
        "negative_zero_C6": negz.cuda(),
    }


def assert_same_as_reference(x, k):
    assert dgcnn.kernel_route(True, x.dtype, tuple(x.shape), x.stride(), k, dgcnn.tf32_matmul())
    want_v, want_i = reference_topk(x, k)
    before = L.launch_count()
    got_i, got_v = dgcnn.knn_features(x, k, values=True)
    assert L.launch_count() == before + 1
    assert got_i.dtype == torch.int64 and got_i.shape == want_i.shape
    assert torch.equal(got_v.view(torch.int32), want_v.view(torch.int32)), "values differ"
    bad = int((got_i != want_i).any(-1).sum())
    assert bad == 0, f"{bad} rows with different indices"
    assert torch.equal(dgcnn.knn(x, k), want_i)


@pytest.mark.parametrize("k", [1, 20, 32])
@pytest.mark.parametrize("B,N,C,permuted", [(1, 24000, 6, True), (1, 24000, 64, False), (2, 4096, 6, True), (2, 4096, 6, False),
                                            (2, 4096, 64, False), (2, 4096, 64, True)])
def test_model_shapes_match_topk(B, N, C, permuted, k):
    assert_same_as_reference(features(B, N, C, permuted), k)


@pytest.mark.parametrize("k", [1, 20, 32])
@pytest.mark.parametrize("name", ["duplicates_C6_permuted", "lattice_C64", "lattice_C6", "zero_vectors_C6", "negative_zero_C6"])
def test_ties_match_topk(name, k):
    assert_same_as_reference(tie_inputs()[name], k)


@pytest.mark.parametrize("B,N,C,k,view", [(1, 2000, 64, 20, "contiguous"), (2, 1500, 6, 32, "permuted"), (1, 1000, 17, 5, "strided"),
                                          (2, 700, 3, 1, "strided"), (1, 40, 64, 32, "contiguous"), (1, 4096, 64, 20, "lattice")])
def test_kernel_matches_oracle(B, N, C, k, view):
    if view == "lattice":
        x = torch.randint(-2, 3, (B, C, N), generator=torch.Generator().manual_seed(5)).float().cuda()
    elif view == "strided":                       # every other channel and every other point of a larger tensor
        x = features(B, 2 * N, 2 * C, False, seed=2)[:, ::2, ::2]
    else:
        x = features(B, N, C, view == "permuted", seed=1)
    got_i, got_v = dgcnn.knn_features(x, k, values=True)
    want_i, want_v = O.dgcnn_knn(x, torch.sum(x ** 2, dim=1, keepdim=True), k)
    assert np.array_equal(got_v.cpu().numpy().view(np.int32), want_v.view(np.int32))
    assert np.array_equal(got_i.cpu().numpy(), want_i)


def test_routing_sends_unpinned_inputs_to_the_reference():
    calls = []

    def reference(x, k):
        calls.append((tuple(x.shape), k))
        return dgcnn.reference_knn(x, k)

    x = features(1, 4096, 64, False)
    before = L.launch_count()
    dgcnn.knn(x, 40, reference=reference)                                   # k > 32
    dgcnn.knn(x[:, :32].contiguous(), 20, reference=reference)              # C not pinned
    dgcnn.knn(features(1, 1000, 6, True), 20, reference=reference)           # N not pinned
    dgcnn.knn(x.double(), 20, reference=reference)                           # not float32
    try:
        torch.backends.cuda.matmul.allow_tf32 = True
        dgcnn.knn(x, 20, reference=reference)                                # TF32 matmuls round differently
    finally:
        torch.backends.cuda.matmul.allow_tf32 = False
    assert L.launch_count() == before and len(calls) == 5
    dgcnn.knn(x, 20, reference=reference)
    assert L.launch_count() == before + 1 and len(calls) == 5


def test_kernel_memory_is_o_of_n_k():
    x = features(1, 24000, 64, False)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    idx = dgcnn.knn_features(x, 20)
    torch.cuda.synchronize()
    grew = torch.cuda.max_memory_allocated() - base
    assert grew < 64 << 20, grew
    assert idx.shape == (1, 24000, 20)


def _reference_dgcnn_module(root, name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(root, "models", "modules", "dgcnn.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.mark.skipif(not ref_models.available(), reason="reference snapshot not staged")
def test_reference_dgcnn_forward_and_backward_bitwise_unchanged():
    root = ref_models.reference_root()
    ref_mod, new_mod = _reference_dgcnn_module(root, "ref_dgcnn_a"), _reference_dgcnn_module(root, "ref_dgcnn_b")
    dropin.accelerate_dgcnn(new_mod)
    dropin.accelerate_dgcnn(new_mod)                                        # idempotent
    assert new_mod.knn.func is dgcnn.knn and new_mod.knn.keywords["reference"] is not dgcnn.knn
    feats = clouds.arch_features(24000).cuda()                              # (1, 6, N)
    x = feats.transpose(1, 2).contiguous().permute(0, 2, 1)                  # the sem pipeline's layout
    labels = torch.randint(0, 17, (1, 24000), generator=torch.Generator().manual_seed(9)).cuda()
    saved = torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False
    torch.use_deterministic_algorithms(True, warn_only=True)
    try:
        results = []
        for mod in (ref_mod, new_mod):
            torch.manual_seed(0)
            model = mod.DGCnnModule(None).cuda().train()
            before = L.launch_count()
            torch.manual_seed(1)
            pred = model([x])["cls_pred"]
            loss = torch.nn.functional.cross_entropy(pred, labels)
            loss.backward()
            torch.cuda.synchronize()
            results.append((pred.detach(), loss.detach(), [p.grad.clone() for p in model.parameters() if p.grad is not None], L.launch_count() - before))
    finally:
        torch.use_deterministic_algorithms(False)
        torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = saved
    (p0, l0, g0, n0), (p1, l1, g1, n1) = results
    assert n0 == 0 and n1 == 3                                               # the three kNN calls ran on the kernel
    assert torch.equal(p0.view(torch.int32), p1.view(torch.int32)), "cls_pred differs"
    assert torch.equal(l0.view(torch.int32), l1.view(torch.int32))
    assert len(g0) == len(g1) and all(torch.equal(a.view(torch.int32), b.view(torch.int32)) for a, b in zip(g0, g1))
