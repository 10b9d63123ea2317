"""Exact feature-space kNN of the DGCNN model on the GPU without the N x N distance matrix (DESIGN §3.11).

``DGCnnModule.forward`` calls ``get_graph_feature`` three times per forward (models/modules/dgcnn.py:102,107,112), and each call
runs ``knn`` (:4-10): the full (B, N, N) matrix ``-xx - inner - xx^T`` from a cuBLAS matmul, then ``topk``.  At N = 24 000 that
matrix is 2.3 GB, and about 6.9 GB is alive at the peak of the expression.  csrc/knn_feat.cu computes the same values pair by pair
in registers, in the order cuBLAS and the two element-wise subtractions round them, and keeps only each row's k best, so its
indices and values are those of ``topk`` bit for bit.

* ``knn_features(x, k, values=False)`` -- the device API: (B, C, N) float32 CUDA, any strides, C <= 64, k <= 32.
* ``knn(x, k)`` -- the drop-in with the reference's signature and return value.  It runs the kernel only where the kernel's
  arithmetic was pinned against cuBLAS on the H100 (``kernel_route``); everything else goes to the reference's own function.
* ``accelerate(module)`` -- points ``module.knn`` (looked up by ``get_graph_feature`` at call time) at the drop-in.

``get_graph_feature``, the convolutions and BatchNorm stay the reference's.  The indices carry no gradient, so autograd and
training see the same graph.
"""
from __future__ import annotations

import functools
import operator
from typing import Sequence

import torch

from . import _lib as L

MAX_C = 64
MAX_K = 32
# the shapes and layouts for which scripts/diag_dgcnn_knn.py found cuBLAS's FP32 dot products equal to the kernel's in-order FFMA
# chain over every pair (DESIGN §3.11): DGCNN's channel counts, batch 1 and 2, 4 096 to 24 000 points
PINNED_C = (6, 64)
PINNED_B = (1, 2)
PINNED_N = (4096, 24000)


def knn_features(x: torch.Tensor, k: int, values: bool = False):
    """x (B, C, N) float32 CUDA, read in place through its strides -> idx (B, N, k) int64 [, values (B, N, k) float32]: the
    indices and values of ``pairwise_distance.topk(k, dim=-1)`` of models/modules/dgcnn.py:4-10 (largest first), on the current
    stream.  1 <= C <= 64, 1 <= k <= min(32, N).  A NaN value is returned as the canonical NaN."""
    k = operator.index(k)
    if not torch.is_tensor(x) or x.dim() != 3:
        raise L.TgnError(f"knn_features: x must be a (B, C, N) tensor, got {tuple(x.shape) if torch.is_tensor(x) else type(x)}")
    if x.dtype != torch.float32:
        raise L.TgnError(f"knn_features: x must be float32, got {x.dtype}")
    B, C, N = x.shape
    if not 1 <= C <= MAX_C:
        raise L.TgnError(f"knn_features: need 1 <= C <= {MAX_C}, got C={C}")
    if not 1 <= k <= min(MAX_K, N):
        raise L.TgnError(f"knn_features: need 1 <= k <= min({MAX_K}, N), got k={k} with N={N}")
    L.require_cuda(x)
    with torch.no_grad():
        xx = torch.sum(x ** 2, dim=1, keepdim=True)     # the reference's own expression on the same tensor: the same bits
    idx = torch.empty((B, N, k), dtype=torch.int64, device=x.device)
    val = torch.empty((B, N, k), dtype=torch.float32, device=x.device) if values else None
    L.call("tgn_knn_feat", B, N, C, k, L.ptr(x), x.stride(0), x.stride(1), x.stride(2), L.ptr(xx.contiguous()), L.ptr(idx),
           L.ptr(val), L.stream_ptr())
    return (idx, val) if values else idx


def kernel_route(is_cuda: bool, dtype: torch.dtype, shape: Sequence[int], strides: Sequence[int], k: int,
                 tf32_matmul: bool) -> bool:
    """True when the kernel's answer is the reference's: a CUDA float32 (B, C, N) tensor in one of the two layouts DGCNN passes
    (a contiguous (B, C, N) tensor, or the permute(0, 2, 1) view of a contiguous (B, N, C) one), a pinned shape, k <= 32, and
    FP32 matmuls without TF32 (with TF32 cuBLAS rounds the products differently)."""
    if not is_cuda or dtype != torch.float32 or len(shape) != 3 or tf32_matmul:
        return False
    B, C, N = shape
    if C not in PINNED_C or B not in PINNED_B or not PINNED_N[0] <= N <= PINNED_N[1] or not 1 <= k <= min(MAX_K, N):
        return False
    # (channel, point) strides of the two layouts; both put the clouds C * N apart (a single cloud's batch stride is free)
    return tuple(strides[1:]) in ((N, 1), (1, C)) and (B == 1 or strides[0] == C * N)


def tf32_matmul() -> bool:
    return bool(torch.backends.cuda.matmul.allow_tf32) or torch.get_float32_matmul_precision() != "highest"


def reference_knn(x: torch.Tensor, k: int) -> torch.Tensor:
    """The reference's kNN (models/modules/dgcnn.py:4-10) as torch evaluates it: the answer for inputs outside the kernel's route
    when ``knn`` is called without the reference's own function."""
    inner = -2 * torch.matmul(x.transpose(2, 1), x)
    xx = torch.sum(x ** 2, dim=1, keepdim=True)
    return (-xx - inner - xx.transpose(2, 1)).topk(k=k, dim=-1)[1]


def knn(x: torch.Tensor, k: int, reference=reference_knn) -> torch.Tensor:
    """Drop-in for ``knn(x, k)`` of models/modules/dgcnn.py: (B, N, k) int64 indices, equal to the reference's.  Inputs outside
    ``kernel_route`` are answered by ``reference``."""
    if torch.is_tensor(x) and kernel_route(x.is_cuda, x.dtype, tuple(x.shape), x.stride(), k, tf32_matmul()):
        return knn_features(x, k)
    return reference(x, k)


def accelerate(module) -> None:
    """Point ``module.knn`` (models/modules/dgcnn.py) at the drop-in, which answers unsupported inputs with the module's own
    ``knn``.  Calling it again leaves the module as it is."""
    current = module.knn
    if isinstance(current, functools.partial) and current.func is knn:
        return
    module.knn = functools.partial(knn, reference=current)
