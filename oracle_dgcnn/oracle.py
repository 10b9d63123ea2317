"""oracle_dgcnn/oracle.py -- Python face of the CPU restatement of DGCNN's feature-space kNN (TEST INFRASTRUCTURE ONLY).

``dgcnn_knn(x, xx, k)`` answers what ``pairwise_distance.topk(k, dim=-1)`` of models/modules/dgcnn.py:4-10 returns on the H100,
through ``dgcnn_knn_oracle.c`` (gcc, -ffp-contract=off).  Nothing under ``toothgroupnetwork_b200/`` may import this module.
"""
from __future__ import annotations

import ctypes
import os
import subprocess
from typing import Tuple

import numpy as np
import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "dgcnn_knn_oracle.c")
_SO = os.path.join(_HERE, "_build", "liboracle_dgcnn.so")
_LIB = None


def build(force: bool = False) -> str:
    """Compile the C restatement with gcc into oracle_dgcnn/_build/ (git-ignored)."""
    if force or not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(_SRC):
        os.makedirs(os.path.dirname(_SO), exist_ok=True)
        subprocess.check_call(["gcc", "-O2", "-ffp-contract=off", "-fopenmp", "-shared", "-fPIC", "-o", _SO + ".tmp", _SRC, "-lm"])
        os.replace(_SO + ".tmp", _SO)
    return _SO


def _lib() -> ctypes.CDLL:
    global _LIB
    if _LIB is None:
        _LIB = ctypes.CDLL(build())
        _LIB.oracle_dgcnn_knn.argtypes = [ctypes.c_int] * 4 + [ctypes.c_void_p] * 4
        _LIB.oracle_dgcnn_knn.restype = None
    return _LIB


def dgcnn_knn(x: torch.Tensor, xx: torch.Tensor, k: int) -> Tuple[np.ndarray, np.ndarray]:
    """x (B, C, N) float32 (any device, any strides), xx (B, 1, N) or (B, N) float32 = torch.sum(x**2, dim=1) as computed for x
    -> (idx (B, N, k) int64, values (B, N, k) float32) in topk's order."""
    xs = np.ascontiguousarray(x.detach().cpu().numpy(), dtype=np.float32)
    B, C, N = xs.shape
    xxs = np.ascontiguousarray(xx.detach().cpu().numpy(), dtype=np.float32).reshape(B, N)
    if not (1 <= k <= 32 and k <= N and 1 <= C):
        raise ValueError(f"dgcnn_knn: need 1 <= k <= min(32, N), got k={k}, N={N}")
    idx = np.empty((B, N, k), np.int64)
    val = np.empty((B, N, k), np.float32)
    _lib().oracle_dgcnn_knn(B, N, C, int(k), xs.ctypes.data, xxs.ctypes.data, idx.ctypes.data, val.ctypes.data)
    return idx, val
