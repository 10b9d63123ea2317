"""oracle/ref_cuda.py -- the reference's OWN CUDA kernels as a GPU-side checker
(TEST INFRASTRUCTURE ONLY; never imported by toothgroupnetwork_b200/).

``oracle/_ref/libpointops_ref.so`` is built by ``make -C oracle ref`` from the six unmodified
``external_libs/pointops/src/*/*_cuda_kernel.cu`` files where they lie under /root/reference
(compiled for sm_90a; nothing is copied into this repo).  It exports the reference's
``extern "C" *_launcher`` entry points, which take raw device pointers and launch on the legacy
default stream -- so every wrapper below synchronises before and after.
"""
from __future__ import annotations

import ctypes
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
SO = os.path.join(_HERE, "_ref", "libpointops_ref.so")
_lib = None


def available() -> bool:
    return os.path.exists(SO)


def lib():
    global _lib
    if _lib is None:
        _lib = ctypes.CDLL(SO)
    return _lib


def _p(t):
    return ctypes.c_void_p(t.data_ptr())


def _sync():
    torch.cuda.synchronize()


def furthestsampling(xyz, offset, new_offset, n_max, m_total):
    """-> idx (m) int32, tmp (n) float32 (final running minima)."""
    idx = torch.zeros(m_total, dtype=torch.int32, device=xyz.device)
    tmp = torch.full((xyz.shape[0],), 1e10, dtype=torch.float32, device=xyz.device)
    _sync()
    lib().furthestsampling_cuda_launcher(int(offset.shape[0]), int(n_max), _p(xyz), _p(offset), _p(new_offset), _p(tmp), _p(idx))
    _sync()
    return idx, tmp


def knnquery(nsample, xyz, new_xyz, offset, new_offset):
    """-> idx (m,k) int32, dist2 (m,k) float32 (squared)."""
    m = new_xyz.shape[0]
    idx = torch.zeros((m, nsample), dtype=torch.int32, device=xyz.device)
    d2 = torch.zeros((m, nsample), dtype=torch.float32, device=xyz.device)
    _sync()
    lib().knnquery_cuda_launcher(int(m), int(nsample), _p(xyz), _p(new_xyz), _p(offset), _p(new_offset), _p(idx), _p(d2))
    _sync()
    return idx, d2


def grouping_forward(inp, idx):
    m, k = idx.shape
    c = inp.shape[1]
    out = torch.empty((m, k, c), dtype=torch.float32, device=inp.device)
    _sync()
    lib().grouping_forward_cuda_launcher(m, k, c, _p(inp), _p(idx), _p(out))
    _sync()
    return out


def grouping_backward(grad_out, idx, n):
    m, k, c = grad_out.shape
    gi = torch.zeros((n, c), dtype=torch.float32, device=grad_out.device)
    _sync()
    lib().grouping_backward_cuda_launcher(m, k, c, _p(grad_out), _p(idx), _p(gi))
    _sync()
    return gi


def interpolation_forward(inp, idx, weight):
    n, k = idx.shape
    c = inp.shape[1]
    out = torch.zeros((n, c), dtype=torch.float32, device=inp.device)
    _sync()
    lib().interpolation_forward_cuda_launcher(n, c, k, _p(inp), _p(idx), _p(weight), _p(out))
    _sync()
    return out


def interpolation_backward(grad_out, idx, weight, m):
    n, c = grad_out.shape
    gi = torch.zeros((m, c), dtype=torch.float32, device=grad_out.device)
    _sync()
    lib().interpolation_backward_cuda_launcher(n, c, idx.shape[1], _p(grad_out), _p(idx), _p(weight), _p(gi))
    _sync()
    return gi


def subtraction_forward(in1, in2, idx):
    n, c = in1.shape
    k = idx.shape[1]
    out = torch.empty((n, k, c), dtype=torch.float32, device=in1.device)
    _sync()
    lib().subtraction_forward_cuda_launcher(n, k, c, _p(in1), _p(in2), _p(idx), _p(out))
    _sync()
    return out


def subtraction_backward(idx, grad_out):
    n, k, c = grad_out.shape
    g1 = torch.zeros((n, c), dtype=torch.float32, device=grad_out.device)
    g2 = torch.zeros((n, c), dtype=torch.float32, device=grad_out.device)
    _sync()
    lib().subtraction_backward_cuda_launcher(n, k, c, _p(idx), _p(grad_out), _p(g1), _p(g2))
    _sync()
    return g1, g2


def aggregation_forward(inp, pos, weight, idx):
    n, k, c = pos.shape
    out = torch.zeros((n, c), dtype=torch.float32, device=inp.device)
    _sync()
    lib().aggregation_forward_cuda_launcher(n, k, c, weight.shape[-1], _p(inp), _p(pos), _p(weight), _p(idx), _p(out))
    _sync()
    return out


def aggregation_backward(inp, pos, weight, idx, grad_out):
    n, k, c = pos.shape
    gi, gp, gw = torch.zeros_like(inp), torch.zeros_like(pos), torch.zeros_like(weight)
    _sync()
    lib().aggregation_backward_cuda_launcher(n, k, c, weight.shape[-1], _p(inp), _p(pos), _p(weight), _p(idx), _p(grad_out),
                                             _p(gi), _p(gp), _p(gw))
    _sync()
    return gi, gp, gw
