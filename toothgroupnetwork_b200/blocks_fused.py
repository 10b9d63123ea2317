"""Fused forwards for the reference's ``models/modules/cbl_point_transformer/blocks.py`` (SURVEY.md 8(f)-3).

``accelerate(blocks_module)`` wraps ``PointTransformerLayer.forward`` (:31-44) and ``TransitionDown.forward`` (:59-79) of an
imported reference ``blocks`` module: when no gradient is needed (the reference's inference and validation run under
``torch.no_grad()``) and the shape is one the kernels take, the layer runs on ``csrc/pt_layer.cu`` / the tensor-core layer chain of
``csrc/pw_mlp.cu``; otherwise the reference's own code runs, untouched.  Parameters, buffers and ``state_dict`` keys are the
reference's; BatchNorm keeps torch's semantics (batch statistics in ``train()``, which the reference's inference leaves on,
running statistics updated with the module's momentum, ``num_batches_tracked`` incremented).

What is saved per transformer layer: two identical kNN searches (one, cached), two grouped (n, K, c) tensors, ~30 torch kernels
of which three are cuDNN BatchNorms over (n, c, K) views -- the largest share of the kernel time of a tgnet_fps step.
"""
from __future__ import annotations

import ctypes
import weakref

import torch

from . import _lib as L
from . import pointnet2_utils as pn2
from . import pointops

_SUPPORTED_C = (16, 32, 64, 128, 256, 512)
_enabled = True


def set_enabled(flag: bool) -> None:
    global _enabled
    _enabled = bool(flag)


def _needs_grad(module, *tensors) -> bool:
    if not torch.is_grad_enabled():
        return False
    return any(t is not None and t.requires_grad for t in tensors) or any(q.requires_grad for q in module.parameters())


def _bn_ok(bn) -> bool:
    return bn.weight is not None and bn.weight.dtype == torch.float32 and not (bn.training and bn.track_running_stats and bn.momentum is None)


def _bn_mode(bn) -> int:
    return 1 if (bn.training or bn.running_mean is None) else 2


def pt_layer_fusable(layer, p, x, o) -> bool:
    if not (_enabled and p.is_cuda and x.is_cuda and p.dtype == torch.float32 and x.dtype == torch.float32):
        return False
    if _needs_grad(layer, p, x):
        return False
    c = layer.out_planes
    if c not in _SUPPORTED_C or layer.mid_planes != c or layer.share_planes != 8 or not (1 <= layer.nsample <= 64):
        return False
    if layer.linear_q.in_features != x.shape[1]:
        return False
    return all(_bn_ok(b) for b in (layer.linear_p[1], layer.linear_w[0], layer.linear_w[3]))


def pt_layer_forward(layer, pxo) -> torch.Tensor:
    """blocks.PointTransformerLayer.forward on csrc/pt_layer.cu: (n,3), (n,c), (b) -> (n,c)."""
    p, x, o = pxo
    x_q, x_k, x_v = layer.linear_q(x), layer.linear_k(x), layer.linear_v(x)         # the model's own nn.Linear GEMMs
    p = p.contiguous()
    idx, _ = pointops.knn_packed(int(layer.nsample), p, p, o, o)                     # one search (the reference does two, :34-35)
    n, c = x_v.shape
    K, cs = idx.shape[1], c // 8
    lin_p0, bn_p, lin_p1 = layer.linear_p[0], layer.linear_p[1], layer.linear_p[3]
    bn_a, lin_a, bn_b, lin_b = layer.linear_w[0], layer.linear_w[2], layer.linear_w[3], layer.linear_w[5]
    stats = torch.zeros(6 + 2 * c + 2 * cs, dtype=torch.float64, device=x.device)
    out = torch.empty((n, c), dtype=torch.float32, device=x.device)
    keep = [x_q.contiguous(), x_k.contiguous(), x_v.contiguous()]
    d = L.PtLayer()
    d.n, d.c, d.K = n, c, K
    d.p, d.xq, d.xk, d.xv, d.idx, d.out = L.ptr(p), L.ptr(keep[0]), L.ptr(keep[1]), L.ptr(keep[2]), L.ptr(idx), L.ptr(out)
    d.p_w0, d.p_b0, d.p_w1, d.p_b1 = L.ptr(lin_p0.weight), L.ptr(lin_p0.bias), L.ptr(lin_p1.weight), L.ptr(lin_p1.bias)
    d.a_w, d.a_b, d.b_w, d.b_b = L.ptr(lin_a.weight), L.ptr(lin_a.bias), L.ptr(lin_b.weight), L.ptr(lin_b.bias)
    for tag, bn in (("p", bn_p), ("a", bn_a), ("b", bn_b)):
        setattr(d, tag + "_gamma", L.ptr(bn.weight))
        setattr(d, tag + "_beta", L.ptr(bn.bias))
        setattr(d, tag + "_rmean", L.ptr(bn.running_mean))
        setattr(d, tag + "_rvar", L.ptr(bn.running_var))
        setattr(d, tag + "_eps", float(bn.eps))
        setattr(d, tag + "_momentum", float(bn.momentum if bn.momentum is not None else 0.0))
    d.stats_p = stats.data_ptr()
    d.stats_a = stats.data_ptr() + 6 * 8
    d.stats_b = stats.data_ptr() + (6 + 2 * c) * 8
    modes = [_bn_mode(b) for b in (bn_p, bn_a, bn_b)]
    d.bn_mode[0], d.bn_mode[1], d.bn_mode[2] = modes
    d.update_running = 1 if any(m == 1 and b.training and b.running_mean is not None for m, b in zip(modes, (bn_p, bn_a, bn_b))) else 0
    L.call("tgn_pt_layer_forward", ctypes.byref(d), L.stream_ptr())
    for b in (bn_p, bn_a, bn_b):
        if b.training and b.num_batches_tracked is not None:
            b.num_batches_tracked.add_(1)
    return out


def transition_down_fusable(td, p, x, o) -> bool:
    if not (_enabled and td.stride != 1 and p.is_cuda and x.is_cuda and p.dtype == torch.float32 and x.dtype == torch.float32):
        return False
    if _needs_grad(td, p, x):
        return False
    if td.linear.in_features != 3 + x.shape[1] or td.linear.weight.dtype != torch.float32:
        return False
    return _bn_ok(td.bn) and td.linear.bias is None and pn2._pw_enabled


_td_chains = weakref.WeakKeyDictionary()          # module -> its packed-weight chain; entries go with the module


def transition_down_forward(td, pxo):
    """blocks.TransitionDown.forward (stride != 1, :59-79): FPS, kNN grouping [xyz_rel | feats], Linear + BatchNorm + ReLU, max over K
    -- a one-layer set abstraction over kNN neighbourhoods -- on the tensor-core layer chain (batch statistics included)."""
    p, x, o = pxo
    host_o = o.cpu().tolist()                                    # the reference reads o[i].item() here too (:64-67)
    n_o, count, prev = [], 0, 0
    for e in host_o:
        count += (e - prev) // td.stride
        n_o.append(count)
        prev = e
    n_o = torch.tensor(n_o, dtype=torch.int32, device=o.device)
    sizes = [host_o[0]] + [host_o[i] - host_o[i - 1] for i in range(1, len(host_o))]
    p = p.contiguous()
    idx = pointops.fps_packed(p, o, n_o, max(sizes), count)
    n_p = p[idx.long(), :]
    gidx, _ = pointops.knn_packed(int(td.nsample), p, n_p, o, n_o)              # (m, K) global row ids
    m, K = gidx.shape
    chain = _td_chains.get(td)
    if chain is None:
        chain = _td_chains[td] = pn2._PwChain()
    out = torch.empty((1, td.linear.out_features, m), dtype=torch.float32, device=x.device)
    pn2._pw_set_abstraction(chain, [td.linear], [td.bn], p.view(1, -1, 3), x.contiguous().view(1, x.shape[0], -1), n_p.view(1, m, 3),
                            gidx.view(1, m, K), True, out, 0)
    return [n_p, pn2.transpose_last2(out)[0], n_o]


def accelerate(blocks_module) -> None:
    """Wrap PointTransformerLayer.forward and TransitionDown.forward of an imported reference ``blocks`` module."""
    ptl, tdc = blocks_module.PointTransformerLayer, blocks_module.TransitionDown
    if getattr(ptl, "_tgn_fused", False):
        return
    ptl_orig, td_orig = ptl.forward, tdc.forward

    def ptl_forward(self, pxo):
        p, x, o = pxo
        if pt_layer_fusable(self, p, x, o):
            return pt_layer_forward(self, pxo)
        return ptl_orig(self, pxo)

    def td_forward(self, pxo):
        p, x, o = pxo
        if transition_down_fusable(self, p, x, o):
            return transition_down_forward(self, pxo)
        return td_orig(self, pxo)

    ptl.forward, tdc.forward = ptl_forward, td_forward
    ptl._tgn_fused = True
