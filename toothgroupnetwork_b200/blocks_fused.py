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

import contextlib
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


def pt_layer_forward(layer, pxo, out_stats: "torch.Tensor | None" = None) -> torch.Tensor:
    """blocks.PointTransformerLayer.forward on csrc/pt_layer.cu: (n,3), (n,c), (b) -> (n,c).  ``out_stats`` (2c float64, zeroed):
    the output pass also adds the batch sums {Σ, Σ²} of each output channel to it (``tgn_pt_layer_forward_sums``)."""
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
    if out_stats is None:
        L.call("tgn_pt_layer_forward", ctypes.byref(d), L.stream_ptr())
    else:
        ds = L.PtLayerSums()
        ds.layer, ds.out_stats = d, L.ptr(out_stats)
        L.call("tgn_pt_layer_forward_sums", ctypes.byref(ds), L.stream_ptr())
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

# True while every offset vector passed to the fused TransitionDown and head-form TransitionUp describes clouds of equal size
# (a network forward on a (B, C, N) batch, where o0 = N, 2N, ..., BN): their host sizes then come from the tensor shapes, and the
# new offsets are made on the device, so no offsets are read back and the forward can be captured into a CUDA graph.
_equal_clouds = False


@contextlib.contextmanager
def equal_clouds():
    global _equal_clouds
    old, _equal_clouds = _equal_clouds, True
    try:
        yield
    finally:
        _equal_clouds = old


def transition_down_forward(td, pxo):
    """blocks.TransitionDown.forward (stride != 1, :59-79): FPS, kNN grouping [xyz_rel | feats], Linear + BatchNorm + ReLU, max over K
    -- a one-layer set abstraction over kNN neighbourhoods -- on the tensor-core layer chain (batch statistics included)."""
    p, x, o = pxo
    if _equal_clouds:
        b, size = o.shape[0], p.shape[0] // o.shape[0]
        sizes, count = [size] * b, b * (size // td.stride)
        n_o = torch.arange(1, b + 1, dtype=torch.int32, device=o.device).mul_(size // td.stride)
    else:
        host_o = o.cpu().tolist()                                # the reference reads o[i].item() here too (:64-67)
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
    ptl._tgn_fused = tdc._tgn_fused = True


# ------------------------------------------------------------------ decoder and heads (blocks.py:82-111, heads.py:13-61)

def _is_lbr(seq, bn: bool) -> bool:
    """seq is exactly Linear [+ BatchNorm1d] + ReLU, float32"""
    kinds = [torch.nn.Linear] + ([torch.nn.BatchNorm1d] if bn else []) + [torch.nn.ReLU]
    if not isinstance(seq, torch.nn.Sequential) or len(seq) != len(kinds) or not all(type(m) is k for m, k in zip(seq, kinds)):
        return False
    return seq[0].weight.dtype == torch.float32 and (not bn or _bn_ok(seq[1]))


def transition_up_structure_ok(tu, head: bool, c_in: int, c_skip: int = 0) -> bool:
    """TransitionUp's layers as blocks.py:84-90 builds them, for inputs of c_in channels (the head form's x, or x2) and c_skip (x1)"""
    lin1, lin2 = tu.linear1, tu.linear2
    if not (_is_lbr(lin1, True) and _is_lbr(lin2, not head)):
        return False
    c = lin1[0].out_features
    if head:
        return lin1[0].in_features == 2 * c_in and c == c_in and lin2[0].in_features == c_in and lin2[0].out_features == c_in
    return lin2[0].in_features == c_in and lin2[0].out_features == c and lin1[0].in_features == c_skip


def _cuda_f32(*ts) -> bool:
    return all(t.is_cuda and t.dtype == torch.float32 and t.dim() == 2 for t in ts)


def transition_up_fusable(tu, pxo1, pxo2=None) -> bool:
    """The fused TransitionUp runs without autograd, on CUDA float32, with the reference's layers; the head form also needs clouds
    of equal size (its per-cloud bias is indexed by row // rows_per_batch), which reads the offsets on the host."""
    if not (_enabled and pn2._pw_enabled):
        return False
    p1, x1, o1 = pxo1
    if pxo2 is None:
        if not _cuda_f32(x1) or _needs_grad(tu, x1) or not transition_up_structure_ok(tu, True, x1.shape[1]):
            return False
        if _equal_clouds:
            return x1.shape[0] % o1.shape[0] == 0
        ends = o1.cpu().tolist()
        return ends[-1] == x1.shape[0] and all(e == (b + 1) * ends[0] for b, e in enumerate(ends))
    p2, x2, o2 = pxo2
    if not (_cuda_f32(x1, x2, p1, p2) and o1.dtype == torch.int32 and o2.dtype == torch.int32):
        return False
    return not _needs_grad(tu, x1, x2) and transition_up_structure_ok(tu, False, x2.shape[1], x1.shape[1])


def _rows_operand(x: torch.Tensor, rows_per_batch: int) -> "L.PwLayer":
    """layer 0 of a chain reading the (rows, c) matrix x through its strides"""
    d = L.PwLayer()
    d.mode, d.rows_per_batch = 0, rows_per_batch
    d.seg_ptr[0], d.seg_channels[0] = L.ptr(x), x.shape[1]
    d.seg_batch_stride[0], d.seg_row_stride[0], d.seg_chan_stride[0] = rows_per_batch * x.stride(0), x.stride(0), x.stride(1)
    return d


_tu_state = weakref.WeakKeyDictionary()           # module -> (its chain, linear1's first c columns)


def transition_up_forward(tu, pxo1, pxo2=None) -> torch.Tensor:
    """blocks.TransitionUp.forward (:92-111) on the layer chain -> (n, c) float32.

    * With pxo2: linear2(x2) is written row-major, linear1(x1) runs on the chain, and its last BatchNorm + ReLU adds the k = 3
      interpolation of linear2(x2) at the positions p1 (``tgn_pt_up_apply``: pointops.interpolation's order, bit for bit given
      the same linear outputs).  The neighbours and weights are what pointops.interpolation computes, from the shared kNN cache.
    * Head form: x = [x | linear2(mean of x over its cloud)] per cloud.  The second half is constant over a cloud, so its product
      with linear1's last c weight columns is one fp64 per-cloud bias (``tgn_pw_cloud_bias``) and the chain only runs linear1's
      first c columns; linear2 runs as the module's own Linear + ReLU on the B cloud means (computed in float64)."""
    st = _tu_state.get(tu)
    if st is None:
        c = tu.linear1[0].out_features
        st = _tu_state[tu] = (pn2._PwChain(), pn2._ColumnSlice(tu.linear1[0], 0, c) if pxo2 is None else None)
    chain, head_cols = st
    lin1, bn1 = tu.linear1[0], tu.linear1[1]
    c = lin1.out_features
    _, x1, o1 = pxo1
    n1 = x1.shape[0]
    out = torch.empty((n1, c), dtype=torch.float32, device=x1.device)
    if pxo2 is None:
        B = o1.shape[0]
        rpb = n1 // B
        g = x1.reshape(B, rpb, c).sum(1, dtype=torch.float64).div_(rpb).float()
        h = tu.linear2(g).contiguous()
        w1 = lin1.weight.detach()
        cloud = torch.empty((B, c), dtype=torch.float32, device=x1.device)
        L.call("tgn_pw_cloud_bias", B, c, c, L.ptr(w1[:, c:]), w1.stride(0), L.ptr(h), h.stride(0), L.ptr(cloud), L.stream_ptr())
        d = _rows_operand(x1, rpb)
        d.cloud_bias = L.ptr(cloud)
        chain.run([head_cols], [bn1], d, n1, out, 0, 1, up=(None, None, None))
        return out
    p1, p2, x2, o2 = pxo1[0].contiguous(), pxo2[0].contiguous(), pxo2[1], pxo2[2]
    f = torch.empty((x2.shape[0], c), dtype=torch.float32, device=x1.device)
    chain.run([tu.linear2[0]], [tu.linear2[1]], _rows_operand(x2, x2.shape[0]), x2.shape[0], f, 0, 1, up=(None, None, None))
    idx, d2 = pointops.knn_packed(3, p2, p1, o2, o1)
    w = pointops._inverse_distance_weights(torch.sqrt(d2)).contiguous()
    chain.run([lin1], [bn1], _rows_operand(x1, n1), n1, out, 0, 1, up=(f, idx, w))
    return out


def multi_head_structure_ok(mh) -> bool:
    """MultiHead as heads.py:14-42 builds it with combine = concat and ftype latent: one Linear + BatchNorm1d + ReLU to 32
    channels per level (at most 8 levels) and one Linear to at most 32 outputs"""
    levels = len(mh.ni_list)
    if not (1 <= levels <= L.HEAD_MAX_LEVELS and len(mh.infer_list) == levels and type(mh.cls) is torch.nn.Linear):
        return False
    if mh.cls.in_features != 32 * levels or not (1 <= mh.cls.out_features <= 32) or mh.cls.weight.dtype != torch.float32:
        return False
    return all(_is_lbr(f.infer, True) and f.infer[0].out_features == 32 for f in mh.infer_list)


def multi_head_fusable(mh, stage_list) -> bool:
    if not (_enabled and pn2._pw_enabled and multi_head_structure_ok(mh)):
        return False
    up0 = stage_list["up"][0]
    n0 = up0["p_out"].shape[0]
    feats = []
    for (n, i), func in zip(mh.ni_list, mh.infer_list):
        st = stage_list[n][i]
        x, p, o = st["f_out"], st["p_out"], st["offset"]
        if not (_cuda_f32(x, p) and o.dtype == torch.int32 and x.shape[1] == func.infer[0].in_features):
            return False
        if i == 0 and x.shape[0] != n0:
            return False
        feats.append(x)
    return _cuda_f32(up0["p_out"]) and up0["offset"].dtype == torch.int32 and not _needs_grad(mh, *feats)


_mh_chains = weakref.WeakKeyDictionary()


def multi_head_forward(mh, stage_list):
    """heads.MultiHead.forward (:53-61) -> (x (n0, k), stage_list).  Each level's Linear + BatchNorm + ReLU runs on the layer chain
    into a (32, n_s) channel-major latent, stored back as stage_list[n][i][ftype] (a (n_s, 32) view of it, as the reference
    stores its output); ``tgn_head_classify`` then gathers every level at the k = 1 neighbours of the level-0 points (the same
    ``pointops.knn_packed`` search pointops.interpolation(k=1) runs, shared between the heads through its cache) and applies
    cls, without the upsampled copies or their concatenation."""
    chain = _mh_chains.get(mh)
    if chain is None:
        chain = _mh_chains[mh] = pn2._PwChain()
    up0 = stage_list["up"][0]
    p0, o0 = up0["p_out"].contiguous(), up0["offset"]
    n0 = p0.shape[0]
    d = L.HeadClassify()
    d.n0, d.k, d.levels = n0, mh.cls.out_features, len(mh.ni_list)
    keep = []
    for s, ((n, i), func) in enumerate(zip(mh.ni_list, mh.infer_list)):
        st = stage_list[n][i]
        x = st["f_out"]
        rows = x.shape[0]
        lat = torch.empty((1, 32, rows), dtype=torch.float32, device=x.device)
        chain.run([func.infer[0]], [func.infer[1]], _rows_operand(x, rows), rows, lat, 0, rows)
        st[mh.ftype] = lat[0].t()
        nn_idx = None
        if i != 0:
            nn_idx, _ = pointops.knn_packed(1, st["p_out"].contiguous(), p0, st["offset"], o0)
        keep += [lat, nn_idx]
        d.lat[s], d.nn[s], d.n[s] = L.ptr(lat), L.ptr(nn_idx), rows
    w = mh.cls.weight.detach().contiguous()
    b = None if mh.cls.bias is None else mh.cls.bias.detach()
    out = torch.empty((n0, d.k), dtype=torch.float32, device=p0.device)
    d.w, d.b, d.out = L.ptr(w), L.ptr(b), L.ptr(out)
    L.call("tgn_head_classify", ctypes.byref(d), L.stream_ptr())
    return out, stage_list


def accelerate_decoder(blocks_module=None, heads_module=None) -> None:
    """Wrap TransitionUp.forward of an imported reference ``blocks`` module and MultiHead.forward of its ``heads`` module (either
    may be None); calls the fused paths do not take, autograd included, run the reference's own code.  Idempotent."""
    if blocks_module is not None and not getattr(blocks_module.TransitionUp, "_tgn_fused", False):
        tuc = blocks_module.TransitionUp
        tu_orig = tuc.forward

        def tu_forward(self, pxo1, pxo2=None):
            if transition_up_fusable(self, pxo1, pxo2):
                return transition_up_forward(self, pxo1, pxo2)
            return tu_orig(self, pxo1, pxo2)

        tuc.forward, tuc._tgn_fused = tu_forward, True
    if heads_module is not None and not getattr(heads_module.MultiHead, "_tgn_fused", False):
        mhc = heads_module.MultiHead
        mh_orig = mhc.forward

        def mh_forward(self, stage_list):
            if multi_head_fusable(self, stage_list):
                return multi_head_forward(self, stage_list)
            return mh_orig(self, stage_list)

        mhc.forward, mhc._tgn_fused = mh_forward, True


# ------------------------------------------------------------------ PointTransformerBlock (blocks.py:114-135)

# The widest block the fused path takes.  Wider blocks (tgnet's first network from 64 channels on) keep the class's previous
# forward: there linear1 / linear3 on the three-part layer chain cost more device time than the module's cuBLAS Linears save in
# launches (scripts/pt_block_bench.py, DESIGN §3.7).  The benchmark sets it to compare the widths.
BLOCK_FUSED_MAX_C = 32


def pt_block_fusable(blk, p, x, o) -> bool:
    """The fused block runs without autograd, on CUDA float32, at widths up to ``BLOCK_FUSED_MAX_C``, with bias-free square
    linear1 / linear3 (as blocks.py:119, :123 build them; the residual needs in_planes == planes), a transformer layer
    ``pt_layer_fusable`` takes and BatchNorms torch's own code would not have to take over (``_bn_ok``)."""
    if not (_enabled and pn2._pw_enabled and _cuda_f32(p, x)):
        return False
    lin1, lin3, c = blk.linear1, blk.linear3, x.shape[1]
    if c > BLOCK_FUSED_MAX_C:
        return False
    if lin1.bias is not None or lin3.bias is not None or lin1.weight.dtype != torch.float32 or lin3.weight.dtype != torch.float32:
        return False
    if tuple(lin1.weight.shape) != (c, c) or tuple(lin3.weight.shape) != (c, c):
        return False
    if not all(type(b) is torch.nn.BatchNorm1d and _bn_ok(b) for b in (blk.bn1, blk.bn2, blk.bn3)):
        return False
    return not _needs_grad(blk, p, x) and pt_layer_fusable(blk.transformer2, p, x, o)


_blk_chains = weakref.WeakKeyDictionary()         # module -> (linear1's chain, linear3's chain)


def pt_block_forward(blk, pxo):
    """blocks.PointTransformerBlock.forward (:127-135) -> [p, (n, c), o], both BatchNorm modes:
    * linear1 on the layer chain reading x row-major, bn1 + ReLU written row-major (``tgn_pt_up_apply`` without an addend);
    * the transformer layer on csrc/pt_layer.cu (the module's own q/k/v Linears), its output pass also forming bn2's batch sums;
    * linear3 on the chain with bn2 + ReLU applied as it reads the layer's output, and ``tgn_pt_res_apply`` for bn3, the residual
      add and the ReLU.  Layers whose BatchNorm uses running statistics run promoted accumulation, as the eval-mode chains do.
    x is only read: the reference's in-place ``+=`` acts on bn3's output."""
    p, x, o = pxo
    n, c = x.shape
    chains = _blk_chains.get(blk)
    if chains is None:
        chains = _blk_chains[blk] = (pn2._PwChain(), pn2._PwChain())
    h = torch.empty((n, c), dtype=torch.float32, device=x.device)
    chains[0].run([blk.linear1], [blk.bn1], _rows_operand(x, n), n, h, 0, 1, up=(None, None, None), promote=True)
    bn2 = blk.bn2
    stats2 = torch.zeros(2 * c, dtype=torch.float64, device=x.device) if pn2._PwChain._bn_mode(bn2) == 1 else None
    y = pt_layer_forward(blk.transformer2, [p, h, o], stats2)
    d = _rows_operand(y, n)
    pn2._PwChain._fill_in_bn(d, bn2, stats2)
    out = torch.empty((n, c), dtype=torch.float32, device=x.device)
    chains[1].run([blk.linear3], [blk.bn3], d, n, out, 0, 1, promote=True, residual=x if x.stride(1) == 1 else x.contiguous())
    if bn2.training and bn2.num_batches_tracked is not None:
        bn2.num_batches_tracked.add_(1)
    return [p, out, o]


def accelerate_blocks(blocks_module) -> None:
    """Wrap PointTransformerBlock.forward of an imported reference ``blocks`` module; calls the fused path does not take,
    autograd included, run the class's previous forward (the reference's, or one whose transformer layer ``accelerate`` wrapped).
    Idempotent."""
    blk = blocks_module.PointTransformerBlock
    if getattr(blk, "_tgn_fused", False):
        return
    blk_orig = blk.forward

    def blk_forward(self, pxo):
        p, x, o = pxo
        if pt_block_fusable(self, p, x, o):
            return pt_block_forward(self, pxo)
        return blk_orig(self, pxo)

    blk.forward, blk._tgn_fused = blk_forward, True
