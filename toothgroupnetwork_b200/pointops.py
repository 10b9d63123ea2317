"""Operator API of ``external_libs/pointops/functions/pointops.py`` on libtgn_b200.so.

Same public names, positional signatures, dtypes and layouts as the reference (packed
``(n_total, C)`` tensors with cumulative int32 ``offset``; see SURVEY.md 8b), so the callers in
``models/modules/cbl_point_transformer/{blocks,heads,basic_operators}.py`` and ``gen_utils.fps``
run unchanged.  Every op launches hand-written sm_90a kernels on the current stream; there is
no CPU path.  Reference line numbers below refer to that file.
"""
from __future__ import annotations

from typing import Optional, Tuple

import torch
from torch.autograd import Function

from . import _lib as L

_RESIDENT_FPS_MAX_POINTS = 8 * 12288   # largest cloud the register-resident FPS clusters hold


def _empty(shape, dtype, like: torch.Tensor) -> torch.Tensor:
    return torch.empty(shape, dtype=dtype, device=like.device)


def _need(t: torch.Tensor, dtype, what: str) -> None:
    if not t.is_cuda:
        raise L.TgnError(f"{what}: CUDA tensor required (no CPU path)")
    if t.dtype != dtype:
        raise L.TgnError(f"{what}: expected {dtype}, got {t.dtype}")
    assert t.is_contiguous(), f"{what} must be contiguous"   # the reference asserts the same (:17,:38,...)


def fps_packed(xyz: torch.Tensor, offset: torch.Tensor, new_offset: torch.Tensor, n_max: int, m_total: int,
               mode: int = 0) -> torch.Tensor:
    """FPS with the host-side sizes already known (no device->host sync).  ``mode``: 0 auto,
    -1 the streaming kernel, otherwise 100*G + CS forces a cluster of CS CTAs with G clouds in
    flight (G omitted = 1), e.g. 8 or 204."""
    _need(xyz, torch.float32, "xyz")
    _need(offset, torch.int32, "offset")
    _need(new_offset, torch.int32, "new_offset")
    idx = torch.zeros((m_total,), dtype=torch.int32, device=xyz.device)   # zero-filled like the reference (:21)
    if m_total == 0:
        return idx
    tmp = None
    if mode == -1 or n_max > _RESIDENT_FPS_MAX_POINTS:
        tmp = torch.full((xyz.shape[0],), 1e10, dtype=torch.float32, device=xyz.device)   # :22
    L.call("tgn_furthestsampling", int(offset.shape[0]), int(n_max), L.ptr(xyz), L.ptr(offset), L.ptr(new_offset),
           L.ptr(tmp), L.ptr(idx), int(mode), L.stream_ptr())
    return idx


def _offset_sizes(offset: torch.Tensor, new_offset: torch.Tensor, n_total: int) -> Tuple[int, int]:
    """(largest segment, total samples) of an (offset, new_offset) pair: ONE host copy of both vectors, where the
    reference reads them back with one blocking ``.item()`` per cloud (:18-21).  The output size is data, so one
    read-back is the floor for this signature; its callers (``blocks.py:64-69``) have just synchronised on
    ``o[i].item()`` themselves.  Callers that know the sizes use ``fps_packed`` directly and never synchronise."""
    host = torch.stack([offset.to(torch.int64), new_offset.to(torch.int64)]).cpu()
    n_max = int(torch.diff(host[0], prepend=host[0].new_zeros(1)).max())
    return n_max, int(host[1][-1])


class FurthestSampling(Function):
    """:10-27.  input: xyz (n,3), offset (b), new_offset (b); output: idx (m) int32 global row ids."""

    @staticmethod
    def forward(ctx, xyz, offset, new_offset):
        if offset.shape[0] == 0:
            return _empty((0,), torch.int32, xyz)
        n_max, m_total = _offset_sizes(offset, new_offset, xyz.shape[0])
        idx = fps_packed(xyz, offset, new_offset, n_max, m_total)
        ctx.mark_non_differentiable(idx)
        return idx


furthestsampling = FurthestSampling.apply


KNN_GRID_MIN_POINTS = 2048      # below this a brute-force scan of the segment is as fast as building a grid
_knn_grid_enabled = True


def set_knn_grid(flag: bool) -> None:
    """Experiments / tests: False keeps every kNN on the brute-force warp kernel (csrc/knn.cu)."""
    global _knn_grid_enabled
    _knn_grid_enabled = bool(flag)


class _Lru:
    """Tiny LRU keyed by tensor identity: an entry keeps its key tensors alive, so a (data_ptr, _version) pair cannot be
    recycled for different contents while the entry exists; an in-place change bumps ``_version`` and misses."""

    def __init__(self, size: int):
        self.size, self.items = size, []

    @staticmethod
    def sig(*tensors) -> tuple:
        return tuple((t.data_ptr(), t._version, tuple(t.shape)) for t in tensors)

    def get(self, key):
        for i, (k, _, val) in enumerate(self.items):
            if k == key:
                self.items.append(self.items.pop(i))
                return val
        return None

    def put(self, key, keep_alive, val) -> None:
        self.items.append((key, keep_alive, val))
        if len(self.items) > self.size:
            self.items.pop(0)

    def clear(self) -> None:
        self.items.clear()


_grid_cache = _Lru(8)       # (xyz, offset) -> grid workspace
_knn_cache = _Lru(16)       # (xyz, new_xyz, offset, new_offset, k) -> (idx, d2): a PointTransformerLayer asks twice (blocks.py:34-35)


def clear_knn_caches() -> None:
    _grid_cache.clear()
    _knn_cache.clear()


def _grid_for(xyz: torch.Tensor, offset: torch.Tensor) -> torch.Tensor:
    key = _Lru.sig(xyz, offset)
    cur = torch.cuda.current_stream()
    hit = _grid_cache.get(key)
    if hit is not None:
        ws, ev, stream = hit
        if stream != cur:                      # built on another stream: order this consumer after the build
            cur.wait_event(ev)
            ws.record_stream(cur)
        return ws
    b, n = int(offset.shape[0]), int(xyz.shape[0])
    ws = torch.empty(L.load().tgn_knn_grid_bytes(b, n), dtype=torch.uint8, device=xyz.device)
    L.call("tgn_knn_grid_build", b, n, L.ptr(xyz), L.ptr(offset), L.ptr(ws), L.stream_ptr())
    ev = torch.cuda.Event()
    ev.record(cur)
    _grid_cache.put(key, (xyz, offset), (ws, ev, cur))
    return ws


def knn_packed(nsample: int, xyz: torch.Tensor, new_xyz: torch.Tensor, offset: torch.Tensor,
               new_offset: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """idx (m,nsample) int32 and SQUARED distances (m,nsample).  Point sets of >= KNN_GRID_MIN_POINTS rows are searched
    through a uniform grid that is built once per (xyz, offset) and cached; identical repeated queries (the two
    ``queryandgroup`` calls of a transformer layer, every layer of a level) return the cached answer.  The cached
    tensors are shared: treat them as read-only (an in-place write invalidates the entry)."""
    _need(xyz, torch.float32, "xyz")
    _need(new_xyz, torch.float32, "new_xyz")
    _need(offset, torch.int32, "offset")
    _need(new_offset, torch.int32, "new_offset")
    m = new_xyz.shape[0]
    n, b = int(xyz.shape[0]), int(offset.shape[0])
    use_grid = _knn_grid_enabled and n >= KNN_GRID_MIN_POINTS and b <= 4096
    key = None
    if use_grid:
        key = _Lru.sig(xyz, new_xyz, offset, new_offset) + (int(nsample),)
        hit = _knn_cache.get(key)
        if hit is not None:
            idx, d2, versions, ev, stream = hit
            if (idx._version, d2._version) == versions:
                cur = torch.cuda.current_stream()
                if stream != cur:
                    cur.wait_event(ev)
                    idx.record_stream(cur)
                    d2.record_stream(cur)
                return idx, d2
    idx = _empty((m, nsample), torch.int32, xyz)
    d2 = _empty((m, nsample), torch.float32, xyz)
    if use_grid:
        ws = _grid_for(xyz, offset)
        L.call("tgn_knn_grid_query", b, n, int(m), int(nsample), L.ptr(xyz), L.ptr(new_xyz), L.ptr(offset), L.ptr(new_offset),
               L.ptr(ws), L.ptr(idx), L.ptr(d2), L.stream_ptr())
        ev = torch.cuda.Event()
        ev.record()
        _knn_cache.put(key, (xyz, new_xyz, offset, new_offset), (idx, d2, (idx._version, d2._version), ev, torch.cuda.current_stream()))
    else:
        L.call("tgn_knnquery", b, int(m), int(nsample), L.ptr(xyz), L.ptr(new_xyz), L.ptr(offset),
               L.ptr(new_offset), L.ptr(idx), L.ptr(d2), L.stream_ptr())
    return idx, d2


class KNNQuery(Function):
    """:30-45.  output: idx (m,nsample) int32, dist (m,nsample) = sqrt of the squared distances."""

    @staticmethod
    def forward(ctx, nsample, xyz, new_xyz, offset, new_offset):
        if new_xyz is None:
            new_xyz = xyz
        idx, d2 = knn_packed(int(nsample), xyz, new_xyz, offset, new_offset)
        idx = idx.view_as(idx)              # a fresh tensor object over the (possibly cached, shared) storage
        dist = torch.sqrt(d2)
        ctx.mark_non_differentiable(idx, dist)
        return idx, dist


knnquery = KNNQuery.apply


_deterministic_backward = True
_csr_cache = _Lru(16)       # index tensor -> inverse index (CSR)


def set_deterministic_backward(flag: bool) -> None:
    """True (default): the scatter-add backwards of grouping / index_points / pointops.interpolation add each
    destination row's contributions in ascending source position through an inverse index -- torch's index_put
    order, i.e. gradients bit-identical to the reference's autograd and reproducible.  False: fp32 atomics."""
    global _deterministic_backward
    _deterministic_backward = bool(flag)


def csr_for(keys: torch.Tensor, n_rows: int) -> torch.Tensor:
    """Inverse index of a flat int32 key tensor (cached per tensor identity; the kNN cache hands the same ``idx`` to
    every layer of a level, so one build serves all their backwards)."""
    key = _Lru.sig(keys) + (int(n_rows),)
    cur = torch.cuda.current_stream()
    hit = _csr_cache.get(key)
    if hit is not None:
        ws, ev, stream = hit
        if stream != cur:
            cur.wait_event(ev)
            ws.record_stream(cur)
        return ws
    M = keys.numel()
    ws = torch.empty(L.load().tgn_csr_bytes(M, int(n_rows)), dtype=torch.uint8, device=keys.device)
    L.call("tgn_csr_build", M, int(n_rows), L.ptr(keys), L.ptr(ws), L.stream_ptr())
    ev = torch.cuda.Event()
    ev.record(cur)
    _csr_cache.put(key, (keys,), (ws, ev, cur))
    return ws


def gather_backward(grad_output: torch.Tensor, idx: torch.Tensor, n_rows: int) -> torch.Tensor:
    """grad wrt ``input`` of ``input[idx]``: grad_output (..., c) with idx.numel() leading rows -> (n_rows, c)."""
    c = grad_output.shape[-1]
    M = idx.numel()
    if _deterministic_backward:
        ws = csr_for(idx, n_rows)
        grad_in = torch.empty((n_rows, c), dtype=torch.float32, device=grad_output.device)
        L.call("tgn_gather_backward_det", M, int(n_rows), int(c), L.ptr(ws), L.ptr(grad_output), L.ptr(grad_in), L.stream_ptr())
        return grad_in
    grad_in = torch.zeros((n_rows, c), dtype=torch.float32, device=grad_output.device)
    L.call("tgn_grouping_backward", M, 1, c, L.ptr(grad_output), L.ptr(idx), L.ptr(grad_in), L.stream_ptr())
    return grad_in


class Grouping(Function):
    """:48-76.  input (n,c), idx (m,nsample) -> (m,nsample,c); backward scatter-adds."""

    @staticmethod
    def forward(ctx, input, idx):
        _need(input, torch.float32, "input")
        _need(idx, torch.int32, "idx")
        m, nsample = idx.shape
        n, c = input.shape
        out = _empty((m, nsample, c), torch.float32, input)
        L.call("tgn_grouping_forward", m, nsample, c, L.ptr(input), L.ptr(idx), L.ptr(out), L.stream_ptr())
        ctx.n = n
        ctx.save_for_backward(idx)
        return out

    @staticmethod
    def backward(ctx, grad_output):
        (idx,) = ctx.saved_tensors
        return gather_backward(grad_output.contiguous(), idx, ctx.n), None


grouping = Grouping.apply


def queryandgroup(nsample, xyz, new_xyz, feat, idx, offset, new_offset, use_xyz=True):
    """:79-100.  kNN (unless idx is given) + gather + centre-subtract + concat.
    output (m, nsample, 3+c) with channel order [xyz_rel, feat], or (m, nsample, c)."""
    assert xyz.is_contiguous() and feat.is_contiguous()
    if new_xyz is None:
        new_xyz = xyz
    assert new_xyz.is_contiguous()
    if idx is None:
        idx, _ = knnquery(nsample, xyz, new_xyz, offset, new_offset)
    grouped_feat = grouping(feat, idx)
    if not use_xyz:
        return grouped_feat
    grouped_xyz = grouping(xyz, idx) - new_xyz.unsqueeze(1)
    return torch.cat((grouped_xyz, grouped_feat), -1)


class Subtraction(Function):
    """:103-130.  out[n,s,:] = input1[n,:] - input2[idx[n,s],:]."""

    @staticmethod
    def forward(ctx, input1, input2, idx):
        _need(input1, torch.float32, "input1")
        _need(input2, torch.float32, "input2")
        _need(idx, torch.int32, "idx")
        n, c = input1.shape
        nsample = idx.shape[-1]
        out = _empty((n, nsample, c), torch.float32, input1)
        L.call("tgn_subtraction_forward", n, nsample, c, L.ptr(input1), L.ptr(input2), L.ptr(idx), L.ptr(out), L.stream_ptr())
        ctx.n2 = input2.shape[0]
        ctx.save_for_backward(idx)
        return out

    @staticmethod
    def backward(ctx, grad_output):
        (idx,) = ctx.saved_tensors
        grad_output = grad_output.contiguous()
        n, nsample, c = grad_output.shape
        g1 = torch.zeros((n, c), dtype=torch.float32, device=grad_output.device)
        g2 = torch.zeros((ctx.n2, c), dtype=torch.float32, device=grad_output.device)
        L.call("tgn_subtraction_backward", n, nsample, c, L.ptr(idx), L.ptr(grad_output), L.ptr(g1), L.ptr(g2), L.stream_ptr())
        return g1, g2, None


subtraction = Subtraction.apply


class Aggregation(Function):
    """:133-161.  out[n,c] = sum_s (input[idx[n,s],c] + position[n,s,c]) * weight[n,s,c % w_c]."""

    @staticmethod
    def forward(ctx, input, position, weight, idx):
        _need(input, torch.float32, "input")
        _need(position, torch.float32, "position")
        _need(weight, torch.float32, "weight")
        _need(idx, torch.int32, "idx")
        n, nsample, c = position.shape
        w_c = weight.shape[-1]
        out = torch.zeros((n, c), dtype=torch.float32, device=input.device)
        L.call("tgn_aggregation_forward", n, nsample, c, w_c, L.ptr(input), L.ptr(position), L.ptr(weight), L.ptr(idx),
               L.ptr(out), L.stream_ptr())
        ctx.save_for_backward(input, position, weight, idx)
        return out

    @staticmethod
    def backward(ctx, grad_output):
        input, position, weight, idx = ctx.saved_tensors
        grad_output = grad_output.contiguous()
        n, nsample, c = position.shape
        w_c = weight.shape[-1]
        gi = torch.zeros_like(input)
        gp = torch.zeros_like(position)
        gw = torch.zeros_like(weight)
        L.call("tgn_aggregation_backward", n, nsample, c, w_c, L.ptr(input), L.ptr(position), L.ptr(weight), L.ptr(idx),
               L.ptr(grad_output), L.ptr(gi), L.ptr(gp), L.ptr(gw), L.stream_ptr())
        return gi, gp, gw, None


aggregation = Aggregation.apply


def _inverse_distance_weights(dist: torch.Tensor) -> torch.Tensor:
    """:171-173 / :192-194: 1/(dist+1e-8), normalised over the k neighbours."""
    rec = 1.0 / (dist + 1e-8)
    return rec / torch.sum(rec, dim=1, keepdim=True)


class _WeightedGather(Function):
    """out[n,:] = sum_i input[idx[n,i],:] * weight[n,i] with a scatter-add backward wrt input."""

    @staticmethod
    def forward(ctx, input, idx, weight, fused=True):
        """``fused``: True = the FMA chain of the reference KERNEL (interpolation_cuda_kernel.cu), atomics backward like it;
        False = pointops.interpolation's torch loop (unfused, k index_put backwards); "sum" = pointnet2's
        torch.sum(index_points(.) * weight, dim=2) (unfused forward, ONE index_put backward)."""
        _need(input, torch.float32, "input")
        _need(idx, torch.int32, "idx")
        _need(weight, torch.float32, "weight")
        n, k = idx.shape
        m, c = input.shape
        out = torch.zeros((n, c), dtype=torch.float32, device=input.device)
        L.call("tgn_weighted_gather", n, c, k, L.ptr(input), L.ptr(idx), L.ptr(weight), L.ptr(out), 1 if fused is True else 0, L.stream_ptr())
        ctx.m, ctx.fused = m, fused
        ctx.save_for_backward(idx, weight)
        return out

    @staticmethod
    def backward(ctx, grad_output):
        idx, weight = ctx.saved_tensors
        grad_output = grad_output.contiguous()
        n, c = grad_output.shape
        k = idx.shape[1]
        if _deterministic_backward and ctx.fused is not True and k <= 8:
            # the torch-loop form (pointops.interpolation): k index_put accumulations summed by autograd, reproduced exactly
            ws = csr_for(idx, ctx.m)
            gi = torch.empty((ctx.m, c), dtype=torch.float32, device=grad_output.device)
            L.call("tgn_weighted_gather_backward_det", idx.numel(), int(ctx.m), int(c), int(k), 1 if ctx.fused == "sum" else 0,
                   L.ptr(ws), L.ptr(grad_output), L.ptr(weight), L.ptr(gi), L.stream_ptr())
            return gi, None, None, None
        gi = torch.zeros((ctx.m, c), dtype=torch.float32, device=grad_output.device)
        L.call("tgn_interpolation_backward", n, c, k, L.ptr(grad_output), L.ptr(idx), L.ptr(weight), L.ptr(gi), L.stream_ptr())
        return gi, None, None, None


def interpolation(xyz, new_xyz, feat, offset, new_offset, k=3):
    """:164-180.  input: xyz (m,3) coarse, new_xyz (n,3) fine, feat (m,c) -> (n,c).
    Weights are constants for autograd (the reference detaches them, :175)."""
    assert xyz.is_contiguous() and new_xyz.is_contiguous() and feat.is_contiguous()
    idx, dist = knnquery(k, xyz, new_xyz, offset, new_offset)
    weight = _inverse_distance_weights(dist).detach().contiguous()
    return _WeightedGather.apply(feat, idx, weight, False)      # the reference accumulates with torch ops here: unfused (:177-179)


class Interpolation(Function):
    """:183-216 (exported as ``interpolation2``; fused kernel form of the same operation)."""

    @staticmethod
    def forward(ctx, xyz, new_xyz, input, offset, new_offset, k=3):
        assert xyz.is_contiguous() and new_xyz.is_contiguous() and input.is_contiguous()
        idx, d2 = knn_packed(int(k), xyz, new_xyz, offset, new_offset)
        weight = _inverse_distance_weights(torch.sqrt(d2)).contiguous()
        n, c, m = new_xyz.shape[0], input.shape[1], input.shape[0]
        out = torch.zeros((n, c), dtype=torch.float32, device=input.device)
        L.call("tgn_interpolation_forward", n, c, int(k), L.ptr(input), L.ptr(idx), L.ptr(weight), L.ptr(out), L.stream_ptr())
        ctx.m, ctx.k = m, int(k)
        ctx.save_for_backward(idx, weight)
        return out

    @staticmethod
    def backward(ctx, grad_output):
        idx, weight = ctx.saved_tensors
        grad_output = grad_output.contiguous()
        n, c = grad_output.shape
        gi = torch.zeros((ctx.m, c), dtype=torch.float32, device=grad_output.device)
        L.call("tgn_interpolation_backward", n, c, ctx.k, L.ptr(grad_output), L.ptr(idx), L.ptr(weight), L.ptr(gi), L.stream_ptr())
        return None, None, gi, None, None, None


interpolation2 = Interpolation.apply
