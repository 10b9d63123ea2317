"""Boundary-aware resampling between the two networks of a tgnet inference, on the GPU (SURVEY.md 8(f)).

``InferencePipeLine.get_boundary_sampled_feats`` (inference_pipelines/inference_pipeline_tgn.py:289-330, called at :48-53)
decides which original mesh vertices lie on a tooth boundary and builds the 24 000-point input of the boundary network from
them.  The reference does it on the host: ``KDTree(sampled_xyz, leaf_size=40).query(org_xyz, k=40)`` in float64 over
1e5 - 2e5 vertices, the share of the 40 neighbours that carry the nearest neighbour's label (``gen_utils.count_unique_by_row``),
a second k = 1 query for the labels, a random subset of the boundary vertices and FPS over the rest.

Here the kNN and the label vote are one call of csrc/knn_f64.cu (exact float64, neighbours ordered by (d2, index), the (m, 40)
index matrix never leaves the kernel), the masks, gathers and FPS (the library's own, bitwise equal to the reference's kernel)
stay on the device, and ``get_boundary_sampled_feats`` keeps the reference method's numpy signature, its results and its use
of numpy's global random generator.  ``accelerate(inference_pipeline_tgn_module)`` swaps the method in.
"""
from __future__ import annotations

from typing import Callable, Tuple, Union

import numpy as np
import torch

from . import _lib as L
from . import pointops

MAX_K = 64
_ws = {}


def _workspace(n: int, device) -> torch.Tensor:
    need = int(L.load().tgn_knn_f64_bytes(int(n)))
    key = (device.index, torch.cuda.current_stream(device).cuda_stream)
    buf = _ws.get(key)
    if buf is None or buf.numel() < need:
        buf = torch.empty(need, dtype=torch.uint8, device=device)
        _ws[key] = buf
    return buf


def _check_knn_args(points: torch.Tensor, queries: torch.Tensor, k: int) -> None:
    for name, t in (("points", points), ("queries", queries)):
        if t.dim() != 2 or t.shape[1] != 3 or t.dtype != torch.float64:
            raise L.TgnError(f"knn_f64: {name} must be (n, 3) float64, got {tuple(t.shape)} {t.dtype}")
    n = points.shape[0]
    if not 1 <= k <= min(n, MAX_K):
        raise L.TgnError(f"knn_f64: need 1 <= k <= min(n, {MAX_K}), got k={k} with n={n}")
    L.require_cuda(points, queries)
    if points.device != queries.device:
        raise L.TgnError("knn_f64: points and queries are on different devices")


def _knn_f64_call(points: torch.Tensor, queries: torch.Tensor, k: int, labels=None, idx=None, dist=None, nn0=None, agree=None) -> None:
    points, queries = points.contiguous(), queries.contiguous()
    n, m = points.shape[0], queries.shape[0]
    if m == 0:
        return
    ws = _workspace(n, points.device)
    L.call("tgn_knn_f64", n, m, int(k), L.ptr(points), L.ptr(queries), L.ptr(ws), L.ptr(labels), L.ptr(idx), L.ptr(dist),
           L.ptr(nn0), L.ptr(agree), L.stream_ptr())


def knn_f64(points: torch.Tensor, queries: torch.Tensor, k: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """points (n,3), queries (m,3) float64 CUDA -> (idx int64 (m,k), dist float64 (m,k)): the answer of
    ``sklearn.neighbors.KDTree(points).query(queries, k)``, neighbours ascending by (squared distance, index).
    1 <= k <= min(n, 64); non-finite coordinates are refused."""
    k = int(k)
    _check_knn_args(points, queries, k)
    if not bool(torch.isfinite(points).all()) or not bool(torch.isfinite(queries).all()):
        raise L.TgnError("knn_f64: non-finite coordinates")
    m = queries.shape[0]
    idx = torch.empty((m, k), dtype=torch.int64, device=points.device)
    dist = torch.empty((m, k), dtype=torch.float64, device=points.device)
    _knn_f64_call(points, queries, k, idx=idx, dist=dist)
    return idx, dist


def neighbour_vote(points: torch.Tensor, queries: torch.Tensor, codes: torch.Tensor, k: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """points (n,3), queries (m,3) float64 CUDA, codes (n) int32 labels -> (nn0 int32 (m), agree int32 (m)): the index of every
    query's nearest point and how many of its k nearest (the neighbours of ``knn_f64``) carry that point's label."""
    k = int(k)
    _check_knn_args(points, queries, k)
    if codes.shape != (points.shape[0],) or codes.dtype != torch.int32 or codes.device != points.device:
        raise L.TgnError(f"neighbour_vote: codes must be ({points.shape[0]},) int32 on {points.device}, got {tuple(codes.shape)} {codes.dtype}")
    m = queries.shape[0]
    nn0 = torch.empty(m, dtype=torch.int32, device=points.device)
    agree = torch.empty(m, dtype=torch.int32, device=points.device)
    _knn_f64_call(points, queries, k, labels=codes.contiguous(), nn0=nn0, agree=agree)
    return nn0, agree


def label_codes(labels: torch.Tensor) -> torch.Tensor:
    """Dense int32 codes of arbitrary labels, equal codes exactly for equal values (np.unique(return_inverse=True))."""
    if labels.is_floating_point() and bool(torch.isnan(labels).any()):
        raise L.TgnError("boundary: NaN labels")
    return torch.unique(labels, return_inverse=True)[1].to(torch.int32)


def boundary_sample(sampled_xyz: torch.Tensor, point_labels: torch.Tensor, org_feats: torch.Tensor, *, k: int = 40,
                    bdl_ratio: float, num_bdl: int, num_all: int,
                    perm: Union[Callable[[int], object], np.ndarray, torch.Tensor]):
    """The computation of get_boundary_sampled_feats on device tensors.

    sampled_xyz (n,3) float64, point_labels (n,) labels of the sampled points, org_feats (m,C) with xyz in columns 0-2.
    A vertex is a boundary vertex when (neighbours among its k nearest sampled points that carry its nearest point's label) / k
    < bdl_ratio.  ``perm`` orders the boundary vertices: a permutation of range(n_bd), or a callable n_bd -> permutation
    (``np.random.permutation`` for the reference's draw); the first num_bdl are kept.  The remaining num_all - kept rows are the
    FPS of the non-boundary vertices' float32 xyz.  Returns (feats (num_all, C), labels (num_all, 1), bd_feats, bd_labels) with
    the dtypes of org_feats and point_labels, boundary rows first."""
    k = int(k)
    if point_labels.dim() != 1 or point_labels.shape[0] != sampled_xyz.shape[0]:
        raise L.TgnError(f"boundary_sample: point_labels must be ({sampled_xyz.shape[0]},), got {tuple(point_labels.shape)}")
    if org_feats.dim() != 2 or org_feats.shape[1] < 3:
        raise L.TgnError(f"boundary_sample: org_feats must be (m, C >= 3), got {tuple(org_feats.shape)}")
    queries = org_feats[:, :3].to(torch.float64)
    _check_knn_args(sampled_xyz, queries, k)
    L.require_cuda(point_labels, org_feats)
    dev = sampled_xyz.device
    if not bool(torch.isfinite(sampled_xyz).all()) or not bool(torch.isfinite(queries).all()):
        raise L.TgnError("boundary_sample: non-finite coordinates")
    nn0, agree = neighbour_vote(sampled_xyz, queries, label_codes(point_labels.to(dev)), k)

    boundary = agree.to(torch.float64) / float(k) < bdl_ratio          # the reference's label_counts[:, 0] / 40. < bdl_ratio
    ps_labels = point_labels.to(dev)[nn0.long()].reshape(-1, 1)
    bd_rows = torch.nonzero(boundary).reshape(-1)
    non_rows = torch.nonzero(~boundary).reshape(-1)
    n_bd = int(bd_rows.shape[0])

    order = perm(n_bd) if callable(perm) else perm
    order = torch.as_tensor(np.asarray(order) if not torch.is_tensor(order) else order).to(dev)
    if order.dim() != 1 or order.shape[0] != n_bd or order.is_floating_point():
        raise L.TgnError(f"boundary_sample: perm must be an integer permutation of range({n_bd}), got {tuple(order.shape)} {order.dtype}")
    keep = order[:num_bdl].long()
    if n_bd and bool(((keep < 0) | (keep >= n_bd)).any()):
        raise L.TgnError(f"boundary_sample: perm holds indices outside range({n_bd})")
    bd_keep = bd_rows[keep]

    need = int(num_all) - int(bd_keep.shape[0])
    n_non = int(non_rows.shape[0])
    if n_non <= need:
        raise L.TgnError(f"boundary_sample: {n_non} non-boundary vertices cannot give {need} FPS samples (the reference raises too)")
    xyz32 = org_feats[non_rows, :3].to(torch.float32).contiguous()
    sel = pointops.fps_packed(xyz32, torch.tensor([n_non], dtype=torch.int32, device=dev),
                              torch.tensor([need], dtype=torch.int32, device=dev), n_non, need)
    non_keep = non_rows[sel.long()]

    bd_feats, bd_labels = org_feats[bd_keep], ps_labels[bd_keep]
    feats = torch.cat([bd_feats, org_feats[non_keep]], 0)
    labels = torch.cat([bd_labels, ps_labels[non_keep]], 0)
    return feats, labels, bd_feats, bd_labels


_ORIGINAL = "_tgn_original_get_boundary_sampled_feats"


def get_boundary_sampled_feats(self, point_labels, org_feats, sampled_feats, sample_output_features):
    """Drop-in for InferencePipeLine.get_boundary_sampled_feats (inference_pipeline_tgn.py:289-330): numpy in, numpy out,
    ``self.config["boundary_sampling_info"]`` read as the reference reads it, the boundary subset drawn by the same single
    ``np.random.permutation`` call.  With ``sample_output_features`` (never passed by the reference's callers) the original
    method runs."""
    if sample_output_features is not None:
        original = getattr(self, _ORIGINAL, None)
        if original is None:
            raise L.TgnError("get_boundary_sampled_feats: the sample_output_features branch needs the original method (use accelerate())")
        return original(point_labels, org_feats, sampled_feats, sample_output_features)
    info = self.config["boundary_sampling_info"]
    point_labels = np.asarray(point_labels)
    org_feats = np.asarray(org_feats)
    sampled_xyz = np.asarray(sampled_feats)[:, :3]
    if not (np.isfinite(sampled_xyz).all() and np.isfinite(org_feats[:, :3]).all()):
        raise L.TgnError("get_boundary_sampled_feats: non-finite coordinates")
    if point_labels.dtype.kind in "fc" and np.isnan(point_labels).any():
        raise L.TgnError("get_boundary_sampled_feats: NaN labels")
    if not torch.cuda.is_available():
        raise L.TgnError("get_boundary_sampled_feats needs a CUDA device (there is no CPU path)")
    dev = torch.device("cuda", torch.cuda.current_device())
    out = boundary_sample(torch.as_tensor(np.ascontiguousarray(sampled_xyz, dtype=np.float64), device=dev),
                          torch.as_tensor(np.ascontiguousarray(point_labels).reshape(-1), device=dev),
                          torch.as_tensor(np.ascontiguousarray(org_feats), device=dev),
                          k=40, bdl_ratio=info["bdl_ratio"], num_bdl=info["num_of_bdl_points"], num_all=info["num_of_all_points"],
                          perm=np.random.permutation)
    return tuple(t.cpu().numpy() for t in out)


def accelerate(inference_pipeline_tgn_module) -> None:
    """Point ``InferencePipeLine.get_boundary_sampled_feats`` of an imported reference module at the device version; the original
    is kept for its ``sample_output_features`` branch."""
    cls = inference_pipeline_tgn_module.InferencePipeLine
    if cls.__dict__.get("get_boundary_sampled_feats") is not get_boundary_sampled_feats:
        setattr(cls, _ORIGINAL, cls.get_boundary_sampled_feats)
        cls.get_boundary_sampled_feats = get_boundary_sampled_feats
