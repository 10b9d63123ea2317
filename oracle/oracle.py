"""oracle/oracle.py -- Python face of the CPU restatement (TEST INFRASTRUCTURE ONLY).

Nothing under ``toothgroupnetwork_b200/`` may import this module.  Callers allowed:
``tests/``, ``__graft_entry__.smoke()``, ``bench.py`` (cpu_baseline / --impl reference).

Two layers:

* thin ctypes wrappers over ``oracle/pointops_oracle.c`` (FPS, kNN, gather family, expanded
  square distance, ball query, 3-NN) operating on numpy arrays;
* torch-CPU restatements of the reference's ``pointnet2_utils`` modules
  (``external_libs/pointnet2_utils/pointnet2_utils.py``) written as pure functions over explicit
  parameter lists, so they can be evaluated in fp32 (the reference's arithmetic) or fp64
  (ground truth for tolerance tests).

Parity pins: ``tests/golden/ref_torch_*.npz`` (reference python imported from /root/reference,
generator ``tests/golden/make_ref_torch_golden.py``) and ``tests/golden/ref_cuda_*.npz``
(reference CUDA kernels compiled verbatim, run on the GPU, generator
``tests/golden/make_ref_cuda_golden.py``).
"""
from __future__ import annotations

import ctypes
import os
import subprocess
from typing import List, Optional, Sequence, Tuple

import numpy as np
import torch
import torch.nn.functional as F

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "_build", "liboracle.so")
_LIB = None

_f32p = ctypes.POINTER(ctypes.c_float)
_i32p = ctypes.POINTER(ctypes.c_int)
_i64p = ctypes.POINTER(ctypes.c_int64)


def build(force: bool = False) -> str:
    """Compile the C restatement with gcc (``make -C oracle``)."""
    src = os.path.join(_HERE, "pointops_oracle.c")
    if force or not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(src):
        subprocess.check_call(["make", "-C", _HERE, "-s"] + (["-B"] if force else []))
    return _SO


def lib() -> ctypes.CDLL:
    global _LIB
    if _LIB is None:
        build()
        _LIB = ctypes.CDLL(_SO)
        _LIB.oracle_opt_n_threads.restype = ctypes.c_int
    return _LIB


def _f(a) -> np.ndarray:
    return np.ascontiguousarray(a, dtype=np.float32)


def _i(a) -> np.ndarray:
    return np.ascontiguousarray(a, dtype=np.int32)


def _p(a: np.ndarray, t):
    return a.ctypes.data_as(t)


def opt_n_threads(n: int) -> int:
    return int(lib().oracle_opt_n_threads(int(n)))


# ----------------------------------------------------------------------------- pointops side
def furthestsampling(xyz, offset, new_offset, return_tmp: bool = False):
    """pointops.furthestsampling (pointops/functions/pointops.py:10-27): packed ``xyz (n,3)``,
    cumulative ``offset (b)``, ``new_offset (b)`` -> global row ids ``(m,) int32``."""
    xyz, offset, new_offset = _f(xyz), _i(offset), _i(new_offset)
    b = offset.shape[0]
    sizes = np.diff(np.concatenate([[0], offset]))
    n_max = int(sizes.max()) if b else 0
    m = int(new_offset[-1]) if b else 0
    idx = np.zeros(m, np.int32)
    tmp = np.full(xyz.shape[0], 1e10, np.float32)
    lib().oracle_furthestsampling(b, n_max, _p(xyz, _f32p), _p(offset, _i32p), _p(new_offset, _i32p),
                                  _p(tmp, _f32p), _p(idx, _i32p))
    return (idx, tmp) if return_tmp else idx


def knnquery(nsample: int, xyz, new_xyz, offset, new_offset):
    """pointops.knnquery (pointops.py:30-45) -> ``idx (m,k) int32``, ``dist (m,k)`` = sqrt(d2),
    plus the raw squared distances as third value."""
    xyz, offset = _f(xyz), _i(offset)
    new_xyz = xyz if new_xyz is None else _f(new_xyz)
    new_offset = _i(new_offset)
    m = new_xyz.shape[0]
    idx = np.zeros((m, nsample), np.int32)
    d2 = np.zeros((m, nsample), np.float32)
    lib().oracle_knnquery(m, nsample, _p(xyz, _f32p), _p(new_xyz, _f32p), _p(offset, _i32p),
                          _p(new_offset, _i32p), _p(idx, _i32p), _p(d2, _f32p))
    return idx, np.sqrt(d2), d2


def grouping_forward(inp, idx):
    inp, idx = _f(inp), _i(idx)
    m, k = idx.shape
    c = inp.shape[1]
    out = np.empty((m, k, c), np.float32)
    lib().oracle_grouping_forward(m, k, c, _p(inp, _f32p), _p(idx, _i32p), _p(out, _f32p))
    return out


def grouping_backward(grad_out, idx, n):
    grad_out, idx = _f(grad_out), _i(idx)
    m, k, c = grad_out.shape
    gi = np.zeros((n, c), np.float32)
    lib().oracle_grouping_backward(m, k, c, _p(grad_out, _f32p), _p(idx, _i32p), _p(gi, _f32p))
    return gi


def interpolation_forward(inp, idx, weight):
    inp, idx, weight = _f(inp), _i(idx), _f(weight)
    n, k = idx.shape
    c = inp.shape[1]
    out = np.zeros((n, c), np.float32)
    lib().oracle_interpolation_forward(n, c, k, _p(inp, _f32p), _p(idx, _i32p), _p(weight, _f32p), _p(out, _f32p))
    return out


def interpolation_backward(grad_out, idx, weight, m):
    grad_out, idx, weight = _f(grad_out), _i(idx), _f(weight)
    n, c = grad_out.shape
    k = idx.shape[1]
    gi = np.zeros((m, c), np.float32)
    lib().oracle_interpolation_backward(n, c, k, _p(grad_out, _f32p), _p(idx, _i32p), _p(weight, _f32p), _p(gi, _f32p))
    return gi


def subtraction_forward(in1, in2, idx):
    in1, in2, idx = _f(in1), _f(in2), _i(idx)
    n, c = in1.shape
    k = idx.shape[1]
    out = np.empty((n, k, c), np.float32)
    lib().oracle_subtraction_forward(n, k, c, _p(in1, _f32p), _p(in2, _f32p), _p(idx, _i32p), _p(out, _f32p))
    return out


def subtraction_backward(idx, grad_out, n2: Optional[int] = None):
    idx, grad_out = _i(idx), _f(grad_out)
    n, k, c = grad_out.shape
    g1 = np.zeros((n, c), np.float32)
    g2 = np.zeros((n if n2 is None else n2, c), np.float32)
    lib().oracle_subtraction_backward(n, k, c, _p(idx, _i32p), _p(grad_out, _f32p), _p(g1, _f32p), _p(g2, _f32p))
    return g1, g2


def aggregation_forward(inp, pos, weight, idx):
    inp, pos, weight, idx = _f(inp), _f(pos), _f(weight), _i(idx)
    n, k, c = pos.shape
    w_c = weight.shape[-1]
    out = np.zeros((n, c), np.float32)
    lib().oracle_aggregation_forward(n, k, c, w_c, _p(inp, _f32p), _p(pos, _f32p), _p(weight, _f32p),
                                     _p(idx, _i32p), _p(out, _f32p))
    return out


def aggregation_backward(inp, pos, weight, idx, grad_out):
    inp, pos, weight, idx, grad_out = _f(inp), _f(pos), _f(weight), _i(idx), _f(grad_out)
    n, k, c = pos.shape
    w_c = weight.shape[-1]
    gi = np.zeros_like(inp)
    gp = np.zeros_like(pos)
    gw = np.zeros_like(weight)
    lib().oracle_aggregation_backward(n, k, c, w_c, _p(inp, _f32p), _p(pos, _f32p), _p(weight, _f32p),
                                      _p(idx, _i32p), _p(grad_out, _f32p), _p(gi, _f32p), _p(gp, _f32p), _p(gw, _f32p))
    return gi, gp, gw


def queryandgroup(nsample, xyz, new_xyz, feat, idx, offset, new_offset, use_xyz=True):
    """pointops.queryandgroup (pointops.py:79-100): kNN (unless idx given), gather xyz and
    features, subtract the query centre, concatenate [xyz_rel, feat]."""
    xyz, feat = _f(xyz), _f(feat)
    new_xyz = xyz if new_xyz is None else _f(new_xyz)
    if idx is None:
        idx, _, _ = knnquery(nsample, xyz, new_xyz, offset, new_offset)
    g_xyz = xyz[idx.reshape(-1)].reshape(idx.shape[0], nsample, 3) - new_xyz[:, None, :]
    g_feat = feat[idx.reshape(-1)].reshape(idx.shape[0], nsample, feat.shape[1])
    return np.concatenate([g_xyz, g_feat], -1) if use_xyz else g_feat


def interpolation(xyz, new_xyz, feat, offset, new_offset, k=3):
    """pointops.interpolation (pointops.py:164-180): weights 1/(dist+1e-8) on the (non-squared)
    kNN distances, normalised, then k successive gather-multiply-adds in neighbour order."""
    idx, dist, _ = knnquery(k, xyz, new_xyz, offset, new_offset)
    rec = (np.float32(1.0) / (dist + np.float32(1e-8))).astype(np.float32)
    w = (rec / rec.sum(1, keepdims=True, dtype=np.float32)).astype(np.float32)
    feat = _f(feat)
    out = np.zeros((idx.shape[0], feat.shape[1]), np.float32)
    for i in range(k):
        out += feat[idx[:, i]] * w[:, i:i + 1]
    return out, idx, w


# ----------------------------------------------------------------------------- pointnet2 side
def square_distance(src, dst):
    """pointnet2_utils.square_distance (pointnet2_utils.py:20-41), batched (B,N,3),(B,M,3)->(B,N,M)."""
    src, dst = _f(src), _f(dst)
    B, N, _ = src.shape
    M = dst.shape[1]
    out = np.empty((B, N, M), np.float32)
    for b in range(B):
        lib().oracle_square_distance(N, M, _p(src[b], _f32p), _p(dst[b], _f32p), _p(out[b], _f32p))
    return out


def radius_sq_f32(radius: float) -> np.float32:
    """The scalar torch actually compares against in ``sqrdists > radius ** 2``
    (pointnet2_utils.py:136): python double squared, then cast to the tensor dtype."""
    return np.float32(float(radius) ** 2)


def query_ball_point(radius, nsample, xyz, new_xyz):
    """pointnet2_utils.query_ball_point (pointnet2_utils.py:120-144) -> (B,S,nsample) int64."""
    xyz, new_xyz = _f(xyz), _f(new_xyz)
    B, N, _ = xyz.shape
    S = new_xyz.shape[1]
    out = np.empty((B, S, nsample), np.int64)
    r2 = ctypes.c_float(float(radius_sq_f32(radius)))
    for b in range(B):
        lib().oracle_query_ball_point(N, S, r2, nsample, _p(xyz[b], _f32p), _p(new_xyz[b], _f32p), _p(out[b], _i64p))
    return out


def three_nn(xyz1, xyz2):
    """Top-3 of the expanded distance matrix (pointnet2_utils.py:333-335). (B,N,3),(B,S,3)."""
    xyz1, xyz2 = _f(xyz1), _f(xyz2)
    B, N, _ = xyz1.shape
    S = xyz2.shape[1]
    d = np.empty((B, N, 3), np.float32)
    i = np.empty((B, N, 3), np.int64)
    for b in range(B):
        lib().oracle_three_nn(N, S, _p(xyz1[b], _f32p), _p(xyz2[b], _f32p), _p(d[b], _f32p), _p(i[b], _i64p))
    return d, i


def farthest_point_sample(xyz, npoint):
    """pointnet2_utils.farthest_point_sample (pointnet2_utils.py:64-98): batched (B,N,3) ->
    per-cloud-local int64 indices (B,npoint) through the packed pointops FPS."""
    xyz = _f(xyz)
    B, N, _ = xyz.shape
    offset = (np.arange(1, B + 1) * N).astype(np.int32)
    new_offset = (np.arange(1, B + 1) * npoint).astype(np.int32)
    idx = furthestsampling(xyz.reshape(-1, 3), offset, new_offset).astype(np.int64)
    return idx.reshape(B, npoint) - (np.arange(B, dtype=np.int64) * N)[:, None]


def fps_torchloop(xyz, npoint, start=0):
    """Reference's CPU-capable FPS loop (pointnet2_utils.py:103-118) with a fixed start."""
    xyz = _f(xyz)
    n = xyz.shape[0]
    dist = np.empty(n, np.float32)
    cent = np.empty(npoint, np.int64)
    lib().oracle_fps_torchloop(n, npoint, start, _p(xyz, _f32p), _p(dist, _f32p), _p(cent, _i64p))
    return cent


def index_points(points: torch.Tensor, idx: torch.Tensor) -> torch.Tensor:
    """pointnet2_utils.index_points (pointnet2_utils.py:44-61): batched row gather."""
    B = points.shape[0]
    flat = idx.reshape(B, -1)
    out = torch.gather(points, 1, flat.unsqueeze(-1).expand(-1, -1, points.shape[-1]))
    return out.reshape(*idx.shape, points.shape[-1])


class MlpParams:
    """One 1x1-conv + BatchNorm layer: weight (Co,Ci), bias (Co), gamma, beta, running mean/var."""

    def __init__(self, weight, bias, gamma, beta, mean, var, eps=1e-5):
        self.weight, self.bias, self.gamma, self.beta, self.mean, self.var, self.eps = \
            weight, bias, gamma, beta, mean, var, eps

    def to(self, dtype):
        return MlpParams(*[t.to(dtype) for t in (self.weight, self.bias, self.gamma, self.beta, self.mean, self.var)], self.eps)


def _conv_bn_relu(x: torch.Tensor, p: MlpParams, train_bn: bool) -> torch.Tensor:
    """x: (B, C, *spatial).  conv1x1 -> BatchNorm -> ReLU (pointnet2_utils.py:232-235)."""
    shp = x.shape
    y = torch.einsum("oc,bcn->bon", p.weight, x.reshape(shp[0], shp[1], -1)) + p.bias.view(1, -1, 1)
    if train_bn:
        mu = y.mean(dim=(0, 2), keepdim=True)
        var = y.var(dim=(0, 2), unbiased=False, keepdim=True)
    else:
        mu, var = p.mean.view(1, -1, 1), p.var.view(1, -1, 1)
    y = (y - mu) / torch.sqrt(var + p.eps) * p.gamma.view(1, -1, 1) + p.beta.view(1, -1, 1)
    return F.relu(y).reshape(shp[0], -1, *shp[2:])


def set_abstraction(xyz: torch.Tensor, points: Optional[torch.Tensor], npoint, radius, nsample,
                    layers: Sequence[MlpParams], group_all=False, train_bn=False, dtype=torch.float32):
    """PointNetSetAbstraction.forward (pointnet2_utils.py:213-239) as a pure function.
    xyz (B,3,N), points (B,D,N) or None -> new_xyz (B,3,S), new_points (B,C_out,S).
    Channel order inside a group is [xyz_rel, feats] (pointnet2_utils.py:169).
    Sampling and ball membership always run in fp32 (indices are dtype-independent inputs to
    the MLP); ``dtype`` selects the arithmetic of the MLP only."""
    xyz_t = xyz.permute(0, 2, 1).contiguous().float()
    pts_t = None if points is None else points.permute(0, 2, 1).contiguous()
    B, N, _ = xyz_t.shape
    if group_all:
        new_xyz = torch.zeros(B, 1, 3)
        grouped = xyz_t.view(B, 1, N, 3).to(dtype)
        if pts_t is not None:
            grouped = torch.cat([grouped, pts_t.view(B, 1, N, -1).to(dtype)], -1)
    else:
        fps = torch.from_numpy(farthest_point_sample(xyz_t.numpy(), npoint))
        new_xyz = index_points(xyz_t, fps)
        gidx = torch.from_numpy(query_ball_point(radius, nsample, xyz_t.numpy(), new_xyz.numpy()))
        grouped = (index_points(xyz_t, gidx) - new_xyz.view(B, npoint, 1, 3)).to(dtype)
        if pts_t is not None:
            grouped = torch.cat([grouped, index_points(pts_t, gidx).to(dtype)], -1)
    h = grouped.permute(0, 3, 2, 1)  # (B, C, K, S)
    for p in layers:
        h = _conv_bn_relu(h, p.to(dtype), train_bn)
    return new_xyz.permute(0, 2, 1), h.max(dim=2)[0]


def set_abstraction_msg(xyz, points, npoint, radius_list, nsample_list,
                        branches: Sequence[Sequence[MlpParams]], train_bn=False, dtype=torch.float32):
    """PointNetSetAbstractionMsg.forward (pointnet2_utils.py:261-299).  One FPS, then per radius
    a ball query + group + MLP + max; channel order inside a group is [feats, xyz_rel] (:285)."""
    xyz_t = xyz.permute(0, 2, 1).contiguous().float()
    pts_t = None if points is None else points.permute(0, 2, 1).contiguous()
    B, N, _ = xyz_t.shape
    fps = torch.from_numpy(farthest_point_sample(xyz_t.numpy(), npoint))
    new_xyz = index_points(xyz_t, fps)
    outs = []
    for radius, K, layers in zip(radius_list, nsample_list, branches):
        gidx = torch.from_numpy(query_ball_point(radius, K, xyz_t.numpy(), new_xyz.numpy()))
        g_xyz = (index_points(xyz_t, gidx) - new_xyz.view(B, npoint, 1, 3)).to(dtype)
        grouped = g_xyz if pts_t is None else torch.cat([index_points(pts_t, gidx).to(dtype), g_xyz], -1)
        h = grouped.permute(0, 3, 2, 1)
        for p in layers:
            h = _conv_bn_relu(h, p.to(dtype), train_bn)
        outs.append(h.max(dim=2)[0])
    return new_xyz.permute(0, 2, 1), torch.cat(outs, 1)


def feature_propagation(xyz1, xyz2, points1, points2, layers: Sequence[MlpParams],
                        train_bn=False, dtype=torch.float32):
    """PointNetFeaturePropagation.forward (pointnet2_utils.py:313-352): 3-NN inverse *squared*
    distance interpolation (weights 1/(d2+1e-8), :337-339), skip concat [points1, interp],
    then conv1x1+BN+ReLU layers.  xyz1 (B,3,N) fine, xyz2 (B,3,S) coarse."""
    x1 = xyz1.permute(0, 2, 1).contiguous().float()
    x2 = xyz2.permute(0, 2, 1).contiguous().float()
    p2 = points2.permute(0, 2, 1).contiguous().to(dtype)
    B, N, _ = x1.shape
    S = x2.shape[1]
    if S == 1:
        interp = p2.repeat(1, N, 1)
    else:
        d, i = three_nn(x1.numpy(), x2.numpy())
        d, i = torch.from_numpy(d).to(dtype), torch.from_numpy(i)
        rec = 1.0 / (d + 1e-8)
        w = rec / rec.sum(dim=2, keepdim=True)
        interp = (index_points(p2, i) * w.unsqueeze(-1)).sum(dim=2)
    if points1 is not None:
        interp = torch.cat([points1.permute(0, 2, 1).to(dtype), interp], -1)
    h = interp.permute(0, 2, 1)
    for p in layers:
        h = _conv_bn_relu(h, p.to(dtype), train_bn)
    return h


def sa_sample_and_search_batch(xyz, npoint, radius, nsample):
    """FPS loop (start 0) + centre gather + ball query for a batch (B,N,3), one cloud per OpenMP
    thread -- the CPU baseline of bench.py.  -> fps (B,S) int64, new_xyz (B,S,3), group_idx (B,S,K)."""
    xyz = _f(xyz)
    B, N, _ = xyz.shape
    fps = np.empty((B, npoint), np.int64)
    new_xyz = np.empty((B, npoint, 3), np.float32)
    gidx = np.empty((B, npoint, nsample), np.int64)
    lib().oracle_sa_sample_and_search_batch(B, N, int(npoint), ctypes.c_float(float(radius_sq_f32(radius))), int(nsample),
                                            _p(xyz, _f32p), _p(fps, _i64p), _p(new_xyz, _f32p), _p(gidx, _i64p))
    return fps, new_xyz, gidx


def sa_group_mlp_max_batch(xyz, feats, new_xyz, gidx, layers: Sequence[MlpParams]):
    """Grouped MLP (eval-mode BatchNorm) + max for a batch, one cloud per OpenMP thread (bench.py's CPU baseline and
    its parity checker).  xyz (B,N,3), feats (B,N,D) point-major or None, new_xyz (B,S,3), gidx (B,S,K) int64
    -> (B, C_out, S) float32; channel order of a group is [xyz_rel, feats] (pointnet2_utils.py:169)."""
    xyz, new_xyz = _f(xyz), _f(new_xyz)
    gidx = np.ascontiguousarray(gidx, dtype=np.int64)
    B, N, _ = xyz.shape
    S, K = gidx.shape[1], gidx.shape[2]
    D = 0 if feats is None else feats.shape[2]
    f = None if feats is None else _f(feats)
    ch = [3 + D] + [int(p.weight.shape[0]) for p in layers]
    wts, scs, shs = [], [], []
    for p in layers:
        w = p.weight.detach().double().numpy()
        scale = (p.gamma.double() / torch.sqrt(p.var.double() + p.eps)).numpy()
        shift = (p.beta.double() - p.mean.double() * torch.from_numpy(scale)).numpy() + scale * p.bias.double().numpy()
        wts.append(_f(w.T))
        scs.append(_f(scale))
        shs.append(_f(shift))
    arr = lambda xs: (ctypes.POINTER(ctypes.c_float) * len(xs))(*[_p(x, _f32p) for x in xs])
    chv = (ctypes.c_int * len(ch))(*ch)
    out = np.empty((B, ch[-1], S), np.float32)
    lib().oracle_sa_group_mlp_max_batch(B, N, S, K, D, _p(xyz, _f32p), None if f is None else _p(f, _f32p), _p(new_xyz, _f32p),
                                        _p(gidx, _i64p), len(layers), chv, arr(wts), arr(scs), arr(shs), _p(out, _f32p))
    return out


# ----------------------------------------------------------------------------- point-transformer blocks (SURVEY 8(f)-3)
def _bn_rows(y: torch.Tensor, bn: dict, prefix: str, train_bn: bool, eps: float = 1e-5) -> torch.Tensor:
    """BatchNorm1d over a (n, K, c) tensor the way blocks.py applies it: transposed to (n, c, K), i.e. statistics per
    channel over all n * K rows (blocks.py:38,40,72)."""
    if train_bn:
        mu = y.mean(dim=(0, 1))
        var = y.var(dim=(0, 1), unbiased=False)
    else:
        mu, var = bn[prefix + ".running_mean"].to(y.dtype), bn[prefix + ".running_var"].to(y.dtype)
    return (y - mu) / torch.sqrt(var + eps) * bn[prefix + ".weight"].to(y.dtype) + bn[prefix + ".bias"].to(y.dtype)


def point_transformer_layer(p, x, o, state: dict, nsample: int, share_planes: int = 8, train_bn: bool = True, dtype=torch.float32):
    """blocks.PointTransformerLayer.forward (models/modules/cbl_point_transformer/blocks.py:31-44) as a pure function of the
    layer's ``state_dict``: p (n,3), x (n,c_in), o (b) -> (n, c).  kNN through the oracle's knnquery on the float32
    coordinates; everything after the gathers in ``dtype`` (float64 = the exact answer for the same neighbours)."""
    p32 = np.ascontiguousarray(p.detach().cpu().numpy(), dtype=np.float32)
    off = np.ascontiguousarray(o.detach().cpu().numpy(), dtype=np.int32)
    idx, _, _ = knnquery(int(nsample), p32, p32, off, off)
    idx = torch.from_numpy(np.ascontiguousarray(idx)).long()
    S = {k: v.detach().cpu().to(dtype) if v.is_floating_point() else v for k, v in state.items()}
    p, x = p.detach().cpu().to(dtype), x.detach().cpu().to(dtype)
    lin = lambda t, name: t @ S[name + ".weight"].t() + S[name + ".bias"]
    x_q, x_k, x_v = lin(x, "linear_q"), lin(x, "linear_k"), lin(x, "linear_v")                   # :33
    n, K = idx.shape
    p_r = p[idx.view(-1)].view(n, K, 3) - p.unsqueeze(1)                                         # queryandgroup use_xyz (:34,36)
    g_k, g_v = x_k[idx.view(-1)].view(n, K, -1), x_v[idx.view(-1)].view(n, K, -1)                # :34-35
    t = lin(p_r, "linear_p.0")                                                                   # :38  Linear(3,3)
    t = F.relu(_bn_rows(t, S, "linear_p.1", train_bn))
    p_r = lin(t, "linear_p.3")                                                                   # Linear(3,c)
    w = g_k - x_q.unsqueeze(1) + p_r                                                             # :39 (out_planes == mid_planes)
    w = F.relu(_bn_rows(w, S, "linear_w.0", train_bn))                                           # :40
    w = lin(w, "linear_w.2")
    w = F.relu(_bn_rows(w, S, "linear_w.3", train_bn))
    w = lin(w, "linear_w.5")
    w = torch.softmax(w, dim=1)                                                                  # :41 over the K neighbours
    c, s = g_v.shape[2], share_planes
    return ((g_v + p_r).view(n, K, s, c // s) * w.unsqueeze(2)).sum(1).view(n, c)                # :43


def transition_down(p, x, o, state: dict, stride: int, nsample: int, train_bn: bool = True, dtype=torch.float32):
    """blocks.TransitionDown.forward with stride != 1 (blocks.py:62-74): FPS to n // stride points per cloud, kNN grouping of
    [xyz_rel | feats], Linear (no bias) + BatchNorm + ReLU, max over the K neighbours -> (new_p, new_x, new_o)."""
    p32 = np.ascontiguousarray(p.detach().cpu().numpy(), dtype=np.float32)
    off = np.ascontiguousarray(o.detach().cpu().numpy(), dtype=np.int32)
    counts = np.diff(np.concatenate([[0], off])) // stride
    n_o = np.cumsum(counts).astype(np.int32)                                                     # :64-68
    sel = furthestsampling(p32, off, n_o)                                                        # :69
    n_p = p32[sel]
    idx, _, _ = knnquery(int(nsample), p32, n_p, off, n_o)                                       # :71
    idx = torch.from_numpy(np.ascontiguousarray(idx)).long()
    S = {k: v.detach().cpu().to(dtype) if v.is_floating_point() else v for k, v in state.items()}
    pd, xd, npd = p.detach().cpu().to(dtype), x.detach().cpu().to(dtype), torch.from_numpy(n_p).to(dtype)
    m, K = idx.shape
    g = torch.cat([pd[idx.view(-1)].view(m, K, 3) - npd.unsqueeze(1), xd[idx.view(-1)].view(m, K, -1)], -1)
    y = g @ S["linear.weight"].t()                                                               # :72
    y = F.relu(_bn_rows(y, S, "bn", train_bn))
    return torch.from_numpy(n_p), y.max(dim=1).values, torch.from_numpy(n_o)                     # :73 MaxPool1d(nsample)


# ----------------------------------------------------------------------------- clustering (SURVEY 8(f)-4)
def dbscan(points, eps: float = 0.03, min_samples: int = 30) -> Tuple[np.ndarray, np.ndarray]:
    """scikit-learn's DBSCAN(eps, min_samples).fit(points) -> (labels_, core_sample_indices_), the call of
    ops_utils.get_clustering_labels (ops_utils.py:98).  scikit-learn is a dependency of the reference that is not vendored in
    its tree (no version pinned there; this image has 1.9.0); its published algorithm, restated:
    sklearn/cluster/_dbscan.py -- neighbourhoods = radius_neighbors(eps) over a KDTree of the float64 copy of the points
    (reduced distance (dx^2 + dy^2) + dz^2 <= eps^2, the point itself included), core = at least min_samples neighbours;
    sklearn/cluster/_dbscan_inner.pyx -- visit points in index order, flood each unlabelled core point's component with a
    stack (non-core points are labelled but not expanded), label numbers in visiting order, the rest stays -1.
    Brute force, for test sizes."""
    x = np.asarray(points, dtype=np.float64)
    n = x.shape[0]
    d = x[:, None, :] - x[None, :, :]
    within = ((d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]) <= eps * eps
    core = within.sum(1) >= min_samples
    labels = np.full(n, -1, dtype=np.int64)
    label = 0
    for i in range(n):
        if labels[i] != -1 or not core[i]:
            continue
        stack = [i]
        while stack:
            v = stack.pop()
            if labels[v] != -1:
                continue
            labels[v] = label
            if core[v]:
                stack.extend(int(u) for u in np.flatnonzero(within[v]) if labels[u] == -1)
        label += 1
    return labels, np.flatnonzero(core).astype(np.int64)
