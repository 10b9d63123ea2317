"""Operator / module API of ``external_libs/pointnet2_utils/pointnet2_utils.py`` on
libtgn_b200.so.

Same public names, signatures, tensor layouts ((B,C,N) channel-first in and out) and
``state_dict`` keys (``mlp_convs.i``, ``mlp_bns.i``, ``conv_blocks.i.j``, ``bn_blocks.i.j``) as the
reference, so ``models/modules/{pointnet_pp,tsg_centroid_module,tsg_seg_module}.py`` and the
losses import it unchanged and checkpoints load.  What changes is underneath:

* FPS, ball query, 3-NN, gathers and transposes are hand-written sm_90a kernels (the reference
  runs ball query / 3-NN as dense torch ops with (S,N) matrices and full sorts);
* in inference (``module.eval()`` and no autograd) a set-abstraction level is ONE fused kernel
  per radius branch: gather -> [xyz_rel|feats] -> (conv1x1+BN+ReLU)* -> max over K, BatchNorm
  folded into the conv weights, nothing materialised (wgmma 3xTF32 engine, fp32 engine as
  fallback);
* when BatchNorm must use batch statistics (``module.training``) or gradients are needed, the
  grouped tensor is built by the CUDA gather (with its scatter-add backward) and the 1x1
  convolutions run through torch (cuBLAS/cuDNN) exactly as in the reference.

There is no CPU path.  Reference line numbers below refer to that file.
"""
from __future__ import annotations

import ctypes
from time import time
from typing import List, Optional, Sequence, Tuple

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F
from torch.autograd import Function

from . import _lib as L
from . import pointops

SA_FUSED_MAX_WIDTH = 128
SA_FUSED_MAX_LAYERS = 4
ENGINE_AUTO, ENGINE_FP32, ENGINE_TC, ENGINE_TCW, ENGINE_TC_HALF = 0, 1, 2, 3, 5     # TCW: wide layers (bf16x2); TC_HALF: engine 2 in half-size CTAs
_sa_engine = ENGINE_AUTO


def set_sa_engine(engine: int) -> None:
    """Select the engine of the fused set-abstraction kernel (0 auto, 1 fp32 CUDA cores, 2 3xTF32 tensor cores, 3 wide
    bf16x2 tensor cores, 5 engine 2 in half-size CTAs)."""
    global _sa_engine
    _sa_engine = int(engine)


def timeit(tag, t):
    print("{}: {}s".format(tag, time() - t))
    return time()


def pc_normalize(pc):
    """:12-18 (host-side numpy helper)."""
    pc = pc - np.mean(pc, axis=0)
    return pc / np.max(np.sqrt(np.sum(pc ** 2, axis=1)))


# ------------------------------------------------------------------------------------------ primitives
def _f32c(t: torch.Tensor) -> torch.Tensor:
    L.require_cuda(t)
    return t.contiguous() if t.dtype == torch.float32 else t.float().contiguous()


def transpose_last2(x: torch.Tensor) -> torch.Tensor:
    """(B, R, C) -> (B, C, R) contiguous through the tiled transpose kernel."""
    x = _f32c(x)
    B, R, C = x.shape
    out = torch.empty((B, C, R), dtype=torch.float32, device=x.device)
    L.call("tgn_transpose_cn", B, R, C, L.ptr(x), L.ptr(out), L.stream_ptr())
    return out


class _Transpose(Function):
    @staticmethod
    def forward(ctx, x):
        return transpose_last2(x)

    @staticmethod
    def backward(ctx, g):
        return transpose_last2(g)


def _transpose(x: torch.Tensor) -> torch.Tensor:
    return _Transpose.apply(x) if x.requires_grad else transpose_last2(x)


class _GatherRows(Function):
    """points (B,N,C), idx (B,M) int32 -> (B,M,C); backward = scatter-add."""

    @staticmethod
    def forward(ctx, points, idx):
        B, N, C = points.shape
        M = idx.shape[1]
        out = torch.empty((B, M, C), dtype=torch.float32, device=points.device)
        L.call("tgn_gather_rows", B, N, M, C, L.ptr(points), L.ptr(idx), L.ptr(out), L.stream_ptr())
        ctx.shape = (B, N, C)
        ctx.save_for_backward(idx)
        return out

    @staticmethod
    def backward(ctx, g):
        (idx,) = ctx.saved_tensors
        B, N, C = ctx.shape
        M = idx.shape[1]
        flat = (idx + (torch.arange(B, device=idx.device, dtype=torch.int32) * N).view(B, 1)).contiguous()
        gi = pointops.gather_backward(g.contiguous().view(B * M, C), flat, B * N)     # torch's index_put order (deterministic)
        return gi.view(B, N, C), None


def square_distance(src, dst):
    """:20-41.  (B,N,C),(B,M,C) -> (B,N,M) in the expanded form -2ab + |a|^2 + |b|^2.
    CUDA float32 3-D coordinates without autograd: one kernel with the reference's arithmetic (the rounding of |p|^2 follows
    the operands' layouts like torch's own reduction does, see ``_alt``) -- bit-identical to the torch formulation below,
    which stays for everything else (CPU tensors, other C, gradients: the losses differentiate through it)."""
    B, N, C = src.shape
    M = dst.shape[1]
    if (C == 3 and src.is_cuda and dst.is_cuda and src.dtype == torch.float32 and dst.dtype == torch.float32
            and N <= 65535 and B <= 65535 and not (torch.is_grad_enabled() and (src.requires_grad or dst.requires_grad))):
        order = _alt(src) | (_alt(dst) << 1)
        s, d = src.contiguous(), dst.contiguous()
        out = torch.empty((B, N, M), dtype=torch.float32, device=src.device)
        L.call("tgn_square_distance", B, N, M, L.ptr(s), L.ptr(d), L.ptr(out), order, L.stream_ptr())
        return out
    dist = -2 * torch.matmul(src, dst.permute(0, 2, 1))
    dist += torch.sum(src ** 2, -1).view(B, N, 1)
    dist += torch.sum(dst ** 2, -1).view(B, 1, M)
    return dist


def index_points(points, idx):
    """:44-61.  points (B,N,C), idx (B,S) or (B,S,K) integer -> (B,S[,K],C)."""
    pts = _f32c(points)
    B = pts.shape[0]
    flat = idx.reshape(B, -1).to(torch.int32).contiguous()
    out = _GatherRows.apply(pts, flat)
    return out.view(*idx.shape, pts.shape[-1])


def _take_rows(packed: torch.Tensor, rows: torch.Tensor) -> torch.Tensor:
    """packed (n,c) float32, rows (m,) int32 -> (m,c) through the gather kernel."""
    m, c = rows.shape[0], packed.shape[1]
    out = torch.empty((m, c), dtype=torch.float32, device=packed.device)
    L.call("tgn_grouping_forward", m, 1, c, L.ptr(packed), L.ptr(rows), L.ptr(out), L.stream_ptr())
    return out


_fps_mode = 0


def set_fps_mode(mode: int) -> None:
    """Default ``mode`` of tgn_furthestsampling for the pointnet2-side callers (0 = by batch size).
    A pipeline that keeps several chunks in flight passes -(10 + W) to pick the CTA shape that
    suits the clouds resident on the GPU rather than the clouds of one call."""
    global _fps_mode
    _fps_mode = int(mode)


def fps_mode_for_clouds_in_flight(clouds: int, n_points: int) -> int:
    """The bucket kernel's own rule (fps_bucket.cu: 16 / 8 / 4 warps per cloud at <= 2 / <= 4 / more
    clouds per SM), applied to a cloud count the caller knows better than a single call does."""
    if n_points <= 4096:
        return 0
    sms = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
    return -(10 + (4 if clouds > 4 * sms else (8 if clouds > 2 * sms else 16)))


def _fps_batched(xyz_t: torch.Tensor, npoint: int, mode: int = None) -> torch.Tensor:
    """xyz_t (B,N,3) contiguous -> GLOBAL int32 row ids (B*npoint,) of the packed (B*N,3) view."""
    if mode is None:
        mode = _fps_mode
    B, N, _ = xyz_t.shape
    dev = xyz_t.device
    offset = torch.arange(1, B + 1, device=dev, dtype=torch.int32) * N
    new_offset = torch.arange(1, B + 1, device=dev, dtype=torch.int32) * npoint
    return pointops.fps_packed(xyz_t.view(-1, 3), offset, new_offset, N, B * npoint, mode)


def farthest_point_sample(xyz, npoint):
    """:64-98.  xyz (B,N,3) -> per-cloud-local indices (B,npoint) int64; first sample = point 0."""
    xyz_t = _f32c(xyz)
    B, N, _ = xyz_t.shape
    gidx = _fps_batched(xyz_t, int(npoint)).view(B, npoint).long()
    return gidx - (torch.arange(B, device=xyz_t.device, dtype=torch.long) * N).view(B, 1)


def farthest_point_sample_np(xyz, npoint):
    """:103-118 samples a numpy cloud with a RANDOM start on whatever device the array lands on;
    the reference never calls it.  Here: same contract (numpy in, numpy out) on the GPU kernel
    with the deterministic start the live path uses."""
    t = torch.from_numpy(np.asarray(xyz, dtype=np.float32)).cuda()
    return farthest_point_sample(t, npoint).cpu().numpy()


def _radius_sq_f32(radius: float) -> float:
    """``sqrdists > radius ** 2`` compares against float32(radius**2) (:136; torch casts the
    python scalar to the tensor dtype)."""
    return float(np.float32(float(radius) ** 2))


BALL_AUTO, BALL_TILE, BALL_GRID = 0, 4, 8     # kernel choice bits of tgn_ball_query's idx64 argument


_ball_path = BALL_AUTO


def set_ball_path(path: int) -> None:
    """Default kernel choice of the ball query (BALL_AUTO / BALL_TILE / BALL_GRID); experiments."""
    global _ball_path
    _ball_path = int(path)


# ---- which torch arithmetic the neighbourhood searches reproduce ---------------------------------------------------
# square_distance (:38-40) adds torch.sum(p ** 2, -1) of both operands.  Measured with torch 2.11
# (scripts/diag_sumsq.py): on CUDA that sum rounds as (x*x + z*z) + y*y when the (..., 3) operand is
# CONTIGUOUS (vectorised reduce) and as (x*x + y*y) + z*z when it is a strided view -- and always the latter on the CPU.
# The reference's modules mix both: new_xyz fresh out of index_points is contiguous, xyz.permute(0, 2, 1) of the raw
# input is a view, the (B,3,S) coordinates a set-abstraction level returns are views that turn contiguous again when
# the next module permutes them back.  To return the reference's indices bit for bit the kernels take the rounding
# per operand, and the Python layer derives it from the layout the REFERENCE's call would see.
_reference_device = "cuda"


def set_reference_device(device: str) -> None:
    """"cuda" (default): reproduce the reference running on the GPU (layout-dependent |p|^2 rounding);
    "cpu": reproduce the reference's functions on CPU tensors (index-order rounding everywhere; the committed
    tests/golden/ref_torch_*.npz fixtures were generated that way)."""
    global _reference_device
    assert device in ("cuda", "cpu")
    _reference_device = device


def _alt(t: torch.Tensor) -> int:
    """1 when torch.sum(t ** 2, -1) of this (..., 3) tensor would take the contiguous-reduce rounding."""
    return 1 if (_reference_device == "cuda" and t.is_contiguous()) else 0


def _alt_fresh() -> int:
    """The same for a tensor fresh out of index_points (always contiguous)."""
    return 1 if _reference_device == "cuda" else 0


def _to_point_major(x: torch.Tensor) -> torch.Tensor:
    """(B,C,N) -> contiguous (B,N,C).  Free when x is the permuted view of a point-major tensor (what a
    set-abstraction level returns for the coordinates, here as in the reference); else the transpose kernel."""
    xt = x.permute(0, 2, 1)
    if xt.is_contiguous() and xt.dtype == torch.float32 and not x.requires_grad:
        return xt
    return _transpose(x)


def _ball_query(radius, nsample, xyz_t, new_xyz_t, idx64: bool, path: int = None, order: int = None) -> torch.Tensor:
    """``path``: BALL_AUTO lets the library pick per cloud (uniform grid for sparse balls on large
    clouds, index-order tile scan otherwise); BALL_TILE / BALL_GRID force one kernel (tests).
    ``order``: bit 0 / bit 1 = |new_xyz|^2 / |xyz|^2 in the contiguous-reduce rounding; default: what a
    set-abstraction level of the reference sees on its raw input (new_xyz contiguous, xyz a permuted view)."""
    B, N, _ = xyz_t.shape
    S = new_xyz_t.shape[1]
    if order is None:
        order = 1 if _reference_device == "cuda" else 0
    out = torch.empty((B, S, nsample), dtype=torch.int64 if idx64 else torch.int32, device=xyz_t.device)
    L.call("tgn_ball_query", B, N, S, ctypes.c_float(_radius_sq_f32(radius)), int(nsample), L.ptr(xyz_t), L.ptr(new_xyz_t),
           L.ptr(out), (1 if idx64 else 0) | int(_ball_path if path is None else path) | ((int(order) & 3) << 4), L.stream_ptr())
    return out


def query_ball_point(radius, nsample, xyz, new_xyz):
    """:120-144.  xyz (B,N,3), new_xyz (B,S,3) -> (B,S,nsample) int64: first nsample indices in
    ascending order inside the ball, padded with the first; N everywhere for an empty ball."""
    L.require_cuda(xyz, new_xyz)
    order = _alt(new_xyz) | (_alt(xyz) << 1)
    return _ball_query(radius, nsample, _f32c(xyz), _f32c(new_xyz), True, None, order)


def three_nn(xyz1, xyz2, order: int = None):
    """Top-3 of square_distance(xyz1, xyz2) (:333-335) without the matrix or the sort:
    (B,N,3),(B,S,3) -> dist (B,N,3) ascending, idx (B,N,3) int32.  ``order`` as in ``_ball_query`` (bit 0: xyz1,
    bit 1: xyz2); default: from the layouts of the tensors passed."""
    L.require_cuda(xyz1, xyz2)
    if order is None:
        order = _alt(xyz1) | (_alt(xyz2) << 1)
    x1, x2 = _f32c(xyz1), _f32c(xyz2)
    B, N, _ = x1.shape
    S = x2.shape[1]
    dist = torch.empty((B, N, 3), dtype=torch.float32, device=x1.device)
    idx = torch.empty((B, N, 3), dtype=torch.int32, device=x1.device)
    L.call("tgn_three_nn_ex", B, N, S, L.ptr(x1), L.ptr(x2), L.ptr(dist), L.ptr(idx), int(order) & 3, L.stream_ptr())
    return dist, idx


def three_interpolate(points2, dist, idx):
    """Inverse squared-distance interpolation (:337-340): points2 (B,S,C) -> (B,N,C).
    Differentiable wrt points2."""
    p2 = _f32c(points2)
    B, S, C = p2.shape
    N = idx.shape[1]
    if not (p2.requires_grad and torch.is_grad_enabled()):
        out = torch.empty((B, N, C), dtype=torch.float32, device=p2.device)
        L.call("tgn_three_interpolate_ex", B, N, S, C, L.ptr(p2), L.ptr(dist), L.ptr(idx), L.ptr(out),
               1 if _reference_device == "cuda" else 0, L.stream_ptr())
        return out
    rec = 1.0 / (dist + 1e-8)
    w = (rec / torch.sum(rec, dim=2, keepdim=True)).reshape(B * N, 3).contiguous()
    flat = (idx + (torch.arange(B, device=idx.device, dtype=torch.int32) * S).view(B, 1, 1)).reshape(B * N, 3).contiguous()
    # unfused products then (a0 + a1) + a2: torch.sum(index_points(points2, idx) * weight, dim=2) (:340)
    return pointops._WeightedGather.apply(p2.reshape(B * S, C), flat, w, "sum").view(B, N, C)


def sample_and_group(npoint, radius, nsample, xyz, points, returnfps=False):
    """:147-175.  xyz (B,N,3), points (B,N,D) -> new_xyz (B,S,3), new_points (B,S,K,3+D) with
    channel order [xyz_rel, feats]."""
    B, N, C = xyz.shape
    fps_idx = farthest_point_sample(xyz, npoint)
    new_xyz = index_points(xyz, fps_idx)
    idx = query_ball_point(radius, nsample, xyz, new_xyz)
    grouped_xyz = index_points(xyz, idx)
    grouped_xyz_norm = grouped_xyz - new_xyz.view(B, npoint, 1, C)
    if points is not None:
        new_points = torch.cat([grouped_xyz_norm, index_points(points, idx)], dim=-1)
    else:
        new_points = grouped_xyz_norm
    if returnfps:
        return new_xyz, new_points, grouped_xyz, fps_idx
    return new_xyz, new_points


def sample_and_group_all(xyz, points):
    """:178-195.  One group holding the whole cloud; new_xyz is the origin."""
    B, N, C = xyz.shape
    new_xyz = torch.zeros(B, 1, C, device=xyz.device, dtype=xyz.dtype)
    grouped_xyz = xyz.view(B, 1, N, C)
    if points is not None:
        return new_xyz, torch.cat([grouped_xyz, points.view(B, 1, N, -1)], dim=-1)
    return new_xyz, grouped_xyz


# ------------------------------------------------------------------------------------------ fused SA body
class _FoldedMlp:
    """conv1x1 + eval-mode BatchNorm folded to (W', b') per layer, cached until a parameter or
    running statistic changes (tensor ``_version`` counters)."""

    def __init__(self):
        self.key = None
        self.weights: List[torch.Tensor] = []
        self.biases: List[torch.Tensor] = []
        self.channels: List[int] = []
        self.w_ptrs = None
        self.b_ptrs = None
        self.event = None
        self.stream = None
        self._previous = None

    def update(self, convs, bns) -> "_FoldedMlp":
        key = tuple((c.weight._version, c.weight.data_ptr(), None if c.bias is None else c.bias._version,
                     b.weight._version, b.bias._version, b.running_mean._version, b.running_var._version, b.running_mean.data_ptr())
                    for c, b in zip(convs, bns))
        on_gpu = convs[0].weight.is_cuda
        cur = torch.cuda.current_stream() if on_gpu else None
        if key == self.key:
            if self.stream is not None and cur != self.stream:
                # folded on another stream (e.g. HostPipeline's second compute stream): order this consumer after the
                # fold and tell the caching allocator about the extra reader
                cur.wait_event(self.event)
                for t in self.weights + self.biases:
                    t.record_stream(cur)
            return self
        self._previous = (self.weights, self.biases)      # a launch queued on another stream may still read them
        self.weights, self.biases, self.channels = [], [], []
        with torch.no_grad():
            for c, b in zip(convs, bns):
                w = c.weight.reshape(c.weight.shape[0], -1).float()
                cb = c.bias.float() if c.bias is not None else torch.zeros(w.shape[0], device=w.device)
                scale = b.weight.float() / torch.sqrt(b.running_var.float() + b.eps)
                self.weights.append((w * scale[:, None]).contiguous())
                self.biases.append(((cb - b.running_mean.float()) * scale + b.bias.float()).contiguous())
                if not self.channels:
                    self.channels.append(w.shape[1])
                self.channels.append(w.shape[0])
        n = len(self.weights)
        self.w_ptrs = (ctypes.c_void_p * n)(*[w.data_ptr() for w in self.weights])
        self.b_ptrs = (ctypes.c_void_p * n)(*[b.data_ptr() for b in self.biases])
        self.key = key
        if on_gpu:
            self.event = torch.cuda.Event()
            self.event.record(cur)
            self.stream = cur
        return self


SA_FUSED_AUTO_MAX_WIDTH = 64      # widest layer of the 3xTF32 single-kernel engine (~2^-21 per product)


def fused_supported(channels: Sequence[int]) -> bool:
    """Shapes the single-kernel (eval-mode BatchNorm) engines take.  On the automatic path only the fp32-grade
    ones are used (3xTF32 tensor cores up to 64 channels, else the layer-per-launch chain of csrc/pw_mlp.cu with
    three-part operands): the wide bf16x2 engine (ENGINE_TCW, ~1e-5 norm-wise) misses the ELEMENT-WISE 1e-4 bound on
    small activations (measured 4e-4 at a 1 % floor, tests/test_gpu_reference_live.py) and is kept for explicit use."""
    widest = SA_FUSED_MAX_WIDTH if _sa_engine != ENGINE_AUTO else SA_FUSED_AUTO_MAX_WIDTH
    return 1 <= len(channels) - 1 <= SA_FUSED_MAX_LAYERS and max(channels) <= widest


def sa_group_mlp_max(xyz_t, feats_t, new_xyz_t, group_idx, xyz_first: bool, folded: _FoldedMlp, out, c_offset: int,
                     engine: Optional[int] = None) -> None:
    """Launch the fused gather -> MLP -> max kernel for one radius branch, writing channels
    [c_offset, c_offset + C_last) of ``out`` (B, C_total, S)."""
    B, N, _ = xyz_t.shape
    S, K = group_idx.shape[1], group_idx.shape[2]
    D = 0 if feats_t is None else feats_t.shape[2]
    ch = (ctypes.c_int * len(folded.channels))(*folded.channels)
    L.call("tgn_sa_group_mlp_max", B, N, S, K, D, L.ptr(xyz_t), L.ptr(feats_t), L.ptr(new_xyz_t), L.ptr(group_idx),
           1 if xyz_first else 0, len(folded.weights), ctypes.cast(ch, ctypes.c_void_p), ctypes.cast(folded.w_ptrs, ctypes.c_void_p),
           ctypes.cast(folded.b_ptrs, ctypes.c_void_p), L.ptr(out), out.shape[1], int(c_offset),
           _sa_engine if engine is None else int(engine), L.stream_ptr())


# ------------------------------------------------------------------------------------------ conv1x1 + BatchNorm chains (any width, any BN mode)
class _PwChain:
    """Launch plan of a [conv1x1 -> BatchNorm -> ReLU]* chain on the tensor-core layer kernel (csrc/pw_mlp.cu):
    one launch per layer, BatchNorm of layer l applied while layer l+1 builds its operand, batch statistics
    (training mode -- what every reference call site runs, inference included) accumulated in fp64 by the
    producing launch, running statistics updated in-kernel like torch does.  Packed bf16 hi/lo weights are
    cached per parameter version."""

    def __init__(self):
        self._packed = {}

    def packed(self, conv) -> torch.Tensor:
        w = conv.weight
        key = (w.data_ptr(), w._version, w.device)
        hit = self._packed.get(id(conv))
        if hit is not None and hit[0] == key:
            return hit[1]
        cout, cin = w.shape[0], w.shape[1]
        w2 = w.detach().reshape(cout, cin).float().contiguous()
        buf = torch.empty(L.load().tgn_pw_packed_bytes(cout, cin), dtype=torch.uint8, device=w.device)
        L.call("tgn_pw_pack_weights", cout, cin, L.ptr(w2), L.ptr(buf), L.stream_ptr())
        ev = torch.cuda.Event()
        ev.record()
        self._packed[id(conv)] = (key, buf, ev, torch.cuda.current_stream())
        return buf

    def wait_packed(self, conv) -> None:
        """A cached pack may have been produced on another stream (ADVICE r1: stream-aware caches)."""
        hit = self._packed.get(id(conv))
        if hit is not None and hit[3] != torch.cuda.current_stream():
            torch.cuda.current_stream().wait_event(hit[2])
            hit[1].record_stream(torch.cuda.current_stream())

    @staticmethod
    def supported(convs, bns) -> bool:
        for c, b in zip(convs, bns):
            if b.training and b.track_running_stats and b.momentum is None:
                return False                  # cumulative moving average: left to torch
            if c.weight.dtype != torch.float32 or (b.weight is not None and b.weight.dtype != torch.float32):
                return False
        return len(convs) >= 1

    @staticmethod
    def _bn_mode(bn) -> int:
        """1 = batch statistics, 2 = running statistics (torch: training or no tracked statistics -> batch)."""
        return 1 if (bn.training or bn.running_mean is None) else 2

    @staticmethod
    def _fill_in_bn(desc: "L.PwLayer", bn, stats_prev) -> None:
        mode = _PwChain._bn_mode(bn)
        desc.in_affine = mode
        desc.in_stats = L.ptr(stats_prev) if mode == 1 else None
        desc.in_gamma, desc.in_beta = L.ptr(bn.weight), L.ptr(bn.bias)
        desc.in_running_mean, desc.in_running_var = L.ptr(bn.running_mean), L.ptr(bn.running_var)
        desc.in_eps = float(bn.eps)
        desc.in_momentum = float(bn.momentum if bn.momentum is not None else 0.0)
        desc.in_update_running = 1 if (mode == 1 and bn.training and bn.running_mean is not None) else 0

    def run(self, convs, bns, first: "L.PwLayer", rows: int, out: torch.Tensor, out_c_offset: int, rows_per_batch_out: int,
            group: int = 0, slopes: Optional[Sequence[float]] = None, relu: bool = True, up: Optional[tuple] = None,
            promote: bool = False, residual: Optional[torch.Tensor] = None) -> None:
        """``first`` describes the operand source of layer 0 (mode / segments / gather fields filled by the
        caller).  group > 0: the last layer reduces max/min over ``group`` consecutive rows (set abstraction)
        and ``out`` is (B, C_total, rows/group/B...); group == 0: ``out`` receives every row (feature propagation).
        ``slopes``: LeakyReLU(slopes[l]) follows BatchNorm l instead of ReLU (DGCNN); None leaves every ReLU launch as it was.
        ``relu=False``: the last BatchNorm is followed by no activation (PointNet's encoder conv3); ``slopes`` takes precedence.
        ``up=(f, idx, w)``: the last BatchNorm goes through ``tgn_pt_up_apply`` instead, ``out`` is (rows, C) row-major and, unless
        f is None, receives the k = 3 interpolation of f (TransitionUp, blocks.py:110) added to each row.
        ``promote=True``: each layer whose own BatchNorm uses running statistics runs the promoted-accumulation kernel
        (``accum`` = 1: 128-row tiles, the tensor-core accumulator rounded to nearest into an fp32 total every 16 values of K);
        layers on batch statistics launch exactly as with False.
        ``residual``: the last BatchNorm goes through ``tgn_pt_res_apply``, ``out`` is (rows, C) row-major and receives
        relu(bn(y) + residual) with the BatchNorm value rounded first (PointTransformerBlock, blocks.py:132-134); residual is a
        (rows, C) matrix with unit channel stride."""
        dev = out.device
        n = len(convs)
        couts = [c.weight.shape[0] for c in convs]
        train = [self._bn_mode(b) == 1 for b in bns]
        stats = [torch.zeros(2 * co, dtype=torch.float64, device=dev) if t else None for co, t in zip(couts, train)]
        prev_y = None
        st = L.stream_ptr()
        keep = []
        for l, (conv, bn) in enumerate(zip(convs, bns)):
            cout, cin = conv.weight.shape[0], conv.weight.shape[1]
            d = first if l == 0 else L.PwLayer()
            d.rows, d.cin, d.cout = rows, cin, cout
            if l > 0:
                d.mode = 0
                d.rows_per_batch = rows
                d.seg_ptr[0], d.seg_channels[0] = L.ptr(prev_y), cin
                d.seg_batch_stride[0], d.seg_row_stride[0], d.seg_chan_stride[0] = 0, 1, rows
                d.seg_channels[1] = 0
                self._fill_in_bn(d, bns[l - 1], stats[l - 1])
                if slopes is not None:
                    d.in_act, d.in_act_slope = 1, float(slopes[l - 1])
            packed = self.packed(conv)
            self.wait_packed(conv)
            d.w_packed = L.ptr(packed)
            bias = None if conv.bias is None else conv.bias.detach()
            d.bias = L.ptr(bias)
            d.stats = L.ptr(stats[l])
            d.accum = 1 if (promote and not train[l]) else 0
            last = l == n - 1
            if last and group > 0:
                ng = rows // group
                ymax = torch.empty((cout, ng), dtype=torch.float32, device=dev)
                ymin = torch.empty((cout, ng), dtype=torch.float32, device=dev)
                atomic = 1 if ((64 if d.accum else 128) % group) != 0 else 0      # half a tile of rows per epilogue thread
                if atomic:
                    L.call("tgn_pw_fill", L.ptr(ymax), ymax.numel(), ctypes.c_float(float("-inf")), st)
                    L.call("tgn_pw_fill", L.ptr(ymin), ymin.numel(), ctypes.c_float(float("inf")), st)
                d.y, d.ymax, d.ymin, d.group, d.extrema_atomic = None, L.ptr(ymax), L.ptr(ymin), group, atomic
                keep += [ymax, ymin]
            else:
                y = torch.empty((cout, rows), dtype=torch.float32, device=dev)
                d.y, d.ymax, d.ymin, d.group, d.extrema_atomic = L.ptr(y), None, None, 0, 0
                prev_y = y
                keep.append(y)
            L.call("tgn_pw_layer_forward", ctypes.byref(d), st)
        bn = bns[-1]
        a = L.PwApply()
        mode = self._bn_mode(bn)
        if group > 0:
            a.rows, a.src, a.ymin = rows // group, L.ptr(keep[-2]), L.ptr(keep[-1])
        else:
            a.rows, a.src, a.ymin = rows, L.ptr(prev_y), None
        a.rows_per_batch, a.channels, a.out_channels, a.out_c_offset, a.relu = rows_per_batch_out, couts[-1], out.shape[1], out_c_offset, int(relu)
        a.out = L.ptr(out)
        a.affine, a.stats, a.stat_rows = mode, L.ptr(stats[-1]), rows
        a.gamma, a.beta = L.ptr(bn.weight), L.ptr(bn.bias)
        a.running_mean, a.running_var = L.ptr(bn.running_mean), L.ptr(bn.running_var)
        a.eps, a.momentum = float(bn.eps), float(bn.momentum if bn.momentum is not None else 0.0)
        a.update_running = 1 if (mode == 1 and bn.training and bn.running_mean is not None) else 0
        if slopes is not None:
            a.act, a.act_slope = 1, float(slopes[-1])
        if residual is not None:
            r = L.PtResApply()
            r.apply, r.identity, r.identity_row_stride = a, L.ptr(residual), residual.stride(0)
            L.call("tgn_pt_res_apply", ctypes.byref(r), st)
        elif up is None:
            L.call("tgn_pw_apply", ctypes.byref(a), st)
        else:
            u = L.PtUpApply()
            u.apply = a
            f, idx, w = up
            u.f, u.idx, u.w, u.f_rows = L.ptr(f), L.ptr(idx), L.ptr(w), 0 if f is None else f.shape[0]
            L.call("tgn_pt_up_apply", ctypes.byref(u), st)
        for b in bns:
            if b.training and b.num_batches_tracked is not None:
                b.num_batches_tracked.add_(1)


class _ColumnSlice:
    """conv's weight columns [lo, hi), with conv's bias, for the packed-weight cache of ``_PwChain`` (keyed by this object): a
    layer whose other input columns are constant over each cloud and are added as a per-cloud bias instead"""

    def __init__(self, conv, lo: int, hi: Optional[int] = None):
        self.conv, self.lo, self.hi, self.bias = conv, lo, hi, conv.bias

    @property
    def weight(self) -> torch.Tensor:
        return self.conv.weight[:, self.lo:self.hi]


def _pw_set_abstraction(chain: _PwChain, convs, bns, xyz_t, feats_t, new_xyz_t, gidx, xyz_first: bool, out, c_offset: int) -> None:
    """Set-abstraction branch on the layer kernel: layer 0 gathers [xyz_rel | feats] / [feats | xyz_rel] itself, the
    last layer keeps only the max / min over each neighbourhood."""
    B, N, _ = xyz_t.shape
    S, K = gidx.shape[1], gidx.shape[2]
    d = L.PwLayer()
    d.mode = 1
    d.rows_per_batch = S * K
    d.xyz, d.feats, d.new_xyz, d.gidx = L.ptr(xyz_t), L.ptr(feats_t), L.ptr(new_xyz_t), L.ptr(gidx)
    d.N, d.S, d.K, d.D, d.xyz_first = N, S, K, 0 if feats_t is None else feats_t.shape[2], 1 if xyz_first else 0
    d.in_affine = 0
    d.seg_channels[0] = d.seg_channels[1] = 0
    chain.run(convs, bns, d, B * S * K, out, c_offset, S, group=K)


_pw_enabled = True


def set_pw_enabled(flag: bool) -> None:
    """Experiments / tests: False sends training-mode and wide chains back to torch's conv + BatchNorm."""
    global _pw_enabled
    _pw_enabled = bool(flag)


def _wants_grad(module: nn.Module, *tensors) -> bool:
    if not torch.is_grad_enabled():
        return False
    if any(t is not None and t.requires_grad for t in tensors):
        return True
    return any(p.requires_grad for p in module.parameters())


class _fp32_convs:
    """The library 1x1 convolutions of the autograd path run in IEEE fp32: torch's default lets cuDNN use
    TF32 (1e-3 relative), which would break the 1e-4 parity bound (SURVEY.md 7.1).  Only the TF32 switch is
    touched; the user's cudnn.enabled / benchmark / deterministic settings stay as they are."""

    def __enter__(self):
        self.saved = torch.backends.cudnn.allow_tf32
        torch.backends.cudnn.allow_tf32 = False

    def __exit__(self, *exc):
        torch.backends.cudnn.allow_tf32 = self.saved


def _mlp_unfused(grouped: torch.Tensor, convs, bns) -> torch.Tensor:
    """grouped (B,S,K,C) -> (B,C_out,S): the reference's permute + conv/BN/ReLU + max (:227-237)."""
    h = grouped.permute(0, 3, 2, 1)
    with _fp32_convs():
        for conv, bn in zip(convs, bns):
            h = F.relu(bn(conv(h)))
    return torch.max(h, 2)[0]


class PointNetSetAbstraction(nn.Module):
    """:198-239.  Single-scale set abstraction; group channel order [xyz_rel, feats]."""

    def __init__(self, npoint, radius, nsample, in_channel, mlp, group_all):
        super().__init__()
        self.npoint, self.radius, self.nsample, self.group_all = npoint, radius, nsample, group_all
        self.mlp_convs = nn.ModuleList()
        self.mlp_bns = nn.ModuleList()
        last = in_channel
        for width in mlp:
            self.mlp_convs.append(nn.Conv2d(last, width, 1))
            self.mlp_bns.append(nn.BatchNorm2d(width))
            last = width
        self._folded = _FoldedMlp()
        self._pw = _PwChain()

    def _fusable(self, xyz, points) -> bool:
        """Single-kernel engines: folded eval-mode BatchNorm, widths <= 128."""
        chans = [self.mlp_convs[0].in_channels] + [c.out_channels for c in self.mlp_convs]
        return (not any(b.training for b in self.mlp_bns)) and fused_supported(chans) and not _wants_grad(self, xyz, points)

    def _pw_ok(self, xyz, points) -> bool:
        """Layer-per-launch tensor-core chain: any width, batch-statistics or running-statistics BatchNorm, no autograd."""
        return _pw_enabled and _PwChain.supported(self.mlp_convs, self.mlp_bns) and not _wants_grad(self, xyz, points)

    def forward(self, xyz, points):
        """xyz (B,3,N), points (B,D,N) or None -> new_xyz (B,3,S), new_points (B,C_out,S)."""
        L.require_cuda(xyz, points)
        order = _alt_fresh() | (_alt(xyz.permute(0, 2, 1)) << 1)   # new_xyz (index_points output) contiguous; xyz as the reference sees it
        xyz_t = _to_point_major(xyz)                              # (B,N,3)
        feats_t = None if points is None else _transpose(points)  # (B,N,D)
        B, N, _ = xyz_t.shape
        if self._fusable(xyz, points):
            folded = self._folded.update(self.mlp_convs, self.mlp_bns)
            if self.group_all:
                S, K = 1, N
                new_xyz_t = torch.zeros((B, 1, 3), dtype=torch.float32, device=xyz_t.device)
                gidx = torch.arange(N, device=xyz_t.device, dtype=torch.int32).view(1, 1, N).expand(B, 1, N).contiguous()
            else:
                S, K = self.npoint, self.nsample
                fps = _fps_batched(xyz_t, S)
                new_xyz_t = _take_rows(xyz_t.view(-1, 3), fps).view(B, S, 3)
                gidx = _ball_query(self.radius, K, xyz_t, new_xyz_t, False, None, order)
            out = torch.empty((B, folded.channels[-1], S), dtype=torch.float32, device=xyz_t.device)
            sa_group_mlp_max(xyz_t, feats_t, new_xyz_t, gidx, True, folded, out, 0)
            return new_xyz_t.permute(0, 2, 1), out
        if self._pw_ok(xyz, points):
            if self.group_all:
                S, K = 1, N
                new_xyz_t = torch.zeros((B, 1, 3), dtype=torch.float32, device=xyz_t.device)
                gidx = torch.arange(N, device=xyz_t.device, dtype=torch.int32).view(1, 1, N).expand(B, 1, N).contiguous()
            else:
                S, K = self.npoint, self.nsample
                fps = _fps_batched(xyz_t, S)
                new_xyz_t = _take_rows(xyz_t.view(-1, 3), fps).view(B, S, 3)
                gidx = _ball_query(self.radius, K, xyz_t, new_xyz_t, False, None, order)
            out = torch.empty((B, self.mlp_convs[-1].out_channels, S), dtype=torch.float32, device=xyz_t.device)
            _pw_set_abstraction(self._pw, self.mlp_convs, self.mlp_bns, xyz_t, feats_t, new_xyz_t, gidx, True, out, 0)
            return new_xyz_t.permute(0, 2, 1), out
        if self.group_all:
            new_xyz_t, grouped = sample_and_group_all(xyz_t, feats_t)
        else:
            # the reference's own call, on the layout the reference passes (its |p|^2 rounding follows the layout)
            new_xyz_t, grouped = sample_and_group(self.npoint, self.radius, self.nsample, xyz.permute(0, 2, 1), feats_t)
        return new_xyz_t.permute(0, 2, 1), _mlp_unfused(grouped, self.mlp_convs, self.mlp_bns)


class PointNetSetAbstractionMsg(nn.Module):
    """:242-299.  Multi-scale grouping: one FPS, per radius a ball query + MLP + max, branches
    concatenated on the channel axis; group channel order [feats, xyz_rel] (:285)."""

    def __init__(self, npoint, radius_list, nsample_list, in_channel, mlp_list):
        super().__init__()
        self.npoint, self.radius_list, self.nsample_list = npoint, radius_list, nsample_list
        self.conv_blocks = nn.ModuleList()
        self.bn_blocks = nn.ModuleList()
        for widths in mlp_list:
            convs, bns = nn.ModuleList(), nn.ModuleList()
            last = in_channel + 3
            for width in widths:
                convs.append(nn.Conv2d(last, width, 1))
                bns.append(nn.BatchNorm2d(width))
                last = width
            self.conv_blocks.append(convs)
            self.bn_blocks.append(bns)
        self._folded = [_FoldedMlp() for _ in mlp_list]
        self._pw = [_PwChain() for _ in mlp_list]

    def _fusable(self, xyz, points) -> bool:
        if any(b.training for bns in self.bn_blocks for b in bns) or _wants_grad(self, xyz, points):
            return False
        return all(fused_supported([convs[0].in_channels] + [c.out_channels for c in convs]) for convs in self.conv_blocks)

    def _pw_ok(self, xyz, points) -> bool:
        return (_pw_enabled and all(_PwChain.supported(c, b) for c, b in zip(self.conv_blocks, self.bn_blocks))
                and not _wants_grad(self, xyz, points))

    def forward(self, xyz, points):
        L.require_cuda(xyz, points)
        order = _alt_fresh() | (_alt(xyz.permute(0, 2, 1)) << 1)
        xyz_t = _to_point_major(xyz)
        feats_t = None if points is None else _transpose(points)
        B, N, _ = xyz_t.shape
        S = self.npoint
        if self._fusable(xyz, points):
            fps = _fps_batched(xyz_t, S)
            new_xyz_t = _take_rows(xyz_t.view(-1, 3), fps).view(B, S, 3)
            folded = [f.update(c, b) for f, c, b in zip(self._folded, self.conv_blocks, self.bn_blocks)]
            out = torch.empty((B, sum(f.channels[-1] for f in folded), S), dtype=torch.float32, device=xyz_t.device)
            c_off = 0
            for radius, K, f in zip(self.radius_list, self.nsample_list, folded):
                gidx = _ball_query(radius, K, xyz_t, new_xyz_t, False, None, order)
                sa_group_mlp_max(xyz_t, feats_t, new_xyz_t, gidx, False, f, out, c_off)
                c_off += f.channels[-1]
            return new_xyz_t.permute(0, 2, 1), out
        if self._pw_ok(xyz, points):
            fps = _fps_batched(xyz_t, S)
            new_xyz_t = _take_rows(xyz_t.view(-1, 3), fps).view(B, S, 3)
            out = torch.empty((B, sum(convs[-1].out_channels for convs in self.conv_blocks), S), dtype=torch.float32, device=xyz_t.device)
            c_off = 0
            for i, (radius, K) in enumerate(zip(self.radius_list, self.nsample_list)):
                gidx = _ball_query(radius, K, xyz_t, new_xyz_t, False, None, order)
                _pw_set_abstraction(self._pw[i], self.conv_blocks[i], self.bn_blocks[i], xyz_t, feats_t, new_xyz_t, gidx, False, out, c_off)
                c_off += self.conv_blocks[i][-1].out_channels
            return new_xyz_t.permute(0, 2, 1), out
        new_xyz_t = index_points(xyz_t, farthest_point_sample(xyz_t, S))
        outs = []
        for i, radius in enumerate(self.radius_list):
            K = self.nsample_list[i]
            gidx = _ball_query(radius, K, xyz_t, new_xyz_t, True, None, order)
            grouped = index_points(xyz_t, gidx) - new_xyz_t.view(B, S, 1, 3)
            if feats_t is not None:
                grouped = torch.cat([index_points(feats_t, gidx), grouped], dim=-1)
            outs.append(_mlp_unfused(grouped, self.conv_blocks[i], self.bn_blocks[i]))
        return new_xyz_t.permute(0, 2, 1), torch.cat(outs, dim=1)


class PointNetFeaturePropagation(nn.Module):
    """:302-352.  3-NN inverse squared-distance interpolation + skip concat + conv1x1/BN/ReLU."""

    def __init__(self, in_channel, mlp):
        super().__init__()
        self.mlp_convs = nn.ModuleList()
        self.mlp_bns = nn.ModuleList()
        last = in_channel
        for width in mlp:
            self.mlp_convs.append(nn.Conv1d(last, width, 1))
            self.mlp_bns.append(nn.BatchNorm1d(width))
            last = width
        self._pw = _PwChain()

    def forward(self, xyz1, xyz2, points1, points2):
        """xyz1 (B,3,N) fine, xyz2 (B,3,S) coarse, points1 (B,D1,N) or None, points2 (B,D2,S)
        -> (B,D',N)."""
        L.require_cuda(xyz1, xyz2, points1, points2)
        nn_order = _alt(xyz1.permute(0, 2, 1)) | (_alt(xyz2.permute(0, 2, 1)) << 1)     # layouts as the reference's square_distance sees them (:330-333)
        x1, x2 = _to_point_major(xyz1), _to_point_major(xyz2)
        p2 = _transpose(points2)                                   # (B,S,D2)
        B, N, _ = x1.shape
        S = x2.shape[1]
        if (_pw_enabled and _PwChain.supported(self.mlp_convs, self.mlp_bns)
                and not _wants_grad(self, xyz1, xyz2, points1, points2)):
            # tensor-core chain: layer 0 reads [points1 (channel-first) | interpolated (point-major)] in place
            if S == 1:
                interp, strides = p2, (p2.shape[2], 0, 1)                      # (B,1,D2): every fine point gets the one coarse row
            else:
                dist, idx = three_nn(x1, x2, nn_order)
                interp = three_interpolate(p2, dist, idx)                       # (B,N,D2)
                strides = (N * interp.shape[2], interp.shape[2], 1)
            d = L.PwLayer()
            d.mode, d.rows_per_batch = 0, N
            D2 = interp.shape[2]
            if points1 is not None:
                p1 = _f32c(points1)
                D1 = p1.shape[1]
                d.seg_ptr[0], d.seg_channels[0] = L.ptr(p1), D1
                d.seg_batch_stride[0], d.seg_row_stride[0], d.seg_chan_stride[0] = D1 * N, 1, N
                d.seg_ptr[1], d.seg_channels[1] = L.ptr(interp), D2
                d.seg_batch_stride[1], d.seg_row_stride[1], d.seg_chan_stride[1] = strides
            else:
                d.seg_ptr[0], d.seg_channels[0] = L.ptr(interp), D2
                d.seg_batch_stride[0], d.seg_row_stride[0], d.seg_chan_stride[0] = strides
                d.seg_channels[1] = 0
            d.in_affine = 0
            out = torch.empty((B, self.mlp_convs[-1].out_channels, N), dtype=torch.float32, device=x1.device)
            self._pw.run(self.mlp_convs, self.mlp_bns, d, B * N, out, 0, N, group=0)
            return out
        if S == 1:
            interp = p2.repeat(1, N, 1)
        else:
            dist, idx = three_nn(x1, x2, nn_order)
            interp = three_interpolate(p2, dist, idx)             # (B,N,D2)
        h = _transpose(interp)                                     # (B,D2,N)
        if points1 is not None:
            h = torch.cat([points1, h], dim=1)
        with _fp32_convs():
            for conv, bn in zip(self.mlp_convs, self.mlp_bns):
                h = F.relu(bn(conv(h)))
        return h
