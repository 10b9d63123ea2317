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

With ``accelerate`` alone, ``get_graph_feature``, the convolutions and BatchNorm stay the reference's.  The indices carry no
gradient, so autograd and training see the same graph.

The no-grad forward of the whole model (DESIGN §3.12) runs on the tensor-core layer chain of csrc/pw_mlp.cu:

* ``forward(module, x_in)`` -- ``DGCnnModule.forward`` (models/modules/dgcnn.py:96-134) without the (B, 2C, N, k) edge tensors;
* ``fusable(module, x_in)`` -- whether ``forward`` takes the call;
* ``eval_fusable(module, x_in)`` -- the same, with BatchNorms on running statistics (eval mode) allowed too;
* ``accelerate_forward(module_or_class, running_stats=False)`` -- wraps ``DGCnnModule.forward``; under autograd the reference's
  own code runs, and eval-mode calls only reach ``forward`` with ``running_stats=True``.
"""
from __future__ import annotations

import functools
import operator
import weakref
from typing import Callable, Optional, Sequence

import torch
from torch import nn

from . import _lib as L
from . import pointnet2_utils as pn2

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


# ------------------------------------------------------------------------------------------ the no-grad forward of DGCnnModule
_EDGE_CONVS = (("conv1", "conv2"), ("conv3", "conv4"), ("conv5",))      # one EdgeConv per get_graph_feature call (:102-114)
_LAYERS = ("conv1", "conv2", "conv3", "conv4", "conv5", "conv6", "conv7", "conv8")


def _layer_ok(seq, cin: int) -> bool:
    """nn.Sequential(Conv{1,2}d(cin, cout, kernel_size=1, bias=False), BatchNorm{1,2}d(cout), LeakyReLU(slope)) in float32."""
    if not isinstance(seq, nn.Sequential) or len(seq) != 3:
        return False
    conv, bn, act = seq[0], seq[1], seq[2]
    if type(conv) not in (nn.Conv1d, nn.Conv2d) or type(bn) not in (nn.BatchNorm1d, nn.BatchNorm2d) or type(act) is not nn.LeakyReLU:
        return False
    n = len(conv.kernel_size)
    if (conv.kernel_size != (1,) * n or conv.stride != (1,) * n or conv.dilation != (1,) * n or conv.padding not in ((0,) * n, "valid")
            or conv.groups != 1 or conv.bias is not None or conv.padding_mode != "zeros" or conv.in_channels != cin):
        return False
    if conv.weight.dtype != torch.float32 or bn.num_features != conv.out_channels:
        return False
    if not bn.affine or bn.weight.dtype != torch.float32 or bn.momentum is None:
        return False
    return bn.running_mean is None or bn.running_mean.dtype == torch.float32


def structure_ok(module) -> bool:
    """The layer structure of the reference's DGCnnModule (:54-91), whatever the widths: three EdgeConvs whose features stay within
    the kNN kernel's C <= 64, conv6 over their concatenation, conv7 over [its max | the concatenation], conv8, dp1, cls_conv."""
    try:
        seqs = {name: getattr(module, name) for name in _LAYERS}
        c_in = seqs["conv1"][0].in_channels // 2
        w = [seqs[n][0].out_channels for n in ("conv2", "conv4", "conv5")]
        cins = {"conv1": 2 * c_in, "conv2": seqs["conv1"][0].out_channels, "conv3": 2 * w[0], "conv4": seqs["conv3"][0].out_channels,
                "conv5": 2 * w[1], "conv6": sum(w), "conv7": seqs["conv6"][0].out_channels + sum(w),
                "conv8": seqs["conv7"][0].out_channels}
        cls = module.cls_conv
        _ = module.dp1, module.k
    except (AttributeError, TypeError, IndexError):
        return False
    if not all(_layer_ok(seqs[n], cins[n]) for n in _LAYERS):
        return False
    if not all(1 <= c <= MAX_C for c in w):
        return False
    return isinstance(cls, nn.Conv1d) and cls.in_channels == seqs["conv8"][0].out_channels


def input_ok(is_cuda: bool, dtype: torch.dtype, shape: Sequence[int], k: int, c_in: int, training: bool) -> bool:
    """A CUDA float32 (B, C_in, N) input with C_in <= 64 and N >= k, 1 <= k <= 32; in training mode BatchNorm needs two values."""
    if not is_cuda or dtype != torch.float32 or len(shape) != 3:
        return False
    B, C, N = shape
    if C != c_in or not 1 <= C <= MAX_C or not isinstance(k, int) or not 1 <= k <= MAX_K or N < k or B < 1:
        return False
    return not training or B * N > 1


def _needs_grad(module, x) -> bool:
    if not torch.is_grad_enabled():
        return False
    return x.requires_grad or any(p.requires_grad for p in module.parameters())


def fusable(module, x_in) -> bool:
    """True when ``forward`` takes the call: no gradient is needed, every BatchNorm runs on batch statistics (train mode, as the
    sem pipeline runs the model), the input is a CUDA float32 (B, C_in <= 64, N) tensor with N >= module.k and module.k <= 32,
    and the module has the reference's layer structure.  Looks at attributes only.

    Eval-mode BatchNorm is refused here: it subtracts running means from conv7 / conv8 outputs whose per-cloud offsets are large,
    and the tensor cores' truncating fp32 accumulation then leaves the fused result 2-3x further from float64 than the
    reference's own fp32 run (DESIGN §3.12).  ``eval_fusable`` accepts those calls for ``forward(..., promote=True)``."""
    return _fusable(module, x_in, False)


def eval_fusable(module, x_in) -> bool:
    """``fusable``, with any of the eight BatchNorms allowed to use running statistics (eval mode, or a mix): the calls that
    ``forward(module, x_in, promote=True)`` takes, its running-statistics layers on promoted accumulation.  Looks at attributes
    only."""
    return _fusable(module, x_in, True)


def _fusable(module, x_in, running_stats: bool) -> bool:
    try:
        x = x_in[0]
    except (TypeError, IndexError, KeyError):
        return False
    if not torch.is_tensor(x) or not structure_ok(module):
        return False
    modes = [pn2._PwChain._bn_mode(getattr(module, n)[1]) for n in _LAYERS]
    if not running_stats and any(m != 1 for m in modes):
        return False                  # running statistics (eval mode): left to the reference's forward (DESIGN §3.12)
    if not input_ok(x.is_cuda, x.dtype, tuple(x.shape), module.k, module.conv1[0].in_channels // 2, 1 in modes):
        return False
    return not _needs_grad(module, x)


_state = weakref.WeakKeyDictionary()           # module -> (packed-weight cache, conv7's x1|x2|x3 columns); entries go with the module


def _chain(module):
    st = _state.get(module)
    if st is None or st[1].conv is not module.conv7[0]:
        st = _state[module] = (pn2._PwChain(), pn2._ColumnSlice(module.conv7[0], module.conv6[0].out_channels))
    return st


def forward(module, x_in, knn: Optional[Callable] = None, keep: Optional[dict] = None, promote: bool = False) -> dict:
    """``DGCnnModule.forward`` (models/modules/dgcnn.py:96-134) under no_grad, on csrc/pw_mlp.cu.  ``x_in[0]`` is (B, C_in, N)
    float32 CUDA in any layout; returns ``{"cls_pred": (B, n_cls, N)}``.  BatchNorm keeps torch's semantics: batch statistics in
    train mode, with the running statistics and ``num_batches_tracked`` updated, running statistics in eval mode (which
    ``fusable`` does not send here), each layer as its own BatchNorm's mode says.  ``promote=True`` runs every layer whose
    BatchNorm uses running statistics on promoted accumulation (``_PwChain.run``), which keeps eval-mode outputs within the
    reference fp32 run's distance from float64 (DESIGN §3.12); batch-statistics layers launch the same either way.

    * kNN: ``knn_features`` on the current features, three times.
    * EdgeConv: layer 0 gathers [x_j - x_i | x_i] itself, the last layer keeps the max and the min over the k neighbours, and the
      final BatchNorm + LeakyReLU writes x1, x2, x3 into one (B, 192, N) buffer -- the reference's ``cat((x1, x2, x3))`` -- whose
      channel slices the next kNN reads in place.
    * conv6 keeps only each cloud's max and min over its N points: the (B, 1024, N) tensor is never written.
    * conv7's input is [g repeated over the N points | x1 x2 x3].  The g part is the same for every point of a cloud, so its
      product with conv7's first 1024 weight columns is computed once per cloud in fp64 and added to each row as a per-cloud bias;
      the tensor cores only run the 192 x1|x2|x3 columns.  (Through the tensor cores, the large per-cloud constant made the
      accumulators' truncation visible after eval-mode BatchNorm subtracted it again: DESIGN §3.12.)
    * ``dp1`` and ``cls_conv`` run as the module's own torch modules, so dropout draws from torch's generator as the reference
      does.  ``offset_conv`` and ``dist_conv``, whose outputs the reference computes and discards (:129-130) and which draw no
      random numbers, are skipped.

    ``knn`` (tests) replaces ``knn_features``: called as ``knn(x, k)``, it returns the (B, N, k) indices.  ``keep`` (tests), when
    given, receives the x1|x2|x3 buffer under "x123" and the conv8 activation (before dropout) under "conv8"."""
    x = x_in[0]
    B, _, N = x.shape
    k = int(module.k)
    find = knn_features if knn is None else knn
    chain, conv7_x = _chain(module)
    dev = x.device
    slope = {n: float(getattr(module, n)[2].negative_slope) for n in _LAYERS}
    widths = [getattr(module, names[-1])[0].out_channels for names in _EDGE_CONVS]
    with torch.no_grad():
        feats = torch.empty((B, sum(widths), N), dtype=torch.float32, device=dev)
        src, off = x, 0
        for names, width in zip(_EDGE_CONVS, widths):
            gidx = find(src, k).to(torch.int32).contiguous()
            d = L.PwLayer()
            d.mode = 2
            d.rows_per_batch = N * k
            d.edge_x, d.edge_C = L.ptr(src), src.shape[1]
            d.edge_stride[0], d.edge_stride[1], d.edge_stride[2] = src.stride()
            d.gidx, d.N, d.K = L.ptr(gidx), N, k
            seqs = [getattr(module, n) for n in names]
            chain.run([s[0] for s in seqs], [s[1] for s in seqs], d, B * N * k, feats, off, N, group=k, slopes=[slope[n] for n in names], promote=promote)
            src = feats[:, off:off + width]
            off += width
        c6 = module.conv6[0].out_channels
        d = L.PwLayer()
        d.mode, d.rows_per_batch = 0, N
        d.seg_ptr[0], d.seg_channels[0] = L.ptr(feats), off
        d.seg_batch_stride[0], d.seg_row_stride[0], d.seg_chan_stride[0] = off * N, 1, N
        g = torch.empty((B, c6, 1), dtype=torch.float32, device=dev)
        chain.run([module.conv6[0]], [module.conv6[1]], d, B * N, g, 0, 1, group=N, slopes=[slope["conv6"]], promote=promote)
        w7 = module.conv7[0].weight.detach()
        c7 = w7.shape[0]
        w7 = w7.reshape(c7, -1)
        cloud = torch.empty((B, c7), dtype=torch.float32, device=dev)
        L.call("tgn_pw_cloud_bias", B, c7, c6, L.ptr(w7), w7.stride(0), L.ptr(g), c6, L.ptr(cloud), L.stream_ptr())
        d = L.PwLayer()
        d.mode, d.rows_per_batch = 0, N
        d.seg_ptr[0], d.seg_channels[0] = L.ptr(feats), off
        d.seg_batch_stride[0], d.seg_row_stride[0], d.seg_chan_stride[0] = off * N, 1, N
        d.cloud_bias = L.ptr(cloud)
        h = torch.empty((B, module.conv8[0].out_channels, N), dtype=torch.float32, device=dev)
        chain.run([conv7_x, module.conv8[0]], [module.conv7[1], module.conv8[1]], d, B * N, h, 0, N,
                  slopes=[slope["conv7"], slope["conv8"]], promote=promote)
        if keep is not None:
            keep["x123"], keep["conv8"] = feats, h
        return {"cls_pred": module.cls_conv(module.dp1(h))}


def accelerate_forward(module_or_class, running_stats: bool = False) -> None:
    """Wrap ``DGCnnModule.forward`` of an imported reference ``dgcnn`` module (or of the class itself): calls that ``fusable``
    accepts run ``forward``; every other call, autograd included, runs the reference's own forward unchanged -- with whatever
    ``knn`` the module has, so it composes with ``accelerate``.  ``running_stats=True`` also sends the calls ``eval_fusable``
    accepts (eval-mode BatchNorm, as in validation) to ``forward(..., promote=True)``.  Calling it again leaves the class as it
    is, except that ``running_stats=True`` turns the eval-mode routing on."""
    cls = getattr(module_or_class, "DGCnnModule", module_or_class)
    original = cls.forward
    if getattr(original, "_tgn_fused", False):
        if running_stats:
            original._tgn_running_stats = True
        return

    @functools.wraps(original)
    def fused_forward(self, x_in):
        if fusable(self, x_in):
            return forward(self, x_in)
        if fused_forward._tgn_running_stats and eval_fusable(self, x_in):
            return forward(self, x_in, promote=True)
        return original(self, x_in)

    fused_forward._tgn_fused = True
    fused_forward._tgn_running_stats = bool(running_stats)
    cls.forward = fused_forward
