"""The no-grad forward of the PointNet model on the tensor-core layer chain of csrc/pw_mlp.cu (DESIGN §3.15).

``get_model.forward`` (models/modules/pointnet.py:23-35) runs ``PointNetEncoder`` (external_libs/pointnet2_utils/
pointnet_utils.py:88-134) with both learned transforms, then a four-layer head.  The sem pipeline calls it under no_grad with
BatchNorm in train mode (inference_pipeline_sem.py never calls ``.eval()``), so every BatchNorm normalises with the batch
statistics of all B * N points and updates its running statistics.

* ``forward(module, x_in)`` -- the same forward without the (B, 2176, N) concatenation, its repeat, or any full-size
  conv3 / BatchNorm output;
* ``fusable(module, x_in)`` -- whether ``forward`` takes the call;
* ``eval_fusable(module, x_in)`` -- the same, with BatchNorms on running statistics (eval mode) allowed too;
* ``accelerate_forward(module_or_class, running_stats=False)`` -- wraps ``get_model.forward``; under autograd the reference's own
  code runs, and eval-mode calls only reach ``forward`` with ``running_stats=True``.
"""
from __future__ import annotations

import functools
import weakref
from typing import Optional, Sequence

import torch
import torch.nn.functional as F
from torch import nn

from . import _lib as L
from . import pointnet2_utils as pn2

C_IN = 6                 # [xyz | normals]: the input transform rotates xyz and passes the normals through
MAX_TRANSFORM = 128      # widest per-cloud transform of tgn_pw_cloud_transform


def _conv_ok(conv, cin: int) -> bool:
    """Conv1d(cin, cout, kernel_size=1) in float32, with or without a bias"""
    if type(conv) is not nn.Conv1d:
        return False
    if (conv.kernel_size != (1,) or conv.stride != (1,) or conv.dilation != (1,) or conv.padding not in ((0,), "valid")
            or conv.groups != 1 or conv.padding_mode != "zeros" or conv.in_channels != cin):
        return False
    return conv.weight.dtype == torch.float32 and (conv.bias is None or conv.bias.dtype == torch.float32)


def _bn_ok(bn, c: int) -> bool:
    """BatchNorm1d(c) with float32 affine parameters and an exponential running average (momentum is not None)"""
    if type(bn) is not nn.BatchNorm1d or bn.num_features != c or not bn.affine or bn.weight.dtype != torch.float32:
        return False
    if bn.momentum is None:
        return False
    return bn.running_mean is None or bn.running_mean.dtype == torch.float32


def _chain_ok(convs, bns, cin: int) -> bool:
    for conv, bn in zip(convs, bns):
        if not _conv_ok(conv, cin) or not _bn_ok(bn, conv.out_channels):
            return False
        cin = conv.out_channels
    return True


def _stn_ok(stn, cin: int, k: int) -> bool:
    """STN3d / STNkd (pointnet_utils.py:10-85): three conv + BatchNorm layers from cin channels, the max over the points, then
    fc1 + LayerNorm, fc2 + LayerNorm and fc3 to k * k values"""
    try:
        convs, bns = [stn.conv1, stn.conv2, stn.conv3], [stn.bn1, stn.bn2, stn.bn3]
        fcs, lns = [stn.fc1, stn.fc2, stn.fc3], [stn.bn4, stn.bn5]
    except AttributeError:
        return False
    if not _chain_ok(convs, bns, cin):
        return False
    if not all(type(f) is nn.Linear for f in fcs) or not all(type(n) is nn.LayerNorm for n in lns):
        return False
    return fcs[0].in_features == convs[2].out_channels and fcs[2].out_features == k * k


def structure_ok(module) -> bool:
    """The layer structure of the reference's get_model (models/modules/pointnet.py:9-20) on PointNetEncoder(global_feat=False,
    feature_transform=True, channel=6), whatever the widths, with a feature transform of at most 128 channels."""
    try:
        feat = module.feat
        stn, fstn = feat.stn, feat.fstn
        enc_convs, enc_bns = [feat.conv1, feat.conv2, feat.conv3], [feat.bn1, feat.bn2, feat.bn3]
        head_convs, head_bns = [module.conv1, module.conv2, module.conv3], [module.bn1, module.bn2, module.bn3]
        conv4, n_cls, scale = module.conv4, module.k, feat.scale
        if feat.global_feat or not feat.feature_transform:
            return False
    except AttributeError:
        return False
    if not _chain_ok(enc_convs, enc_bns, C_IN):
        return False
    c1, c3 = feat.conv1.out_channels, feat.conv3.out_channels
    if not 1 <= c1 <= MAX_TRANSFORM or getattr(fstn, "k", None) != c1 or c3 != 1024 * scale:
        return False
    if not _stn_ok(stn, C_IN, 3) or not _stn_ok(fstn, c1, c1):
        return False
    if not _chain_ok(head_convs, head_bns, c3 + c1):
        return False
    return _conv_ok(conv4, module.conv3.out_channels) and conv4.out_channels == n_cls


def _bns(module):
    f = module.feat
    return [f.stn.bn1, f.stn.bn2, f.stn.bn3, f.fstn.bn1, f.fstn.bn2, f.fstn.bn3, f.bn1, f.bn2, f.bn3,
            module.bn1, module.bn2, module.bn3]


def input_ok(is_cuda: bool, dtype: torch.dtype, shape: Sequence[int], training: bool) -> bool:
    """A CUDA float32 (B, 6, N) input; in training mode BatchNorm needs two values per channel."""
    if not is_cuda or dtype != torch.float32 or len(shape) != 3:
        return False
    B, C, N = shape
    if C != C_IN or not 1 <= B <= 65535 or N < 1 or B * N >= 2 ** 31:
        return False
    return not training or B * N > 1


def _needs_grad(module, x) -> bool:
    if not torch.is_grad_enabled():
        return False
    return x.requires_grad or any(p.requires_grad for p in module.parameters())


def fusable(module, x_in) -> bool:
    """True when ``forward`` takes the call: no gradient is needed, all twelve BatchNorms of the convolutions run on batch
    statistics (train mode, as the sem pipeline runs the model), the input is a CUDA float32 (B, 6, N) tensor, and the module
    has the reference's layer structure.  Looks at attributes only.

    Eval-mode BatchNorm is refused here for the reason given for DGCNN (DESIGN §3.12): subtracting running means from layers
    whose per-cloud offsets are large makes the tensor cores' truncating accumulation visible.  ``eval_fusable`` accepts those
    calls for ``forward(..., promote=True)``."""
    return _fusable(module, x_in, False)


def eval_fusable(module, x_in) -> bool:
    """``fusable``, with any of the twelve BatchNorms allowed to use running statistics (eval mode, or a mix): the calls that
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
    modes = [pn2._PwChain._bn_mode(b) for b in _bns(module)]
    if not running_stats and any(m != 1 for m in modes):
        return False
    if not input_ok(x.is_cuda, x.dtype, tuple(x.shape), 1 in modes):
        return False
    return not _needs_grad(module, x)


_state = weakref.WeakKeyDictionary()      # module -> (packed-weight cache, head conv1's pointfeat columns); entries go with the module


def _chain(module):
    st = _state.get(module)
    if st is None or st[1].conv is not module.conv1:
        st = _state[module] = (pn2._PwChain(), pn2._ColumnSlice(module.conv1, module.feat.conv3.out_channels))
    return st


def _source(t: torch.Tensor) -> "L.PwLayer":
    """layer-0 descriptor reading the (B, C, N) tensor t in place through its strides"""
    d = L.PwLayer()
    d.mode, d.rows_per_batch = 0, t.shape[2]
    d.seg_ptr[0], d.seg_channels[0] = L.ptr(t), t.shape[1]
    d.seg_batch_stride[0], d.seg_chan_stride[0], d.seg_row_stride[0] = t.stride()
    return d


def cloud_transform(x: torch.Tensor, t: torch.Tensor, out: torch.Tensor) -> torch.Tensor:
    """out[b, j, n] = sum_i x[b, i, n] t[b, i, j] for j < C_t = t.shape[1], and out[b, C_t + c, n] = x[b, C_t + c, n]: the
    reference's ``bmm(x.transpose(2, 1), t)`` on the first C_t channels and ``cat`` with the rest (pointnet_utils.py:106-121).
    x and out are (B, C, N) float32 CUDA in any strides, t is (B, C_t, C_t) with C_t <= 128."""
    B, C, N = x.shape
    ct = t.shape[1]
    if tuple(t.shape) != (B, ct, ct) or ct > C or tuple(out.shape) != (B, C, N):
        raise L.TgnError(f"cloud_transform: shapes x {tuple(x.shape)}, t {tuple(t.shape)}, out {tuple(out.shape)} do not fit")
    if x.dtype != torch.float32 or t.dtype != torch.float32 or out.dtype != torch.float32:
        raise L.TgnError("cloud_transform: x, t and out must be float32")
    L.require_cuda(x, t, out)
    t = t.contiguous()
    L.call("tgn_pw_cloud_transform", B, N, ct, C - ct, L.ptr(x), *x.stride(), L.ptr(t), ct * ct, L.ptr(out), *out.stride(),
           L.stream_ptr())
    return out


def _stn(chain, stn, src: torch.Tensor, promote: bool) -> torch.Tensor:
    """STN3d / STNkd.forward (pointnet_utils.py:27-45, 68-85) on src (B, C, N): the conv chain keeps only each cloud's extrema
    over its N points, the apply writes relu(bn3(max)) (B, 1024); the fc layers run as the module's own, in the reference's
    expression order"""
    B, _, N = src.shape
    c3 = stn.conv3.out_channels
    g = torch.empty((B, c3, 1), dtype=torch.float32, device=src.device)
    chain.run([stn.conv1, stn.conv2, stn.conv3], [stn.bn1, stn.bn2, stn.bn3], _source(src), B * N, g, 0, 1, group=N, promote=promote)
    x = g.view(-1, c3)
    x = F.relu(stn.bn4(stn.fc1(x)))
    x = F.relu(stn.bn5(stn.fc2(x)))
    x = stn.fc3(x)
    k = round(stn.fc3.out_features ** 0.5)
    iden = torch.eye(k, dtype=torch.float32, device=x.device).view(1, k * k)     # the reference's repeat(batchsize, 1), broadcast
    x = x + iden
    return x.view(-1, k, k)


def forward(module, x_in, keep: Optional[dict] = None, promote: bool = False):
    """``get_model.forward`` (models/modules/pointnet.py:23-35) under no_grad, on csrc/pw_mlp.cu and csrc/pw_transform.cu.
    ``x_in[0]`` is (B, 6, N) float32 CUDA in any layout; returns ``(log-probabilities (B, k, N), trans_feat (B, 128, 128))``.
    BatchNorm keeps torch's semantics, each layer as its own BatchNorm's mode says: batch statistics, running statistics and
    ``num_batches_tracked`` updated once per layer in train mode; running statistics, untouched, in eval mode.  ``promote=True``
    runs every layer whose BatchNorm uses running statistics on promoted accumulation (``_PwChain.run``, DESIGN §3.15); layers
    on batch statistics launch the same either way.

    * STN3d: three layers read x through its strides, the last keeps only each cloud's max and min over its N points, and one
      apply writes relu(bn3(max)); fc1-fc3 and the identity run as the module's own layers -> trans.
    * ``tgn_pw_cloud_transform``: [xyz . trans | normals]; enc conv1, and an apply writes relu(bn1(y1)) (B, 128, N).
    * STNkd on relu(bn1(y1)) the same way -> trans_feat; ``tgn_pw_cloud_transform`` writes pointfeat = x . trans_feat.
    * conv2 from pointfeat, conv3 keeping the extrema only, and an apply with no activation -> g (B, 2048).
    * Head conv1's input is [g repeated over the N points | pointfeat].  The g part is the same for every point of a cloud, so
      its product with conv1's first 2048 weight columns is one fp64 per-cloud bias (``tgn_pw_cloud_bias``) and the tensor
      cores run only pointfeat's 128 columns.  Then conv2, conv3 and the apply.
    * conv4 and the log_softmax run as the reference writes them.

    ``keep`` (tests), when given, receives "trans", "g" (B, 2048), "pointfeat" and "head3" (the head's conv3 activation)."""
    x = x_in[0]
    B, C, N = x.shape
    feat = module.feat
    chain, head1 = _chain(module)
    rows = B * N
    dev = x.device
    with torch.no_grad():
        trans = _stn(chain, feat.stn, x, promote)
        xt = cloud_transform(x, trans, torch.empty((B, C, N), dtype=torch.float32, device=dev))
        c1 = feat.conv1.out_channels
        a1 = torch.empty((B, c1, N), dtype=torch.float32, device=dev)
        chain.run([feat.conv1], [feat.bn1], _source(xt), rows, a1, 0, N, promote=promote)
        del xt
        trans_feat = _stn(chain, feat.fstn, a1, promote)
        pointfeat = cloud_transform(a1, trans_feat, torch.empty((B, c1, N), dtype=torch.float32, device=dev))
        del a1
        c3 = feat.conv3.out_channels
        g = torch.empty((B, c3, 1), dtype=torch.float32, device=dev)
        chain.run([feat.conv2, feat.conv3], [feat.bn2, feat.bn3], _source(pointfeat), rows, g, 0, 1, group=N, relu=False, promote=promote)
        w1 = module.conv1.weight.detach()
        co = w1.shape[0]
        w1 = w1.reshape(co, -1)
        cloud = torch.empty((B, co), dtype=torch.float32, device=dev)
        L.call("tgn_pw_cloud_bias", B, co, c3, L.ptr(w1), w1.stride(0), L.ptr(g), c3, L.ptr(cloud), L.stream_ptr())
        d = _source(pointfeat)
        d.cloud_bias = L.ptr(cloud)
        h = torch.empty((B, module.conv3.out_channels, N), dtype=torch.float32, device=dev)
        chain.run([head1, module.conv2, module.conv3], [module.bn1, module.bn2, module.bn3], d, rows, h, 0, N, promote=promote)
        if keep is not None:
            keep.update(trans=trans, g=g.view(B, c3), pointfeat=pointfeat, head3=h)
        out = module.conv4(h)
        out = out.transpose(2, 1).contiguous()
        out = F.log_softmax(out.view(-1, module.k), dim=-1)
        out = out.view(B, N, module.k).permute(0, 2, 1)
        return out, trans_feat


def accelerate_forward(module_or_class, running_stats: bool = False) -> None:
    """Wrap ``get_model.forward`` of an imported reference ``pointnet`` module (or of the class itself): calls that ``fusable``
    accepts run ``forward``; every other call, autograd included, runs the reference's own forward unchanged.
    ``running_stats=True`` also sends the calls ``eval_fusable`` accepts (eval-mode BatchNorm, as in validation) to
    ``forward(..., promote=True)``.  Calling it again leaves the class as it is, except that ``running_stats=True`` turns the
    eval-mode routing on."""
    cls = getattr(module_or_class, "get_model", module_or_class)
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
