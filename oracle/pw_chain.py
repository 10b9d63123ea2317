"""oracle/pw_chain.py -- float64 restatement of the batch-statistics layer chain's descriptors (TEST INFRASTRUCTURE ONLY).

``layer_forward`` is one ``tgn_pw_layer_forward`` launch (include/tgn_b200.h, tgn_pw_layer_t), ``apply`` one ``tgn_pw_apply``
launch (tgn_pw_apply_t), ``running_update`` the momentum update either of them performs.  Keyword names are the descriptor's
field names; tensors are CPU tensors (``weight`` is the (cout, cin) float32 weight the packed operand was made from, ``seg_ptr``
/ ``edge_x`` are flat views of the storage the descriptor points into, read through the descriptor's strides in elements).

The operand is built as the kernel builds it, in the inputs' dtype (float32, as the kernel reads them): strided segments, ``xyz - centre`` and the EdgeConv difference as
float32 subtractions, zero rows for out-of-range indices (which skip the input BatchNorm).  Everything after that is float64:
the input BatchNorm (batch sums or running statistics) and its ReLU / LeakyReLU, the product, ``bias`` and ``cloud_bias``.
Chain-level checks reuse ``oracle._conv_bn_relu`` / ``set_abstraction`` / ``feature_propagation`` instead.
"""
from __future__ import annotations

from typing import Optional, Sequence

import torch

_F64 = torch.float64


def _bn_scale(mode: int, c: int, stats, count: float, gamma, beta, eps: float, rmean, rvar):
    """(mean, scale, beta) of a BatchNorm from batch sums (mode 1: {sum[c], sumsq[c]} over ``count`` rows) or running
    statistics (mode 2), as float64 vectors; gamma / beta None act as 1 / 0 (affine=False)."""
    if mode == 1:
        s = stats.to(_F64)
        mean = s[:c] / count
        var = (s[c:2 * c] / count - mean * mean).clamp(min=0.0)
    else:
        mean, var = rmean.to(_F64), rvar.to(_F64)
    g = torch.ones(c, dtype=_F64) if gamma is None else gamma.to(_F64)
    b = torch.zeros(c, dtype=_F64) if beta is None else beta.to(_F64)
    # eps is a float32 field of the descriptor
    scale = g / torch.sqrt(var + float(torch.tensor(eps, dtype=torch.float32)))
    return mean, scale, b


def _act(v: torch.Tensor, act: int, slope: float, relu: bool = True) -> torch.Tensor:
    if act == 1:
        return torch.where(v > 0, v, v * float(torch.tensor(slope, dtype=torch.float32)))
    return v.clamp(min=0.0) if relu else v


def running_update(stats, count: float, momentum: float, running_mean, running_var):
    """torch's training-mode side effect: running = (1 - m) running + m batch, the batch variance unbiased -> (mean, var) float64"""
    c = running_mean.numel()
    s = stats.to(_F64)
    mean = s[:c] / count
    var = (s[c:2 * c] / count - mean * mean).clamp(min=0.0)
    if count > 1:
        var = var * count / (count - 1)
    m = float(torch.tensor(momentum, dtype=torch.float32))
    return (1 - m) * running_mean.to(_F64) + m * mean, (1 - m) * running_var.to(_F64) + m * var


def _operand(rows: int, cin: int, mode: int, rows_per_batch: int, seg_ptr, seg_channels, seg_batch_stride, seg_row_stride,
             seg_chan_stride, xyz, feats, new_xyz, gidx, N, S, K, D, xyz_first, edge_x, edge_stride, edge_C):
    """-> (x (rows, cin) float32, row_ok (rows,) bool)"""
    r = torch.arange(rows, dtype=torch.int64)
    ok = torch.ones(rows, dtype=torch.bool)
    if mode == 0:
        b, n = r // rows_per_batch, r % rows_per_batch
        parts = []
        for i in range(2):
            ch = int(seg_channels[i]) if i < len(seg_channels) else 0
            if ch <= 0:
                continue
            k = torch.arange(ch, dtype=torch.int64)
            off = (b * int(seg_batch_stride[i]) + n * int(seg_row_stride[i])).unsqueeze(1) + k.unsqueeze(0) * int(seg_chan_stride[i])
            parts.append(seg_ptr[i].reshape(-1)[off])
        return torch.cat(parts, 1), ok
    g = gidx.reshape(-1).long()
    if mode == 1:
        grp = r // K
        b = grp // S
        ok = (g >= 0) & (g < N)
        j = g.clamp(0, N - 1)
        x3 = xyz.reshape(-1, N, 3)
        rel = x3[b, j] - new_xyz.reshape(-1, 3)[grp]                          # float32 subtraction
        cols = [rel] if D == 0 else ([rel, feats.reshape(-1, N, D)[b, j]] if xyz_first else
                                     [feats.reshape(-1, N, D)[b, j], rel])
        x = torch.cat(cols, 1)
    else:
        pt = r // K
        b, n = pt // N, pt % N
        ok = (g >= 0) & (g < N)
        m = g.clamp(0, N - 1)
        flat = edge_x.reshape(-1)
        c = torch.arange(edge_C, dtype=torch.int64).unsqueeze(0) * int(edge_stride[1])
        base = (b * int(edge_stride[0])).unsqueeze(1)
        xe = flat[base + (n * int(edge_stride[2])).unsqueeze(1) + c]
        xf = flat[base + (m * int(edge_stride[2])).unsqueeze(1) + c]
        x = torch.cat([xf - xe, xe], 1)                                         # [x_j - x_i | x_i], float32 subtraction
    x = torch.where(ok.unsqueeze(1), x, torch.zeros((), dtype=x.dtype))
    assert x.shape == (rows, cin)
    return x, ok


def layer_forward(*, rows: int, cin: int, cout: int, weight: torch.Tensor, bias: Optional[torch.Tensor] = None, mode: int = 0,
                  rows_per_batch: int = 0, seg_ptr: Sequence = (), seg_channels: Sequence[int] = (0, 0),
                  seg_batch_stride: Sequence[int] = (0, 0), seg_row_stride: Sequence[int] = (0, 0),
                  seg_chan_stride: Sequence[int] = (0, 0), xyz=None, feats=None, new_xyz=None, gidx=None, N: int = 0, S: int = 0,
                  K: int = 0, D: int = 0, xyz_first: int = 0, edge_x=None, edge_stride: Sequence[int] = (0, 0, 0), edge_C: int = 0,
                  in_affine: int = 0, in_stats=None, in_gamma=None, in_beta=None, in_running_mean=None, in_running_var=None,
                  in_eps: float = 1e-5, in_act: int = 0, in_act_slope: float = 0.0, cloud_bias=None, group: int = 0, **_ignored):
    """One tgn_pw_layer_forward launch in float64 -> dict(y (cout, rows), stats (2 cout) = {sum y, sum y^2},
    ymax / ymin (cout, rows / group) when group > 0).  Descriptor fields the result does not depend on (precision,
    extrema_atomic, the running-statistics update) are accepted and ignored."""
    x, ok = _operand(rows, cin, mode, rows_per_batch, seg_ptr, seg_channels, seg_batch_stride, seg_row_stride, seg_chan_stride,
                     xyz, feats, new_xyz, gidx, N, S, K, D, xyz_first, edge_x, edge_stride, edge_C)
    x = x.to(_F64)
    if in_affine:
        mean, scale, beta = _bn_scale(in_affine, cin, in_stats, float(rows), in_gamma, in_beta, in_eps, in_running_mean,
                                      in_running_var)
        h = _act((x - mean) * scale + beta, in_act, in_act_slope)
        x = torch.where(ok.unsqueeze(1), h, x)                                 # zero rows stay zero
    y = weight.to(_F64) @ x.t()
    if bias is not None:
        y = y + bias.to(_F64).unsqueeze(1)
    if cloud_bias is not None:
        b = torch.arange(rows) // rows_per_batch
        y = y + cloud_bias.reshape(-1, cout).to(_F64)[b].t()
    out = {"y": y, "stats": torch.cat([y.sum(1), (y * y).sum(1)])}
    if group:
        g = y.reshape(cout, rows // group, group)
        out["ymax"], out["ymin"] = g.amax(2), g.amin(2)
    return out


def apply(*, src: torch.Tensor, rows_per_batch: int, channels: int, out_channels: int = 0, out_c_offset: int = 0, relu: int = 1,
          ymin: Optional[torch.Tensor] = None, affine: int = 0, stats=None, stat_rows: int = 0, gamma=None, beta=None,
          running_mean=None, running_var=None, eps: float = 1e-5, act: int = 0, act_slope: float = 0.0, **_ignored) -> torch.Tensor:
    """One tgn_pw_apply launch in float64 -> the channels it writes, (B, channels, rows_per_batch): act(BatchNorm(v)) with
    v = src, or, when ymin is given, v = src (the max) where the scale is >= 0 and ymin where it is negative."""
    rows = src.shape[1]
    v = src.to(_F64)
    if affine:
        mean, scale, b = _bn_scale(affine, channels, stats, float(stat_rows), gamma, beta, eps, running_mean, running_var)
        if ymin is not None:
            v = torch.where((scale < 0).unsqueeze(1), ymin.to(_F64), v)
        v = (v - mean.unsqueeze(1)) * scale.unsqueeze(1) + b.unsqueeze(1)
    v = _act(v, act, act_slope, bool(relu))
    return v.reshape(channels, rows // rows_per_batch, rows_per_batch).permute(1, 0, 2)
