"""oracle/pt_block.py -- float64 restatement of the point-transformer block (TEST INFRASTRUCTURE ONLY).

``block`` is blocks.PointTransformerBlock.forward (models/modules/cbl_point_transformer/blocks.py:127-135) as a pure function of
the module's ``state_dict`` and of given neighbour indices (the kNN is tested elsewhere): linear1, bn1, ReLU, the transformer
layer, bn2, ReLU, linear3, bn3, the residual add and the ReLU, everything in float64, with torch's BatchNorm (batch statistics
with the biased variance for the normalisation and the unbiased one for the running update, or running statistics).

``res_apply`` is one ``tgn_pt_res_apply`` launch: relu(bn3(y) + identity) for a channel-major y, with a first-order bound on the
error of the float32 evaluation (u = 2^-24): the subtract-first BatchNorm's own roundings, u (5 |y - mean| |scale| + |beta|), plus
what the batch statistics carry when y carries an error (``pt_decoder.batchnorm``), then u |z + identity| for the add; ReLU is
1-Lipschitz.
"""
from __future__ import annotations

from typing import Dict

import torch

from . import pt_decoder

_F64 = torch.float64
U = pt_decoder.U
_t = pt_decoder._t


def res_apply(y, state: Dict[str, torch.Tensor], prefix: str, identity, train: bool, ey=None, eps: float = 1e-5,
              momentum: float = 0.1):
    """y (c, rows) channel-major, identity (rows, c) -> (out (rows, c), bound, running statistics after the step)"""
    yr = _t(y).t()
    ey = torch.zeros_like(yr) if ey is None else _t(ey).t()
    z, e, after = pt_decoder.batchnorm(yr, ey, state, prefix, train, eps, momentum)
    s = z + _t(identity)
    return s.clamp(min=0), e + U * s.abs(), after


def _bn(y, state, prefix, train, after, eps=1e-5, momentum=0.1):
    """torch's BatchNorm1d over the rows of y (n, c) -> normalised y; the running statistics after the step go into ``after``"""
    gamma, beta = _t(state[prefix + "weight"]), _t(state[prefix + "bias"])
    if train:
        n = y.shape[0]
        mean, var = y.mean(0), y.var(0, unbiased=False)
        after[prefix + "running_mean"] = (1 - momentum) * _t(state[prefix + "running_mean"]) + momentum * mean
        after[prefix + "running_var"] = (1 - momentum) * _t(state[prefix + "running_var"]) + momentum * var * n / max(n - 1, 1)
        after[prefix + "num_batches_tracked"] = torch.as_tensor(state[prefix + "num_batches_tracked"]) + 1
    else:
        mean, var = _t(state[prefix + "running_mean"]), _t(state[prefix + "running_var"])
    return (y - mean) / torch.sqrt(var + eps) * gamma + beta


def _lin(x, state, name):
    y = x @ _t(state[name + ".weight"]).t()
    return y + _t(state[name + ".bias"]) if state.get(name + ".bias") is not None else y


def transformer_layer(state: Dict[str, torch.Tensor], prefix: str, p, x, idx, train: bool, after: dict, share: int = 8):
    """blocks.PointTransformerLayer.forward (:31-44) with the neighbours idx (n, K) of every point: BatchNorms over all n K rows"""
    p, x, idx = _t(p), _t(x), torch.as_tensor(idx).long()
    n, K = idx.shape
    q, k, v = (_lin(x, state, prefix + name) for name in ("linear_q", "linear_k", "linear_v"))
    c = v.shape[1]
    rows = lambda t: t.reshape(n * K, -1)
    rel = p[idx] - p.unsqueeze(1)
    t = _bn(rows(_lin(rel, state, prefix + "linear_p.0")), state, prefix + "linear_p.1.", train, after).clamp(min=0)
    pr = _lin(t, state, prefix + "linear_p.3").view(n, K, c)
    w = k[idx] - q.unsqueeze(1) + pr
    w = _bn(rows(w), state, prefix + "linear_w.0.", train, after).clamp(min=0)
    w = _bn(_lin(w, state, prefix + "linear_w.2"), state, prefix + "linear_w.3.", train, after).clamp(min=0)
    w = torch.softmax(_lin(w, state, prefix + "linear_w.5").view(n, K, c // share), dim=1)
    return ((v[idx] + pr).view(n, K, share, c // share) * w.unsqueeze(2)).sum(1).view(n, c)


def block(state: Dict[str, torch.Tensor], p, x, idx, train: bool):
    """PointTransformerBlock.forward -> (out (n, c), running statistics after the step {state_dict key: tensor})"""
    x = _t(x)
    after: dict = {}
    h = _bn(_lin(x, state, "linear1"), state, "bn1.", train, after).clamp(min=0)
    h = _bn(transformer_layer(state, "transformer2.", p, h, idx, train, after), state, "bn2.", train, after).clamp(min=0)
    h = _bn(_lin(h, state, "linear3"), state, "bn3.", train, after)
    return (h + x).clamp(min=0), after
