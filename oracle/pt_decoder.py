"""oracle/pt_decoder.py -- float64 restatement of the point-transformer decoder and heads (TEST INFRASTRUCTURE ONLY).

``transition_up`` is blocks.TransitionUp.forward (models/modules/cbl_point_transformer/blocks.py:92-111) in both forms and
``multi_head`` is heads.MultiHead.forward (heads.py:53-61, combine = concat), written as pure functions of the modules'
``state_dict`` and of given neighbour indices (the kNN is tested elsewhere; the k = 3 weights are inputs too, as
pointops.interpolation computes them from the float32 distances).  Tensors may be CPU or CUDA tensors; BatchNorm is torch's (batch
statistics with biased variance for the normalisation and the unbiased one for the running update, or running statistics).

Every value carries a first-order bound on the error of a float32 evaluation of the same steps (u = 2^-24):
* a product-and-sum of d terms plus a bias: |W| err(x) + (d + 1) u (|W| |x| + |b|) -- this also covers the layer chain's
  three-part bf16 products, whose dropped terms are ~2^-23 of each product;
* BatchNorm of y with batch statistics: |scale| (err(y) + mean err(y)) + |x_hat scale| mean(|y - mean| err(y)) / (var + eps)
  for the statistics, plus u (5 |y - mean| |scale| + |beta|) for its own roundings; ReLU is 1-Lipschitz;
* the k = 3 interpolation: sum_j w_j err(f_j) + 3 u sum_j |f_j w_j|, and u |sum| for the final add.
"""
from __future__ import annotations

from typing import Dict, Optional, Sequence, Tuple

import torch

_F64 = torch.float64
U = 2.0 ** -24


def _t(v) -> torch.Tensor:
    return torch.as_tensor(v).to(_F64)


def linear(x, ex, w, b=None) -> Tuple[torch.Tensor, torch.Tensor]:
    """x (n, d) @ w.T + b with its bound"""
    w = _t(w)
    aw = w.abs()
    y = x @ w.t()
    mag = x.abs() @ aw.t()
    if b is not None:
        y = y + _t(b)
        mag = mag + _t(b).abs()
    return y, ex @ aw.t() + (w.shape[1] + 1) * U * mag


def batchnorm(y, ey, state: Dict[str, torch.Tensor], prefix: str, train: bool, eps: float = 1e-5, momentum: float = 0.1):
    """-> (z, err, running statistics after the step {name: tensor})"""
    gamma, beta = _t(state[prefix + "weight"]), _t(state[prefix + "bias"])
    rm, rv = _t(state[prefix + "running_mean"]), _t(state[prefix + "running_var"])
    after = {}
    if train:
        n = y.shape[0]
        mean = y.mean(0)
        var = ((y - mean) ** 2).mean(0)
        after[prefix + "running_mean"] = (1 - momentum) * rm + momentum * mean
        after[prefix + "running_var"] = (1 - momentum) * rv + momentum * var * n / max(n - 1, 1)
        after[prefix + "num_batches_tracked"] = torch.as_tensor(state[prefix + "num_batches_tracked"]) + 1
    else:
        mean, var = rm, rv
    scale = gamma / torch.sqrt(var + eps)
    d = y - mean
    z = d * scale + beta
    e = scale.abs() * ey + U * (5 * d.abs() * scale.abs() + beta.abs())
    if train:
        e = e + scale.abs() * ey.mean(0) + (d * scale).abs() * (d.abs() * ey).mean(0) / (var + eps)
    return z, e, after


def lbr(x, ex, state, prefix: str, train: bool, bn: bool = True):
    """Sequential(Linear, [BatchNorm1d,] ReLU) at ``prefix`` (``prefix + "0."``, ``prefix + "1."``)"""
    y, e = linear(x, ex, state[prefix + "0.weight"], state.get(prefix + "0.bias"))
    after = {}
    if bn:
        y, e, after = batchnorm(y, e, state, prefix + "1.", train)
    return y.clamp(min=0), e, after


def interpolate(f, ef, idx, w):
    """((0 + f[i0] w0) + f[i1] w1) + f[i2] w2 per row (pointops.interpolation) with its bound"""
    idx, w = torch.as_tensor(idx).long(), _t(w)
    terms = f[idx] * w.unsqueeze(-1)                               # (n, k, c)
    return terms.sum(1), (ef[idx] * w.abs().unsqueeze(-1)).sum(1) + idx.shape[1] * U * terms.abs().sum(1)


def transition_up(state: Dict[str, torch.Tensor], x1, offsets: Sequence[int], train: bool, x2=None, idx=None, w=None):
    """TransitionUp.forward -> (out, err, running statistics after).  Without x2 the head form: x1's rows split into clouds at
    ``offsets`` (the o tensor), each concatenated with linear2 of its column mean.  With x2: linear1(x1) + the k = 3 interpolation
    of linear2(x2) through idx / w, (n1, 3)."""
    x1 = _t(x1)
    z = torch.zeros_like(x1)
    after = {}
    if x2 is None:
        c = x1.shape[1]
        parts, starts = [], [0] + list(offsets[:-1])
        for s, e in zip(starts, offsets):
            g = x1[s:e].mean(0, keepdim=True)
            h, eh, _ = lbr(g, U * g.abs(), state, "linear2.", train, bn=False)
            parts.append((torch.cat([x1[s:e], h.expand(e - s, c)], 1), torch.cat([z[s:e], eh.expand(e - s, c)], 1)))
        xc, ec = torch.cat([p[0] for p in parts]), torch.cat([p[1] for p in parts])
        out, err, after = lbr(xc, ec, state, "linear1.", train)
        return out, err, after
    x2 = _t(x2)
    a, ea, after1 = lbr(x1, z, state, "linear1.", train)
    f, ef, after2 = lbr(x2, torch.zeros_like(x2), state, "linear2.", train)
    s, es = interpolate(f, ef, idx, w)
    out = a + s
    return out, ea + es + U * out.abs(), {**after1, **after2}


def head_classify(lats: Sequence[torch.Tensor], errs: Sequence[torch.Tensor], nns: Sequence[Optional[torch.Tensor]], w, b=None):
    """sum_s W[:, 32 s:32 s + 32] lat_s[nn_s] + b with lat_s (n_s, 32) row-major and nn_s (n0,) or None (identity)"""
    cols = [lat if nn is None else lat[torch.as_tensor(nn).long().reshape(-1)] for lat, nn in zip(lats, nns)]
    ecols = [e if nn is None else e[torch.as_tensor(nn).long().reshape(-1)] for e, nn in zip(errs, nns)]
    return linear(torch.cat(cols, 1), torch.cat(ecols, 1), w, b)


def multi_head(state: Dict[str, torch.Tensor], feats: Sequence, nns: Sequence[Optional[torch.Tensor]], train: bool):
    """MultiHead.forward with combine = concat -> (out, err, latents [(n_s, 32)], running statistics after).  ``state`` is the
    head's state_dict (infer_list.{s}.infer.{0,1}, cls); nns[s] is the k = 1 neighbour of each level-0 point in level s, or None
    for a level-0 stage."""
    lats, errs, after = [], [], {}
    for s, x in enumerate(feats):
        x = _t(x)
        lat, e, a = lbr(x, torch.zeros_like(x), state, f"infer_list.{s}.infer.", train)
        lats.append(lat)
        errs.append(e)
        after.update(a)
    out, err = head_classify(lats, errs, nns, state["cls.weight"], state.get("cls.bias"))
    return out, err, lats, after

