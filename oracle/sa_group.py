"""oracle/sa_group.py -- float64 restatement of one ``tgn_sa_group_mlp_max`` launch (TEST INFRASTRUCTURE ONLY).

``group_mlp_max`` follows the header's contract (include/tgn_b200.h): the operand row of neighbour j of centre s in cloud b is
built in float32 as every engine builds it -- ``xyz[b, j] - new_xyz[b, s]`` as a float32 subtraction, the features verbatim,
``[xyz_rel | feats]`` when ``xyz_first`` else ``[feats | xyz_rel]``, and a zero row when j is outside [0, N).  From there on
everything is float64: each layer's product, bias and ReLU, then the max over the K rows of the neighbourhood.

The second result is the MAGNITUDE pass: the same network on |x|, |W| and |b| (ReLU is the identity there), reduced by max over
the neighbourhood.  An evaluation whose every layer computes ``relu(W x + b)`` with a relative error of at most kappa per
product-and-sum (|error| <= kappa * (|W| |x| + |b|) element-wise) is within ``kappa * L * mag`` of the float64 result: ReLU and the
max are 1-Lipschitz, and layer l's inherited error, l * kappa * m_l, maps through |W| to at most l * kappa * m_(l+1).
"""
from __future__ import annotations

from typing import Optional, Sequence, Tuple

import torch

_F64 = torch.float64


def operand_rows(N: int, D: int, xyz, feats, new_xyz, gidx, xyz_first: int, b: torch.Tensor, s: torch.Tensor) -> torch.Tensor:
    """The float32 operand of neighbourhoods (b[i], s[i]) -> (M, K, 3 + D)"""
    j = gidx[b, s].long()                                                     # (M, K)
    ok = (j >= 0) & (j < N)
    jc = j.clamp(0, N - 1)
    bb = b.unsqueeze(1).expand_as(jc)
    rel = xyz[bb, jc].float() - new_xyz[b, s].float().unsqueeze(1)            # float32 subtraction
    if D == 0:
        x = rel
    else:
        f = feats[bb, jc].float()
        x = torch.cat([rel, f] if xyz_first else [f, rel], -1)
    return torch.where(ok.unsqueeze(-1), x, torch.zeros((), dtype=x.dtype))


def group_mlp_max(B: int, N: int, S: int, K: int, D: int, xyz, feats, new_xyz, gidx, xyz_first: int,
                  channels: Sequence[int], weights: Sequence[torch.Tensor], biases: Sequence[torch.Tensor],
                  select: Optional[Sequence[Tuple[int, int]]] = None, chunk: int = 2048):
    """One launch in float64.  xyz (B,N,3), feats (B,N,D) point-major or None, new_xyz (B,S,3), gidx (B,S,K), weights[l]
    (C_{l+1}, C_l), biases[l] (C_{l+1}); CPU tensors.  -> (out, mag), each float64 (B, C_last, S); with ``select`` (a list of
    (b, s) neighbourhoods) each is (len(select), C_last) instead, in the order given."""
    assert len(channels) == len(weights) + 1 == len(biases) + 1 and channels[0] == 3 + D
    for l, w in enumerate(weights):
        assert tuple(w.shape) == (channels[l + 1], channels[l])
    ws = [w.to(_F64) for w in weights]
    bs = [b.to(_F64) for b in biases]
    was = [w.abs() for w in ws]
    bas = [b.abs() for b in bs]
    if select is None:
        bsel = torch.arange(B).repeat_interleave(S)
        ssel = torch.arange(S).repeat(B)
    else:
        sel = torch.as_tensor(select, dtype=torch.int64).reshape(-1, 2)
        bsel, ssel = sel[:, 0], sel[:, 1]
    outs, mags = [], []
    for i in range(0, bsel.numel(), chunk):
        b, s = bsel[i:i + chunk], ssel[i:i + chunk]
        x = operand_rows(N, D, xyz, feats, new_xyz, gidx, xyz_first, b, s).to(_F64)     # (M, K, C0)
        m = x.abs()
        for w, bias, wa, ba in zip(ws, bs, was, bas):
            x = (x @ w.t() + bias).clamp(min=0.0)
            m = m @ wa.t() + ba
        outs.append(x.amax(1))
        mags.append(m.amax(1))
    out, mag = torch.cat(outs), torch.cat(mags)
    if select is None:
        c = channels[-1]
        out = out.reshape(B, S, c).permute(0, 2, 1).contiguous()
        mag = mag.reshape(B, S, c).permute(0, 2, 1).contiguous()
    return out, mag
