"""oracle/pw_chain.py, the float64 restatement of tgn_pw_layer_forward / tgn_pw_apply, pinned against float64 torch modules:
Conv1d / Conv2d + BatchNorm (train and eval mode) + ReLU / LeakyReLU, chained through the descriptors the way the library
chains them (layer l + 1 applies BatchNorm l while it builds its operand; tgn_pw_apply finishes the last one, from the max or
the min of a neighbourhood by the sign of the scale)."""
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle import pw_chain

F64 = torch.float64


def _close(a, b, tol=1e-10):
    a, b = a.detach().double(), b.detach().double()
    return float((a - b).abs().max()) <= tol * max(1.0, float(b.abs().max()))


def _bns(widths, dim, affine, momentum, gen):
    """BatchNorms with negative, zero and positive scales (affine) and non-trivial running statistics"""
    out = []
    for c in widths:
        bn = (nn.BatchNorm1d if dim == 1 else nn.BatchNorm2d)(c, affine=affine, momentum=momentum).double()
        with torch.no_grad():
            if affine:
                g = torch.randn(c, generator=gen, dtype=F64)
                g[::5] = 0.0
                bn.weight.copy_(g)
                bn.bias.copy_(torch.randn(c, generator=gen, dtype=F64) * 0.2)
            bn.running_mean.copy_(torch.randn(c, generator=gen, dtype=F64) * 0.3)
            bn.running_var.copy_(torch.rand(c, generator=gen, dtype=F64) + 0.5)
        out.append(bn)
    return out


def _act(h, slope):
    return F.leaky_relu(h, slope) if slope is not None else F.relu(h)


def _bn_fields(bn, prefix, stats, train):
    mode = 1 if train else 2
    return {prefix + "affine": mode, prefix + "stats": stats if train else None, prefix + "gamma": bn.weight, prefix + "beta": bn.bias,
            prefix + "running_mean": bn.running_mean, prefix + "running_var": bn.running_var, prefix + "eps": bn.eps}


def _chain(first, widths, weights, biases, bns, train, slope, rows, rows_per_batch_out, group=0):
    """layer 0 from ``first`` (its operand fields), layers 1.. from the previous y, then tgn_pw_apply -> (out, running stats)"""
    act = {"in_act": 1, "in_act_slope": slope} if slope is not None else {}
    prev, running = None, []
    for l, (w, b) in enumerate(zip(weights, biases)):
        last = l == len(weights) - 1
        d = dict(first) if l == 0 else {"mode": 0, "rows_per_batch": rows, "seg_ptr": (prev["y"],), "seg_channels": (widths[l], 0),
                                         "seg_batch_stride": (0, 0), "seg_row_stride": (1, 0), "seg_chan_stride": (rows, 0), **act}
        if l > 0:
            d.update(_bn_fields(bns[l - 1], "in_", prev["stats"], train))
            if train:
                running.append(pw_chain.running_update(prev["stats"], rows, bns[l - 1].momentum, bns[l - 1].running_mean,
                                                       bns[l - 1].running_var))
        prev = pw_chain.layer_forward(rows=rows, cin=widths[l], cout=widths[l + 1], weight=w, bias=b, group=group if last else 0, **d)
    bn = bns[-1]
    a = {"affine": 1 if train else 2, "stats": prev["stats"], "stat_rows": rows, "gamma": bn.weight, "beta": bn.bias,
         "running_mean": bn.running_mean, "running_var": bn.running_var, "eps": bn.eps, "relu": 1}
    if slope is not None:
        a.update(act=1, act_slope=slope)
    if group:
        out = pw_chain.apply(src=prev["ymax"], ymin=prev["ymin"], rows_per_batch=rows_per_batch_out, channels=widths[-1], **a)
    else:
        out = pw_chain.apply(src=prev["y"], rows_per_batch=rows_per_batch_out, channels=widths[-1], **a)
    if train:
        running.append(pw_chain.running_update(prev["stats"], rows, bn.momentum, bn.running_mean, bn.running_var))
    return out, running


@pytest.mark.parametrize("train", [True, False])
@pytest.mark.parametrize("affine", [True, False])
@pytest.mark.parametrize("momentum", [0.1, 0.01])
@pytest.mark.parametrize("slope", [None, 0.25])            # a float32 value: the descriptor carries the slope as float32
def test_conv1d_chain_matches_float64_modules(train, affine, momentum, slope):
    """feature-propagation form: [skip (channel-first) | interpolated (point-major)] -> two Conv1d + BatchNorm1d layers"""
    gen = torch.Generator().manual_seed(7 + int(train) + 2 * int(affine))
    B, N, D1, D2, widths = 2, 150, 5, 7, [12, 9, 6]
    skip = torch.randn(B, D1, N, generator=gen)                                     # float32 values, as the kernel reads them
    interp = torch.randn(B, N, D2, generator=gen)
    convs = [nn.Conv1d(widths[i], widths[i + 1], 1).double() for i in range(2)]
    for c in convs:
        with torch.no_grad():
            c.weight.copy_(c.weight.float().double())
            c.bias.copy_(c.bias.float().double())
    bns = _bns(widths[1:], 1, affine, momentum, gen)
    ref_bns = [nn.BatchNorm1d(c, affine=affine, momentum=momentum).double() for c in widths[1:]]
    for r, b in zip(ref_bns, bns):
        r.load_state_dict(b.state_dict())
        r.train(train)
    h = torch.cat([skip, interp.transpose(1, 2)], 1).double()
    for l, (c, bn) in enumerate(zip(convs, ref_bns)):
        h = _act(bn(c(h)), slope)
    first = {"mode": 0, "rows_per_batch": N, "seg_ptr": (skip, interp), "seg_channels": (D1, D2),
             "seg_batch_stride": (D1 * N, N * D2), "seg_row_stride": (1, D2), "seg_chan_stride": (N, 1)}
    out, running = _chain(first, widths, [c.weight.detach().reshape(c.weight.shape[0], -1) for c in convs],
                          [c.bias.detach() for c in convs], bns, train, slope, B * N, N)
    assert _close(out, h.detach())
    if train:
        for (m, v), r in zip(running, ref_bns):
            assert _close(m, r.running_mean, 1e-7) and _close(v, r.running_var, 1e-7)


@pytest.mark.parametrize("xyz_first,D,K", [(1, 0, 5), (0, 4, 6), (1, 4, 1)])
@pytest.mark.parametrize("train", [True, False])
def test_grouped_conv2d_chain_and_max_matches_float64_modules(xyz_first, D, K, train):
    """set-abstraction form: gather [xyz - centre | feats] (or [feats | xyz - centre]), two Conv2d + BatchNorm2d layers, max over
    the K neighbours; negative scales take the min; an out-of-range index is a zero row"""
    gen = torch.Generator().manual_seed(11 + K)
    B, N, S, widths = 2, 40, 7, [D + 3, 10, 8]
    xyz = torch.rand(B, N, 3, generator=gen)
    feats = torch.randn(B, N, D, generator=gen) if D else None
    new_xyz = xyz[:, :S].contiguous()
    gidx = torch.randint(0, N, (B, S, K), generator=gen, dtype=torch.int32)
    gidx[0, 1, K - 1] = N
    convs = [nn.Conv2d(widths[i], widths[i + 1], 1).double() for i in range(2)]
    for c in convs:
        with torch.no_grad():
            c.weight.copy_(c.weight.float().double())
    bns = _bns(widths[1:], 2, True, 0.1, gen)
    ref_bns = [nn.BatchNorm2d(c).double() for c in widths[1:]]
    for r, b in zip(ref_bns, bns):
        r.load_state_dict(b.state_dict())
        r.train(train)
    g = gidx.long().clamp(max=N - 1)
    bi = torch.arange(B).view(B, 1, 1)
    rel = xyz[bi, g] - new_xyz.view(B, S, 1, 3)
    grouped = rel if D == 0 else (torch.cat([rel, feats[bi, g]], -1) if xyz_first else torch.cat([feats[bi, g], rel], -1))
    grouped[(gidx == N)] = 0.0
    h = grouped.double().permute(0, 3, 2, 1)                                         # (B, C, K, S)
    for l, (c, bn) in enumerate(zip(convs, ref_bns)):
        h = F.relu(bn(c(h)))
    want = h.max(dim=2)[0]
    first = {"mode": 1, "rows_per_batch": S * K, "xyz": xyz, "feats": feats, "new_xyz": new_xyz, "gidx": gidx, "N": N, "S": S,
             "K": K, "D": D, "xyz_first": xyz_first}
    out, _ = _chain(first, widths, [c.weight.detach().reshape(c.weight.shape[0], -1) for c in convs], [c.bias.detach() for c in convs],
                    bns, train, None, B * S * K, S, group=K)
    assert _close(out, want.detach())


def test_edge_conv_leaky_max_matches_float64_modules():
    """DGCNN form: [x_j - x_i | x_i] from a neighbour index and a strided (B, C, N) view, Conv2d (no bias) + BatchNorm2d +
    LeakyReLU (slope 0.25, a float32 value), max over K; index -1 is a zero row"""
    gen = torch.Generator().manual_seed(23)
    B, C, N, K, cout = 2, 5, 30, 4, 9
    base = torch.randn(B, 2 * C, N, generator=gen)
    x = base[:, ::2]                                                                 # strided channels
    idx = torch.randint(0, N, (B, N, K), generator=gen, dtype=torch.int32)
    idx[1, 3, 2] = -1
    conv = nn.Conv2d(2 * C, cout, 1, bias=False).double()
    with torch.no_grad():
        conv.weight.copy_(conv.weight.float().double())
    bn = _bns([cout], 2, True, 0.1, gen)[0]
    ref = nn.BatchNorm2d(cout).double()
    ref.load_state_dict(bn.state_dict())
    xt = x.transpose(2, 1)
    feat = torch.stack([xt[b][idx[b].long().clamp(min=0)] for b in range(B)])
    cen = xt.unsqueeze(2).expand_as(feat)
    edge = torch.cat((feat - cen, cen), dim=3)
    edge[idx < 0] = 0.0
    want = F.leaky_relu(ref(conv(edge.double().permute(0, 3, 1, 2))), 0.25).max(dim=-1)[0]
    first = {"mode": 2, "rows_per_batch": N * K, "edge_x": base, "edge_stride": (x.stride(0), x.stride(1), x.stride(2)), "edge_C": C,
             "gidx": idx, "N": N, "K": K}
    y = pw_chain.layer_forward(rows=B * N * K, cin=2 * C, cout=cout, weight=conv.weight.detach().reshape(cout, -1), group=K, **first)
    out = pw_chain.apply(src=y["ymax"], ymin=y["ymin"], rows_per_batch=N, channels=cout, affine=1, stats=y["stats"], stat_rows=B * N * K,
                         gamma=bn.weight, beta=bn.bias, eps=bn.eps, act=1, act_slope=0.25)
    assert _close(out, want.detach())
    assert bool((bn.weight < 0).any()) and bool((bn.weight == 0).any())


def test_apply_without_batchnorm_and_cloud_bias():
    """affine = 0 is the identity before the activation; cloud_bias adds one row per cloud after the bias"""
    gen = torch.Generator().manual_seed(5)
    src = torch.randn(3, 8, generator=gen)
    got = pw_chain.apply(src=src, rows_per_batch=4, channels=3, relu=0)
    assert torch.equal(got, src.double().reshape(3, 2, 4).permute(1, 0, 2))
    x = torch.randn(2, 3, 4, generator=gen)
    w, cb = torch.randn(5, 3, generator=gen), torch.randn(2, 5, generator=gen)
    y = pw_chain.layer_forward(rows=8, cin=3, cout=5, weight=w, mode=0, rows_per_batch=4, seg_ptr=(x,), seg_channels=(3, 0),
                               seg_batch_stride=(12, 0), seg_row_stride=(1, 0), seg_chan_stride=(4, 0), cloud_bias=cb)["y"]
    want = torch.einsum("oc,bcn->obn", w.double(), x.double()) + cb.double().t().unsqueeze(2)
    assert _close(y, want.reshape(5, 8))
