"""oracle/sa_group.py, the float64 restatement of one tgn_sa_group_mlp_max launch, pinned on the CPU: against the reference
formulation in float64 torch (index_points gather, cat in SSG and MSG channel order, Conv2d(1x1), ReLU, max over K), against the
float64 set-abstraction oracles with BatchNorm folded in float64, on its edge rows, and the soundness of its magnitude bound."""
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle import oracle, sa_group

F64 = torch.float64


def _net(gen, widths, dtype=torch.float32):
    ws = [torch.randn(co, ci, generator=gen, dtype=dtype) / ci ** 0.5 for ci, co in zip(widths[:-1], widths[1:])]
    bs = [torch.randn(co, generator=gen, dtype=dtype) * 0.1 for co in widths[1:]]
    return ws, bs


def _case(gen, B, N, S, K, D, scale=1.0):
    xyz = torch.rand(B, N, 3, generator=gen) * scale
    feats = torch.randn(B, N, D, generator=gen) if D else None
    new_xyz = xyz[:, torch.randperm(N, generator=gen)[:S]].contiguous()
    gidx = torch.randint(0, N, (B, S, K), generator=gen, dtype=torch.int32)
    return xyz, feats, new_xyz, gidx


def _reference(xyz, feats, new_xyz, gidx, xyz_first, ws, bs):
    """pointnet2_utils.py:160-170 / :276-294 in float64 torch, the grouped offsets subtracted in float32 as the module does"""
    B, S, K = gidx.shape
    g_xyz = oracle.index_points(xyz, gidx.long()) - new_xyz.view(B, S, 1, 3)
    if feats is None:
        grouped = g_xyz.to(F64)
    else:
        g_f = oracle.index_points(feats, gidx.long())
        grouped = torch.cat([g_xyz, g_f] if xyz_first else [g_f, g_xyz], -1).to(F64)
    h = grouped.permute(0, 3, 2, 1)                                           # (B, C, K, S)
    for w, b in zip(ws, bs):
        conv = nn.Conv2d(w.shape[1], w.shape[0], 1).double()
        with torch.no_grad():
            conv.weight.copy_(w.to(F64).view(*w.shape, 1, 1))
            conv.bias.copy_(b.to(F64))
            h = F.relu(conv(h))
    return h.max(dim=2)[0]


@pytest.mark.parametrize("D", [0, 1, 6, 13])
@pytest.mark.parametrize("xyz_first", [1, 0])
@pytest.mark.parametrize("widths", [[1], [16, 7], [33, 64, 128], [64, 48, 17, 128]])
@pytest.mark.parametrize("K", [1, 20, 131])
def test_oracle_matches_reference_formulation(D, xyz_first, widths, K):
    gen = torch.Generator().manual_seed(D * 1000 + K + len(widths) * 7 + xyz_first)
    B, N, S = 2, 300, 9
    xyz, feats, new_xyz, gidx = _case(gen, B, N, S, K, D)
    ws, bs = _net(gen, [3 + D] + widths)
    want = _reference(xyz, feats, new_xyz, gidx, xyz_first, ws, bs)
    got, mag = sa_group.group_mlp_max(B, N, S, K, D, xyz, feats, new_xyz, gidx, xyz_first, [3 + D] + widths, ws, bs)
    assert got.dtype == F64 and got.shape == (B, widths[-1], S)
    assert float((got - want).abs().max()) <= 1e-12 * max(1.0, float(want.abs().max()))
    assert bool((mag >= got).all())
    # select: the same neighbourhoods one by one, in the order given
    sel = [(1, 4), (0, 0), (1, 8), (0, 3)]
    g2, m2 = sa_group.group_mlp_max(B, N, S, K, D, xyz, feats, new_xyz, gidx, xyz_first, [3 + D] + widths, ws, bs, select=sel)
    assert torch.equal(g2, torch.stack([got[b, :, s] for b, s in sel]))
    assert torch.equal(m2, torch.stack([mag[b, :, s] for b, s in sel]))


def _layers(gen, widths):
    out = []
    for ci, co in zip(widths[:-1], widths[1:]):
        out.append(oracle.MlpParams(torch.randn(co, ci, generator=gen) / ci ** 0.5, torch.randn(co, generator=gen) * 0.1,
                                    torch.randn(co, generator=gen), torch.randn(co, generator=gen) * 0.1,
                                    torch.randn(co, generator=gen) * 0.1, torch.rand(co, generator=gen) + 0.5))
    return out


def _fold(layers):
    """eval-mode BatchNorm folded into the conv in float64, as the caller of tgn_sa_group_mlp_max does"""
    ws, bs = [], []
    for p in layers:
        scale = p.gamma.to(F64) / torch.sqrt(p.var.to(F64) + p.eps)
        ws.append(p.weight.to(F64) * scale[:, None])
        bs.append((p.bias.to(F64) - p.mean.to(F64)) * scale + p.beta.to(F64))
    return ws, bs


@pytest.mark.parametrize("D,widths", [(0, [16, 32]), (6, [32, 32, 64]), (13, [20, 40, 24, 60])])
def test_oracle_with_folded_batchnorm_matches_set_abstraction(D, widths):
    gen = torch.Generator().manual_seed(11 + D)
    B, N, S, K, r = 2, 1500, 64, 32, 0.15
    feats = torch.cat([torch.cat([oracle_arch(N, 40 + b), torch.randn(1, max(D - 3, 0), N, generator=gen)], 1)
                       for b in range(B)], 0)
    xyz = feats[:, :3].contiguous()
    points = feats[:, 3:3 + D] if D else None
    layers = _layers(gen, [3 + D] + widths)
    new_xyz, want = oracle.set_abstraction(xyz, points, S, r, K, layers, dtype=F64)
    xyz_t, nx_t = xyz.permute(0, 2, 1).contiguous(), new_xyz.permute(0, 2, 1).contiguous()
    gidx = torch.from_numpy(oracle.query_ball_point(r, K, xyz_t.numpy(), nx_t.numpy()))
    ws, bs = _fold(layers)
    pts_t = None if points is None else points.permute(0, 2, 1).contiguous()
    got, _ = sa_group.group_mlp_max(B, N, S, K, D, xyz_t, pts_t, nx_t, gidx, 1, [3 + D] + widths, ws, bs)
    assert float((got - want).abs().max()) <= 1e-12 * float(want.abs().max())


def test_oracle_with_folded_batchnorm_matches_set_abstraction_msg():
    gen = torch.Generator().manual_seed(5)
    B, N, S, D = 2, 1500, 48, 6
    feats = torch.cat([oracle_arch(N, 50 + b) for b in range(B)], 0)
    xyz, points = feats[:, :3].contiguous(), feats
    radii, ks, widths = [0.05, 0.1], [16, 32], [[16, 32], [32, 48]]
    branches = [_layers(gen, [3 + D] + w) for w in widths]
    new_xyz, want = oracle.set_abstraction_msg(xyz, points, S, radii, ks, branches, dtype=F64)
    xyz_t, nx_t, pts_t = (t.permute(0, 2, 1).contiguous() for t in (xyz, new_xyz, points))
    outs = []
    for r, K, w, layers in zip(radii, ks, widths, branches):
        gidx = torch.from_numpy(oracle.query_ball_point(r, K, xyz_t.numpy(), nx_t.numpy()))
        ws, bs = _fold(layers)
        outs.append(sa_group.group_mlp_max(B, N, S, K, D, xyz_t, pts_t, nx_t, gidx, 0, [3 + D] + w, ws, bs)[0])
    got = torch.cat(outs, 1)
    assert float((got - want).abs().max()) <= 1e-12 * float(want.abs().max())


def oracle_arch(n, seed):
    from toothgroupnetwork_b200 import clouds
    return clouds.arch_features(n, seed)


def test_edge_rows():
    gen = torch.Generator().manual_seed(3)
    B, N, S, K, D = 1, 50, 4, 6, 2
    xyz, feats, new_xyz, gidx = _case(gen, B, N, S, K, D)
    widths = [3 + D, 8, 5]
    ws, bs = _net(gen, widths)
    # out-of-range indices (N, a large one, negative ones) give zero rows
    gidx[0, 0] = torch.tensor([N, N + 7, -1, -(2 ** 31), N, N], dtype=torch.int32)
    x = sa_group.operand_rows(N, D, xyz, feats, new_xyz, gidx, 1, torch.tensor([0]), torch.tensor([0]))
    assert torch.equal(x, torch.zeros(1, K, 3 + D))
    got, mag = sa_group.group_mlp_max(B, N, S, K, D, xyz, feats, new_xyz, gidx, 1, widths, ws, bs)
    h = torch.zeros(3 + D, dtype=F64)
    for w, b in zip(ws, bs):
        h = (w.to(F64) @ h + b.to(F64)).clamp(min=0.0)
    assert torch.equal(got[0, :, 0], h)
    # padding with the first hit (query_ball_point :141-143) leaves the max unchanged
    gidx[0, 1] = torch.tensor([7, 9, 30, 7, 7, 7], dtype=torch.int32)
    g2 = gidx.clone()
    g2[0, 1] = torch.tensor([7, 9, 30, 9, 30, 30], dtype=torch.int32)
    a, _ = sa_group.group_mlp_max(B, N, S, K, D, xyz, feats, new_xyz, gidx, 1, widths, ws, bs)
    b, _ = sa_group.group_mlp_max(B, N, S, K, D, xyz, feats, new_xyz, g2, 1, widths, ws, bs)
    assert torch.equal(a[0, :, 1], b[0, :, 1])
    # a last layer that is negative on every row of a neighbourhood gives exactly 0
    bs_neg = bs[:-1] + [torch.full((widths[-1],), -1e3)]
    z, _ = sa_group.group_mlp_max(B, N, S, K, D, xyz, feats, new_xyz, gidx, 1, widths, ws, bs_neg)
    assert torch.equal(z, torch.zeros_like(z))
    # channel order: [xyz_rel | feats] against [feats | xyz_rel]
    x1 = sa_group.operand_rows(N, D, xyz, feats, new_xyz, gidx, 1, torch.tensor([0]), torch.tensor([2]))
    x0 = sa_group.operand_rows(N, D, xyz, feats, new_xyz, gidx, 0, torch.tensor([0]), torch.tensor([2]))
    assert torch.equal(x1[..., :3], x0[..., D:]) and torch.equal(x1[..., 3:], x0[..., :D])


def _fp32_eval(N, D, xyz, feats, new_xyz, gidx, xyz_first, ws, bs):
    B, S, K = gidx.shape
    b = torch.arange(B).repeat_interleave(S)
    s = torch.arange(S).repeat(B)
    x = sa_group.operand_rows(N, D, xyz, feats, new_xyz, gidx, xyz_first, b, s)
    for w, bias in zip(ws, bs):
        x = (x @ w.t() + bias).clamp(min=0.0)
    return x.amax(1).reshape(B, S, -1).permute(0, 2, 1)


@pytest.mark.parametrize("seed", range(6))
def test_magnitude_bounds_fp32_evaluation(seed):
    """Any fp32 evaluation (every dot product of length C within gamma_C) stays inside (C_max + 2) 2^-24 L mag: the bound form
    the GPU tests use is sound before any kernel runs.  Offset clouds and channels spanning 1e-3..1e3 make the cancellation real."""
    gen = torch.Generator().manual_seed(100 + seed)
    B, N, S, K = 2, 400, 24, [1, 7, 32, 64, 129, 16][seed]
    D = [0, 1, 6, 13, 6, 13][seed]
    widths = [[64], [17, 33], [64, 128], [64, 64, 64, 64], [128, 128, 128], [32, 65]][seed]
    xyz, feats, new_xyz, gidx = _case(gen, B, N, S, K, D)
    xyz = xyz + 50.0
    new_xyz = new_xyz + 50.0
    if D:
        feats = feats * torch.logspace(-3, 3, D)
    gidx.view(-1)[::11] = N
    ch = [3 + D] + widths
    ws, bs = _net(gen, ch)
    bs[-1] = bs[-1] - 0.3
    truth, mag = sa_group.group_mlp_max(B, N, S, K, D, xyz, feats, new_xyz, gidx, 1, ch, ws, bs)
    got = _fp32_eval(N, D, xyz, feats, new_xyz, gidx, 1, ws, bs)
    bound = (max(ch) + 2) * 2.0 ** -24 * len(widths) * mag
    err = (got.to(F64) - truth).abs()
    assert bool((err <= bound).all()), float((err / bound.clamp(min=1e-300)).max())
    assert float(err.max()) > 0                                                # the case is not trivially exact
