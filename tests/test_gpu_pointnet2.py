"""GPU parity of the PointNet++ side: ball query / 3-NN indices bit-exact, set-abstraction and
feature-propagation outputs within 1e-4 relative (fp32) of (a) the CPU oracle on seeded inputs and
(b) fixtures produced by the reference's own python code (tests/golden/ref_torch_*.npz)."""
import os

import numpy as np
import pytest
import torch

from oracle import oracle
from toothgroupnetwork_b200 import _lib as L
from toothgroupnetwork_b200 import clouds
from toothgroupnetwork_b200 import pointnet2_utils as pn2

pytestmark = pytest.mark.gpu
REL_TOL = 1e-4   # north_star: "segmentation logits within 1e-4 rel fp32"
TCW_TOL = 1e-3   # ENGINE_TCW (two bf16 parts per operand, explicit request only): ~1e-5 norm-wise, up to ~5e-4 element-wise
FLOOR = 0.05     # element-wise: |a-b| / max(|b|, FLOOR * max|b|); elements below 5% of the tensor's range get the absolute bound


def tol_of(engine):
    """The automatic path only uses fp32-grade engines (1e-4 element-wise); the bf16x2 wide engine is kept for explicit use."""
    return TCW_TOL if engine == pn2.ENGINE_TCW else REL_TOL


def rel_err(a, b):
    """ELEMENT-WISE relative error (worst element) of a against the reference b, with the stated floor."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    scale = np.abs(b).max() + 1e-30
    return float((np.abs(a - b) / np.maximum(np.abs(b), FLOOR * scale)).max())


@pytest.fixture(autouse=True)
def _reference_on_cpu():
    """The fixtures / oracle of this file restate the reference's functions on CPU tensors, where torch.sum(p ** 2, -1)
    rounds in index order for every layout; tests/test_gpu_reference_live.py covers the CUDA rounding."""
    pn2.set_reference_device("cpu")
    yield
    pn2.set_reference_device("cuda")


def load(golden_dir, name):
    return np.load(os.path.join(golden_dir, name))


def layers_from(fix, n, prefix=""):
    out = []
    for i in range(n):
        t = lambda k: torch.from_numpy(fix[f"{prefix}{k}{i}"])
        out.append(oracle.MlpParams(t("w"), t("b"), t("gamma"), t("beta"), t("mean"), t("var")))
    return out


def fill_module(convs, bns, layers):
    with torch.no_grad():
        for c, b, p in zip(convs, bns, layers):
            c.weight.copy_(p.weight.view_as(c.weight))
            c.bias.copy_(p.bias)
            b.weight.copy_(p.gamma)
            b.bias.copy_(p.beta)
            b.running_mean.copy_(p.mean)
            b.running_var.copy_(p.var)


# ------------------------------------------------------------------------------------ ball query
@pytest.mark.parametrize("r,k", [(0.025, 32), (0.05, 64), (0.1, 32), (0.2, 16)])
def test_ball_query_matches_reference_fixture(golden_dir, r, k):
    fix = load(golden_dir, "ref_torch_ball.npz")
    xyz = torch.from_numpy(fix["xyz"])
    new = xyz[torch.from_numpy(fix["sel"]).long()]
    got = pn2.query_ball_point(r, k, xyz[None].cuda(), new[None].cuda())
    assert got.dtype == torch.int64
    assert np.array_equal(got[0].cpu().numpy(), fix[f"ball_r{r}_k{k}"].astype(np.int64))


def test_ball_query_empty_ball_sentinel(golden_dir):
    fix = load(golden_dir, "ref_torch_ball.npz")
    xyz = torch.from_numpy(fix["xyz"])
    far = torch.tensor([[[5.0, 5.0, 5.0]]])
    got = pn2.query_ball_point(0.1, 8, xyz[None].cuda(), far.cuda())
    assert np.array_equal(got[0].cpu().numpy(), fix["ball_far"].astype(np.int64))


@pytest.mark.parametrize("N,S,r,K", [(24000, 1024, 0.1, 32), (24000, 1024, 0.025, 32), (24000, 1024, 0.05, 64),
                                     (4096, 1024, 0.1, 16), (16384, 4096, 0.1, 64), (65536, 2048, 0.1, 32), (1000, 37, 0.2, 7)])
def test_ball_query_matches_oracle_full_size(N, S, r, K):
    """BASELINE C2/C5 sizes, batch of 2 different clouds, int32 and int64 outputs."""
    xs = [clouds.dental_arch(N, s)[0] for s in (0, 1)]
    fps = [oracle.furthestsampling(x.numpy(), [N], [S]) for x in xs]
    xyz = torch.stack(xs)
    new = torch.stack([x[torch.from_numpy(f).long()] for x, f in zip(xs, fps)])
    want = oracle.query_ball_point(r, K, xyz.numpy(), new.numpy())
    got64 = pn2.query_ball_point(r, K, xyz.cuda(), new.cuda())
    got32 = pn2._ball_query(r, K, xyz.cuda(), new.cuda(), False)
    assert np.array_equal(got64.cpu().numpy(), want)
    assert np.array_equal(got32.cpu().numpy().astype(np.int64), want)


GRID_CASES = [
    # (N, S, r, K, offset, scale)   every case through BOTH kernels, forced
    (24000, 1024, 0.1, 32, 0.0, 1.0),       # bench shape: sparse balls
    (24000, 512, 0.4, 32, 0.0, 1.0),        # dense balls (the estimate would pick the tile kernel)
    (24000, 512, 0.01, 16, 0.0, 1.0),       # mostly empty / tiny balls, padding with the first member
    (9000, 300, 0.1, 64, 40.0, 1.0),        # cloud far from the origin: the expanded form is noisy, members far outside r
    (9000, 300, 2.0, 32, 0.0, 25.0),        # millimetre-like coordinates
    (1000, 64, 0.15, 8, 0.0, 1.0),          # small cloud (grid only when forced)
    (70000, 256, 0.05, 32, 0.0, 1.0),       # large cloud, many bitmap words per lane
    (5000, 100, 5.0, 32, 0.0, 1.0),         # radius larger than the cloud: one cell
]


@pytest.mark.parametrize("N,S,r,K,offset,scale", GRID_CASES)
def test_ball_query_grid_and_tile_kernels_match_oracle(N, S, r, K, offset, scale):
    xs = [clouds.dental_arch(N, s)[0] * scale + offset for s in (4, 5)]
    g = torch.Generator().manual_seed(N + S)
    news = []
    for x in xs:
        q = x[torch.randperm(N, generator=g)[:S]].clone()
        q[: S // 8] += (torch.rand(S // 8, 3, generator=g) - 0.5) * 4 * r        # queries off the surface
        q[0] = x.max(0).values + 3 * r + 1.0                                     # outside the bounding box: empty ball
        news.append(q)
    xyz, new = torch.stack(xs).contiguous(), torch.stack(news).contiguous()
    want = oracle.query_ball_point(r, K, xyz.numpy(), new.numpy())
    for path in (pn2.BALL_GRID, pn2.BALL_TILE, pn2.BALL_AUTO):
        got = pn2._ball_query(r, K, xyz.cuda(), new.cuda(), True, path)
        assert np.array_equal(got.cpu().numpy(), want), f"path {path}"
    got32 = pn2._ball_query(r, K, xyz.cuda(), new.cuda(), False, pn2.BALL_GRID)
    assert np.array_equal(got32.cpu().numpy().astype(np.int64), want)


def test_ball_query_agrees_with_torch_reference_formula_on_device():
    """The reference's own formulation (square_distance + mask + sort) evaluated by torch ON THE
    GPU (cuBLAS fp32, TF32 off): membership must agree pair for pair with the kernel."""
    pn2.set_reference_device("cuda")          # the comparison below IS torch on the GPU (contiguous operands)
    torch.backends.cuda.matmul.allow_tf32 = False
    N, S, r, K = 8192, 512, 0.1, 32
    xyz = clouds.dental_arch(N, 3)[0].cuda()
    new = xyz[torch.randperm(N, generator=torch.Generator().manual_seed(0))[:S].cuda()]
    d = pn2.square_distance(new[None], xyz[None])
    gi = torch.arange(N, device="cuda").view(1, 1, N).repeat(1, S, 1)
    gi[d > r ** 2] = N
    gi = gi.sort(dim=-1)[0][:, :, :K]
    first = gi[:, :, 0:1].repeat(1, 1, K)
    gi[gi == N] = first[gi == N]
    got = pn2.query_ball_point(r, K, xyz[None], new[None])
    assert torch.equal(got, gi)


# ------------------------------------------------------------------------------------ 3-NN / FP
def test_three_nn_matches_oracle_and_fixture(golden_dir):
    fix = load(golden_dir, "ref_torch_fp.npz")
    x1 = torch.from_numpy(fix["xyz1"])
    x2 = x1[torch.from_numpy(fix["fps"]).long()]
    d, i = pn2.three_nn(x1[None].cuda(), x2[None].cuda())
    assert np.array_equal(d[0].cpu().numpy().view(np.uint32), fix["nn3_d"].view(np.uint32))
    ties = (fix["nn3_d"][:, 0] == fix["nn3_d"][:, 1]) | (fix["nn3_d"][:, 1] == fix["nn3_d"][:, 2])
    assert np.array_equal(i[0].cpu().numpy()[~ties], fix["nn3_idx"][~ties])
    wd, wi = oracle.three_nn(x1[None].numpy(), x2[None].numpy())
    assert np.array_equal(i.cpu().numpy().astype(np.int64), wi) and np.array_equal(d.cpu().numpy(), wd)


def test_three_nn_full_size():
    x1 = clouds.dental_arch(24000, 0)[0]
    fps = oracle.furthestsampling(x1.numpy(), [24000], [1024])
    x2 = x1[torch.from_numpy(fps).long()]
    d, i = pn2.three_nn(x1[None].cuda(), x2[None].cuda())
    wd, wi = oracle.three_nn(x1[None].numpy(), x2[None].numpy())
    assert np.array_equal(i.cpu().numpy().astype(np.int64), wi)
    assert np.array_equal(d.cpu().numpy().view(np.uint32), wd.view(np.uint32))


@pytest.mark.parametrize("mode", ["eval", "train"])
def test_feature_propagation_matches_reference_fixture(golden_dir, mode):
    fix = load(golden_dir, "ref_torch_fp.npz")
    x1 = torch.from_numpy(fix["xyz1"])
    x2 = x1[torch.from_numpy(fix["fps"]).long()]
    fp = pn2.PointNetFeaturePropagation(30, [32, 16]).cuda()
    fill_module(fp.mlp_convs, fp.mlp_bns, layers_from(fix, 2))
    fp.train(mode == "train")
    with torch.no_grad():
        out = fp(x1.t()[None].contiguous().cuda(), x2.t()[None].contiguous().cuda(),
                 torch.from_numpy(fix["points1"]).cuda(), torch.from_numpy(fix["points2"]).cuda())
    assert rel_err(out.cpu().numpy(), fix[f"out_{mode}"]) < REL_TOL


def test_interpolation_forward_backward_bitwise_vs_dense_torch_form():
    """3-NN + inverse-distance interpolation through the CUDA kernels (three_nn, weighted gather with the order-exact
    backward) == the reference's dense formulation (:333-340: square_distance, sort, reciprocal, normalise, weighted sum)
    evaluated by torch on the GPU -- forward values and the gradient wrt the coarse features, bit for bit, including
    fine points that coincide with a coarse one (expanded-form distances of -6e-8 there)."""
    pn2.set_reference_device("cuda")     # the dense form below IS torch on the GPU
    g = torch.Generator().manual_seed(0)
    x1 = clouds.dental_arch(1500, 1)[0].cuda()
    x2 = x1[:200].contiguous()
    p2 = torch.randn(1, 12, 200, generator=g).cuda().requires_grad_(True)
    c1, c2 = x1.t()[None].contiguous(), x2.t()[None].contiguous()
    v1, v2 = c1.permute(0, 2, 1), c2.permute(0, 2, 1)                    # the strided views the module's square_distance sees
    dist, idx = pn2.three_nn(pn2._to_point_major(c1), pn2._to_point_major(c2), pn2._alt(v1) | (pn2._alt(v2) << 1))
    dd, ii = pn2.square_distance(v1, v2).sort(dim=-1)
    assert torch.equal(dist, dd[:, :, :3]) and torch.equal(idx.long(), ii[:, :, :3])
    interp = pn2.three_interpolate(pn2._transpose(p2), dist, idx)        # autograd path
    rec = 1.0 / (dd[:, :, :3] + 1e-8)
    w = rec / rec.sum(2, keepdim=True)
    dense = (p2.permute(0, 2, 1)[0][ii[0, :, :3]] * w[0].unsqueeze(-1)).sum(1)[None]
    assert torch.equal(interp, dense)
    assert torch.equal(pn2.three_interpolate(pn2._transpose(p2).detach(), dist, idx), dense)      # fused no-grad kernel
    go = torch.randn(interp.shape, generator=g).cuda()
    (ga,) = torch.autograd.grad(interp, p2, go)
    (gb,) = torch.autograd.grad(dense, p2, go)
    assert torch.equal(ga, gb)


# ------------------------------------------------------------------------------------ set abstraction
@pytest.mark.parametrize("engine", [pn2.ENGINE_FP32, pn2.ENGINE_TC, pn2.ENGINE_TCW])
def test_set_abstraction_eval_matches_reference_fixture(golden_dir, engine):
    fix = load(golden_dir, "ref_torch_sa.npz")
    feats = torch.from_numpy(fix["feats"]).cuda()
    sa = pn2.PointNetSetAbstraction(128, 0.1, 32, 9, [32, 32, 64], False).cuda().eval()
    fill_module(sa.mlp_convs, sa.mlp_bns, layers_from(fix, 3))
    pn2.set_sa_engine(engine)
    try:
        with torch.no_grad():
            nx, npts = sa(feats[:, :3].contiguous(), feats)
    finally:
        pn2.set_sa_engine(pn2.ENGINE_AUTO)
    assert np.array_equal(nx.cpu().numpy(), fix["new_xyz_eval"])
    assert rel_err(npts.cpu().numpy(), fix["new_points_eval"]) < tol_of(engine)


def test_set_abstraction_train_mode_matches_reference_fixture(golden_dir):
    fix = load(golden_dir, "ref_torch_sa.npz")
    feats = torch.from_numpy(fix["feats"]).cuda()
    sa = pn2.PointNetSetAbstraction(128, 0.1, 32, 9, [32, 32, 64], False).cuda().train()
    fill_module(sa.mlp_convs, sa.mlp_bns, layers_from(fix, 3))
    torch.backends.cudnn.allow_tf32 = False
    with torch.no_grad():
        nx, npts = sa(feats[:, :3].contiguous(), feats)
    assert np.array_equal(nx.cpu().numpy(), fix["new_xyz_train"])
    assert rel_err(npts.cpu().numpy(), fix["new_points_train"]) < REL_TOL


@pytest.mark.parametrize("engine", [pn2.ENGINE_FP32, pn2.ENGINE_TC, pn2.ENGINE_TCW])
def test_set_abstraction_msg_eval_matches_reference_fixture(golden_dir, engine):
    fix = load(golden_dir, "ref_torch_msg.npz")
    feats = torch.from_numpy(fix["feats"]).cuda()
    msg = pn2.PointNetSetAbstractionMsg(128, [0.05, 0.1], [16, 32], 6, [[16, 32], [32, 48]]).cuda().eval()
    for bi in range(2):
        fill_module(msg.conv_blocks[bi], msg.bn_blocks[bi], layers_from(fix, 2, f"br{bi}_"))
    pn2.set_sa_engine(engine)
    try:
        with torch.no_grad():
            nx, npts = msg(feats[:, :3].contiguous(), feats)
    finally:
        pn2.set_sa_engine(pn2.ENGINE_AUTO)
    assert np.array_equal(nx.cpu().numpy(), fix["new_xyz_eval"])
    assert rel_err(npts.cpu().numpy(), fix["new_points_eval"]) < tol_of(engine)


@pytest.mark.parametrize("engine", [pn2.ENGINE_AUTO, pn2.ENGINE_TCW, pn2.ENGINE_FP32])
def test_real_pointnet_pp_sa1_shape_matches_reference_fixture(golden_dir, engine):
    """The real pointnet_pp SA1 (pointnet_pp.py:13: two 9->128->128 branches, K = 32 / 64) against a fixture made
    by the reference's own Python (tests/golden/make_ref_torch_msg128_golden.py).  AUTO takes the wide tensor-core engine."""
    fix = load(golden_dir, "ref_torch_msg128.npz")
    feats = torch.from_numpy(fix["feats"]).cuda()
    msg = pn2.PointNetSetAbstractionMsg(128, [0.05, 0.1], [32, 64], 6, [[128, 128], [128, 128]]).cuda().eval()
    for bi in range(2):
        fill_module(msg.conv_blocks[bi], msg.bn_blocks[bi], layers_from(fix, 2, f"br{bi}_"))
    pn2.set_sa_engine(engine)
    try:
        with torch.no_grad():
            nx, npts = msg(feats[:, :3].contiguous(), feats)
    finally:
        pn2.set_sa_engine(pn2.ENGINE_AUTO)
    assert np.array_equal(nx.cpu().numpy(), fix["new_xyz_eval"])
    assert rel_err(npts.cpu().numpy(), fix["new_points_eval"]) < tol_of(engine)


def test_set_abstraction_msg_train_mode_matches_reference_fixture(golden_dir):
    fix = load(golden_dir, "ref_torch_msg.npz")
    feats = torch.from_numpy(fix["feats"]).cuda()
    msg = pn2.PointNetSetAbstractionMsg(128, [0.05, 0.1], [16, 32], 6, [[16, 32], [32, 48]]).cuda().train()
    for bi in range(2):
        fill_module(msg.conv_blocks[bi], msg.bn_blocks[bi], layers_from(fix, 2, f"br{bi}_"))
    torch.backends.cudnn.allow_tf32 = False
    with torch.no_grad():
        nx, npts = msg(feats[:, :3].contiguous(), feats)
    assert rel_err(npts.cpu().numpy(), fix["new_points_train"]) < REL_TOL


def test_group_all_matches_reference_fixture(golden_dir):
    fix = load(golden_dir, "ref_torch_groupall.npz")
    feats = torch.from_numpy(fix["feats"]).cuda()
    ga = pn2.PointNetSetAbstraction(None, None, None, 9, [16, 32], True).cuda().eval()
    fill_module(ga.mlp_convs, ga.mlp_bns, layers_from(fix, 2))
    with torch.no_grad():
        nx, npts = ga(feats[:, :3].contiguous(), feats.contiguous())
    assert np.array_equal(nx.cpu().numpy(), fix["new_xyz_eval"])
    assert rel_err(npts.cpu().numpy(), fix["new_points_eval"]) < REL_TOL


def _random_layers(widths, seed):
    g = torch.Generator().manual_seed(seed)
    out = []
    for ci, co in zip(widths[:-1], widths[1:]):
        out.append(oracle.MlpParams(torch.randn(co, ci, generator=g) / ci ** 0.5, torch.randn(co, generator=g) * 0.1,
                                    torch.rand(co, generator=g) + 0.5, torch.randn(co, generator=g) * 0.1,
                                    torch.randn(co, generator=g) * 0.1, torch.rand(co, generator=g) + 0.5))
    return out


SA_SHAPES = [
    # (N, S, r, K, D, widths, engine)        BASELINE C2(i) at full size first
    (24000, 1024, 0.1, 32, 6, [32, 32, 64], pn2.ENGINE_TC),
    (24000, 1024, 0.1, 32, 6, [32, 32, 64], pn2.ENGINE_FP32),
    (24000, 1024, 0.1, 32, 6, [32, 32, 64], pn2.ENGINE_TC_HALF),  # the tensor-core engine in half-size CTAs
    (4096, 1024, 0.1, 16, 6, [32, 32, 64], pn2.ENGINE_TCW),       # eight neighbourhoods per tile on the wide engine
    (6000, 1001, 0.1, 32, 6, [32, 32, 64], pn2.ENGINE_TC),        # S not a multiple of 4: partial last tile
    (3000, 300, 0.15, 16, 0, [16], pn2.ENGINE_TC),                # xyz only, single layer
    (5000, 512, 0.1, 32, 13, [20, 40, 24, 60], pn2.ENGINE_TC),    # four layers, odd widths, full 16-channel input
    (4096, 1024, 0.1, 16, 6, [32, 32, 64], pn2.ENGINE_TC),
    (16384, 700, 0.1, 64, 6, [32, 32, 64], pn2.ENGINE_TC),
    (3000, 200, 0.15, 24, 6, [20, 40], pn2.ENGINE_TC),          # K that does not divide 128, odd widths
    (3000, 200, 0.15, 24, 0, [16], pn2.ENGINE_TC),              # xyz only, single layer
    (3000, 200, 0.15, 20, 6, [20, 40], pn2.ENGINE_TC),          # K not a multiple of 8: neighbourhoods split fragment blocks
    (3000, 200, 0.15, 24, 61, [64, 64, 128], pn2.ENGINE_FP32),   # tsg_centroid sa2-like width
    (2000, 50, 0.3, 200, 6, [32, 48], pn2.ENGINE_FP32),          # K > 128: chunked groups
]


@pytest.mark.parametrize("N,S,r,K,D,widths,engine", SA_SHAPES)
def test_fused_sa_matches_oracle(N, S, r, K, D, widths, engine):
    B = 2
    feats = torch.cat([clouds.arch_features(N, 20), clouds.arch_features(N, 21)], 0)    # (B,6,N)
    if D == 0:
        points = None
    elif D == 6:
        points = feats
    else:
        points = torch.randn(B, D, N, generator=torch.Generator().manual_seed(5))
    xyz = feats[:, :3].contiguous()
    layers = _random_layers([3 + D] + widths, 7)
    want_xyz, want = oracle.set_abstraction(xyz, points, S, r, K, layers)
    sa = pn2.PointNetSetAbstraction(S, r, K, 3 + D, widths, False).cuda().eval()
    fill_module(sa.mlp_convs, sa.mlp_bns, layers)
    pn2.set_sa_engine(engine)
    try:
        with torch.no_grad():
            nx, npts = sa(xyz.cuda(), None if points is None else points.cuda())
    finally:
        pn2.set_sa_engine(pn2.ENGINE_AUTO)
    assert np.array_equal(nx.cpu().numpy(), want_xyz.numpy())
    assert rel_err(npts.cpu().numpy(), want.numpy()) < tol_of(engine)


WIDE_SHAPES = [
    # (N, S, r, K, D, widths)   the wide tensor-core engine (tf32 first layer, bf16x2-split later layers)
    (24000, 1024, 0.05, 64, 6, [128, 128]),          # real pointnet_pp SA1 branch (pointnet_pp.py:13)
    (24000, 1024, 0.025, 32, 6, [128, 128]),
    (6000, 500, 0.1, 16, 6, [64, 64, 128]),          # three layers, partial last tile
    (3000, 200, 0.2, 128, 0, [32, 100]),             # xyz only, K = 128, odd last width
]


@pytest.mark.parametrize("N,S,r,K,D,widths", WIDE_SHAPES)
def test_wide_tensor_core_engine_matches_oracle(N, S, r, K, D, widths):
    B = 2
    feats = torch.cat([clouds.arch_features(N, 30), clouds.arch_features(N, 31)], 0)
    points = feats if D == 6 else None
    xyz = feats[:, :3].contiguous()
    layers = _random_layers([3 + D] + widths, 11)
    want_xyz, want = oracle.set_abstraction(xyz, points, S, r, K, layers)
    sa = pn2.PointNetSetAbstraction(S, r, K, 3 + D, widths, False).cuda().eval()
    fill_module(sa.mlp_convs, sa.mlp_bns, layers)
    outs = {}
    for engine in (pn2.ENGINE_TCW, pn2.ENGINE_FP32):
        pn2.set_sa_engine(engine)
        try:
            with torch.no_grad():
                nx, npts = sa(xyz.cuda(), None if points is None else points.cuda())
        finally:
            pn2.set_sa_engine(pn2.ENGINE_AUTO)
        assert np.array_equal(nx.cpu().numpy(), want_xyz.numpy())
        outs[engine] = npts.cpu().numpy()
        assert rel_err(outs[engine], want.numpy()) < tol_of(engine), f"engine {engine}"
    # the bf16x2 split keeps 16 mantissa bits per operand: ~1e-5 norm-wise against the exact-FMA engine
    a, b = outs[pn2.ENGINE_TCW], outs[pn2.ENGINE_FP32]
    assert float(np.abs(a - b).max() / np.abs(b).max()) < 5e-5


def test_fused_engines_agree_and_auto_prefers_tensor_cores():
    feats = clouds.arch_features(6000, 3).cuda()
    sa = pn2.PointNetSetAbstraction(512, 0.1, 32, 9, [32, 32, 64], False).cuda().eval()
    outs = {}
    for e in (pn2.ENGINE_FP32, pn2.ENGINE_TC, pn2.ENGINE_AUTO):
        pn2.set_sa_engine(e)
        with torch.no_grad():
            outs[e] = sa(feats[:, :3].contiguous(), feats)[1]
    pn2.set_sa_engine(pn2.ENGINE_AUTO)
    # 3xTF32 (~2^-21 per product) against exact FMA: element-wise at the 5 % floor a few 1e-5, norm-wise ~1e-6
    assert rel_err(outs[pn2.ENGINE_TC].cpu().numpy(), outs[pn2.ENGINE_FP32].cpu().numpy()) < 5e-5
    assert torch.equal(outs[pn2.ENGINE_AUTO], outs[pn2.ENGINE_TC])


def test_unsupported_width_falls_back_to_unfused_cuda_path_not_cpu():
    """Widths > 128 are outside the fused kernel: the module must still run on CUDA kernels
    (gather + library GEMM), never on the CPU."""
    feats = clouds.arch_features(2048, 3).cuda()
    sa = pn2.PointNetSetAbstraction(64, 0.2, 16, 9, [196, 256], False).cuda().eval()
    before = L.launch_count()
    with torch.no_grad():
        nx, npts = sa(feats[:, :3].contiguous(), feats)
    assert npts.is_cuda and npts.shape == (1, 256, 64) and L.launch_count() > before


def test_sa_training_backward_runs_through_cuda_gather():
    feats = clouds.arch_features(2048, 4).cuda()
    sa = pn2.PointNetSetAbstractionMsg(128, [0.1, 0.2], [16, 32], 6, [[16, 32], [16, 32]]).cuda().train()
    pts = feats.clone().requires_grad_(True)
    nx, npts = sa(feats[:, :3].contiguous(), pts)
    npts.square().mean().backward()
    assert pts.grad is not None and torch.isfinite(pts.grad).all() and float(pts.grad.abs().sum()) > 0
    assert all(p.grad is not None for p in sa.parameters())


def test_state_dict_keys_match_reference_layout():
    sa = pn2.PointNetSetAbstraction(16, 0.1, 8, 9, [8, 8], False)
    msg = pn2.PointNetSetAbstractionMsg(16, [0.1], [8], 6, [[8]])
    fp = pn2.PointNetFeaturePropagation(12, [8])
    assert "mlp_convs.0.weight" in sa.state_dict() and "mlp_bns.1.running_var" in sa.state_dict()
    assert "conv_blocks.0.0.weight" in msg.state_dict() and "bn_blocks.0.0.running_mean" in msg.state_dict()
    assert "mlp_convs.0.weight" in fp.state_dict() and fp.state_dict()["mlp_convs.0.weight"].dim() == 3


@pytest.mark.parametrize("shape", [(2, 3, 1000), (2, 1000, 3), (2, 6, 24000), (1, 24000, 6), (3, 40, 70), (1, 8, 300), (2, 1, 5)])
def test_transpose_kernels(shape):
    x = torch.randn(*shape, generator=torch.Generator().manual_seed(0)).cuda()
    assert torch.equal(pn2.transpose_last2(x), x.permute(0, 2, 1).contiguous())


def test_farthest_point_sample_wrapper_and_index_points():
    xyz = torch.stack([clouds.cube(5000, 1), clouds.cube(5000, 2)]).cuda()
    idx = pn2.farthest_point_sample(xyz, 256)
    want = oracle.farthest_point_sample(xyz.cpu().numpy(), 256)
    assert idx.dtype == torch.int64 and np.array_equal(idx.cpu().numpy(), want)
    got = pn2.index_points(xyz, idx)
    assert torch.equal(got, torch.gather(xyz, 1, idx.unsqueeze(-1).expand(-1, -1, 3)))
