"""GPU parity against the REFERENCE ITSELF running on the same GPU: the reference's unmodified
``pointnet2_utils.py`` / ``pointops.py`` / ``models/modules/*.py`` (staged as ``oracle/_ref/reference_py.tgz`` by
``__graft_entry__.build()``, or read from /root/reference) on the verbatim ``pointops`` kernels of ``oracle/_ref``.
Skipped when that snapshot is absent.  What the CPU fixtures cannot pin -- the reference's CUDA arithmetic
(cuBLAS K=3 products, the layout-dependent rounding of torch.sum(p ** 2, -1), cuDNN convolutions with batch-statistics
BatchNorm) -- is pinned here, with the call patterns the reference's modules actually use."""
import os
import sys

import numpy as np
import pytest
import torch

from oracle import ref_cuda, ref_models
from toothgroupnetwork_b200 import clouds
from toothgroupnetwork_b200 import pointnet2_utils as pn2

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not (ref_models.available() and ref_cuda.available()), reason="reference snapshot not staged")]
REL_TOL = 1e-4
FLOOR = 0.05      # element-wise |a-b| / max(|b|, FLOOR * max|b|)

_world = {}


def world(ops):
    if ops not in _world:
        _world[ops] = ref_models.World(ops)
    return _world[ops]


def refpn():
    return world("reference").mod("external_libs.pointnet2_utils.pointnet2_utils")


def elementwise(a, b):
    a, b = a.detach().double(), b.detach().double()
    scale = float(b.abs().max()) + 1e-30
    return float(((a - b).abs() / b.abs().clamp(min=FLOOR * scale)).max())


@pytest.fixture(autouse=True)
def _fp32_library_convs():
    saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    pn2.set_reference_device("cuda")
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved


def arch(B, N):
    return torch.stack([clouds.arch_features(N, s)[0] for s in range(B)]).cuda()      # (B,6,N)


# ------------------------------------------------------------------------------------ ball query / 3-NN: indices bit-exact
@pytest.mark.parametrize("B", [1, 16])
@pytest.mark.parametrize("r,K", [(0.025, 32), (0.05, 64), (0.1, 32), (0.2, 64)])
@pytest.mark.parametrize("pattern", ["module", "contiguous"])
def test_ball_query_bit_exact_vs_reference_on_gpu(B, r, K, pattern):
    """``module``: the layouts PointNetSetAbstraction(Msg).forward produces (xyz = permuted view of the (B,3,N) slice of
    the feature tensor, new_xyz = contiguous index_points output); ``contiguous``: both operands contiguous."""
    feats = arch(B, 24000)
    xyz = feats[:, :3, :].permute(0, 2, 1)                                  # view, strides (6N, 1, N)
    with world("reference"):
        fps = refpn().farthest_point_sample(xyz, 1024)
        new_xyz = refpn().index_points(xyz, fps)
        if pattern == "contiguous":
            xyz = xyz.contiguous()
        want = refpn().query_ball_point(r, K, xyz, new_xyz)
    got = pn2.query_ball_point(r, K, xyz, new_xyz)
    bad = int((got != want).any(-1).sum())
    assert bad == 0, f"{bad} of {B * 1024} queries differ"


@pytest.mark.parametrize("pattern", ["views", "contiguous", "mixed"])
def test_square_distance_kernel_bitwise_vs_reference_on_gpu(pattern):
    """pointnet2_utils.square_distance (:20-41) as the losses and tsegnet.get_ddf call it: the kernel against the reference's
    matmul + two reductions on the GPU, for the layouts that change torch's |p|^2 rounding."""
    feats = arch(2, 6000)
    a = feats[:, :3, :].permute(0, 2, 1)                   # strided view (B,N,3)
    b = a[:, :512, :].contiguous()
    if pattern == "contiguous":
        a = a.contiguous()
    elif pattern == "views":
        b = b.permute(0, 2, 1).contiguous().permute(0, 2, 1)
    with world("reference"):
        want = refpn().square_distance(a, b)
    before = pn2.L.launch_count()
    got = pn2.square_distance(a, b)
    assert pn2.L.launch_count() == before + 1
    assert torch.equal(got, want)
    # tsegnet.get_ddf (tsegnet.py:24-33): crops (8,3072,3) as a permuted view against one centre each, (1,8,3).permute(1,0,2)
    crops = feats[:1, :3, :3072].expand(8, 3, 3072).contiguous().permute(0, 2, 1)
    centres = torch.rand(1, 8, 3, device="cuda").permute(1, 0, 2)
    with world("reference"):
        want = refpn().square_distance(crops, centres)
    assert torch.equal(pn2.square_distance(crops, centres), want)
    # under autograd the torch formulation is kept (the losses differentiate through it)
    ag = a.clone().requires_grad_(True)
    pn2.square_distance(ag, b).sum().backward()
    assert ag.grad is not None


@pytest.mark.parametrize("pattern", ["views", "contiguous", "mixed"])
def test_three_nn_bit_exact_vs_reference_on_gpu(pattern):
    feats = arch(2, 24000)
    x1 = feats[:, :3, :].permute(0, 2, 1)
    with world("reference"):
        x2 = refpn().index_points(x1, refpn().farthest_point_sample(x1, 1024))        # contiguous (B,1024,3)
        if pattern == "contiguous":
            x1 = x1.contiguous()
        elif pattern == "views":
            x2 = x2.permute(0, 2, 1).contiguous().permute(0, 2, 1)                    # strided view
        d = refpn().square_distance(x1, x2)
        wd, wi = d.sort(dim=-1)
        wd, wi = wd[:, :, :3], wi[:, :, :3]
    gd, gi = pn2.three_nn(x1, x2)
    assert torch.equal(gd, wd)
    assert torch.equal(gi.long(), wi) or float((torch.gather(d, 2, gi.long()) - wd).abs().max()) == 0.0   # equal distances may swap


def test_three_interpolate_bit_exact_vs_reference_lines_on_gpu():
    """pointnet2_utils.py:333-340 evaluated by torch on the GPU (sort, reciprocal, normalise, weighted sum) against the
    3-NN + interpolation kernels: identical bits, including the normaliser's CUDA reduce order."""
    feats = arch(2, 24000)
    x1 = feats[:, :3, :].permute(0, 2, 1)
    g = torch.Generator(device="cuda").manual_seed(9)
    with world("reference"):
        x2 = refpn().index_points(x1, refpn().farthest_point_sample(x1, 1024))
        p2 = torch.randn(2, 1024, 64, device="cuda", generator=g)
        dists = refpn().square_distance(x1, x2)
        dists, idx = dists.sort(dim=-1)
        dists, idx = dists[:, :, :3], idx[:, :, :3]
        dist_recip = 1.0 / (dists + 1e-8)
        norm = torch.sum(dist_recip, dim=2, keepdim=True)
        weight = dist_recip / norm
        want = torch.sum(refpn().index_points(p2, idx) * weight.view(2, 24000, 3, 1), dim=2)
    gd, gi = pn2.three_nn(x1, x2)
    got = pn2.three_interpolate(p2, gd, gi)
    assert torch.equal(gd, dists)
    bad = int((got != want).sum())
    assert bad == 0, f"{bad} of {got.numel()} interpolated values differ"


# ------------------------------------------------------------------------------------ modules with batch-statistics BatchNorm
def _copy(src, dst):
    dst.load_state_dict(src.state_dict())
    return dst


@pytest.mark.parametrize("train_bn", [True, False])
@pytest.mark.parametrize("B", [1, 3])
def test_set_abstraction_ssg_vs_reference_module(train_bn, B):
    feats = arch(B, 8192)
    xyz = feats[:, :3, :]
    torch.manual_seed(0)
    ours = pn2.PointNetSetAbstraction(512, 0.1, 32, 9, [32, 32, 64], False).cuda().train(train_bn)
    with world("reference"), torch.no_grad():
        ref = _copy(ours, refpn().PointNetSetAbstraction(512, 0.1, 32, 9, [32, 32, 64], False).cuda()).train(train_bn)
        want_xyz, want = ref(xyz, feats)
    before = pn2.L.launch_count()
    with torch.no_grad():
        got_xyz, got = ours(xyz, feats)
    assert pn2.L.launch_count() > before
    assert torch.equal(got_xyz, want_xyz)
    assert elementwise(got, want) < REL_TOL
    if train_bn:      # torch's side effects of a training-mode BatchNorm
        for a, b in zip(ours.mlp_bns, ref.mlp_bns):
            assert elementwise(a.running_mean, b.running_mean) < 1e-4 and elementwise(a.running_var, b.running_var) < 1e-4
            assert int(a.num_batches_tracked) == int(b.num_batches_tracked)


@pytest.mark.parametrize("train_bn", [True, False])
@pytest.mark.parametrize("cfg", [
    (1024, [0.025, 0.05], [32, 64], 6, [[128, 128], [128, 128]]),           # pointnet_pp.py:13 (scale 4)
    (1024, [0.025, 0.05], [32, 64], 6, [[32, 32], [32, 32]]),               # tsg_centroid_module.py:10
    (256, [0.1, 0.2], [32, 64], 6, [[196, 256], [196, 256]]),               # widths of tsg sa3 on raw features
])
def test_set_abstraction_msg_vs_reference_module(train_bn, cfg):
    feats = arch(1, 24000)
    xyz = feats[:, :3, :]
    torch.manual_seed(0)
    ours = pn2.PointNetSetAbstractionMsg(*cfg).cuda().train(train_bn)
    with world("reference"), torch.no_grad():
        ref = _copy(ours, refpn().PointNetSetAbstractionMsg(*cfg).cuda()).train(train_bn)
        want_xyz, want = ref(xyz, feats)
    with torch.no_grad():
        got_xyz, got = ours(xyz, feats)
    assert torch.equal(got_xyz, want_xyz)
    assert got_xyz.stride() == want_xyz.stride()           # same view layout as the reference hands on
    assert elementwise(got, want) < REL_TOL


@pytest.mark.parametrize("train_bn", [True, False])
def test_group_all_wide_vs_reference_module(train_bn):
    """tsg_seg_module.py:26 flatten_sa: PointNetSetAbstraction(None, None, None, 512+3, [256, 512], True) on 256 points."""
    g = torch.Generator(device="cuda").manual_seed(3)
    xyz = torch.rand(2, 3, 256, device="cuda", generator=g)
    pts = torch.randn(2, 512, 256, device="cuda", generator=g)
    torch.manual_seed(0)
    ours = pn2.PointNetSetAbstraction(None, None, None, 515, [256, 512], True).cuda().train(train_bn)
    with world("reference"), torch.no_grad():
        ref = _copy(ours, refpn().PointNetSetAbstraction(None, None, None, 515, [256, 512], True).cuda()).train(train_bn)
        _, want = ref(xyz, pts)
    with torch.no_grad():
        _, got = ours(xyz, pts)
    assert elementwise(got, want) < REL_TOL


@pytest.mark.parametrize("train_bn", [True, False])
@pytest.mark.parametrize("shape", [(24000, 1024, 6, 128, [64, 32]), (512, 256, 512, 1024, [1024, 1024]), (1024, 1, 64, 128, [64])])
def test_feature_propagation_vs_reference_module(train_bn, shape):
    """Against the reference module on the GPU and against the same module evaluated in float64 (the exact answer):
    within 1e-4 of the reference, or -- batch-statistics BatchNorm over few rows amplifies fp32 rounding, and the
    reference's own fp32 run then sits further than 1e-4 from the exact result -- as close to the exact result as the
    reference is (factor 2)."""
    N, S, D1, D2, mlp = shape
    B = 2
    feats = arch(B, N)
    xyz1 = feats[:, :3, :]
    g = torch.Generator(device="cuda").manual_seed(5)
    with world("reference"):
        x1v = xyz1.permute(0, 2, 1)
        if S >= 3:
            new = refpn().index_points(x1v, refpn().farthest_point_sample(x1v, S))
        else:
            new = x1v[:, :1, :].contiguous()
        xyz2 = new.permute(0, 2, 1)                                             # the view a set-abstraction level returns
    p1 = torch.randn(B, D1, N, device="cuda", generator=g)
    p2 = torch.randn(B, D2, S, device="cuda", generator=g)
    torch.manual_seed(0)
    ours = pn2.PointNetFeaturePropagation(D1 + D2, mlp).cuda().train(train_bn)
    with world("reference"), torch.no_grad():
        ref = _copy(ours, refpn().PointNetFeaturePropagation(D1 + D2, mlp).cuda()).train(train_bn)
        state = {k: v.clone() for k, v in ref.state_dict().items()}
        want = ref(xyz1, xyz2, p1, p2)
        ref.load_state_dict(state)
        truth = ref.double()(xyz1.double(), xyz2.double(), p1.double(), p2.double())
    with torch.no_grad():
        got = ours(xyz1, xyz2, p1, p2)
    err, err_ours_t, err_ref_t = elementwise(got, want), elementwise(got, truth), elementwise(want, truth)
    assert err < REL_TOL or err_ours_t <= max(REL_TOL, 2.0 * err_ref_t), (err, err_ours_t, err_ref_t)


def test_feature_propagation_forward_backward_under_autograd_bitwise():
    """Training step through PointNetFeaturePropagation (autograd on): 3-NN, interpolation (CUDA gather with the order-exact
    backward) and the reference's own conv/BN torch code -> output and every gradient bit-identical to the reference module."""
    N, S, D1, D2, mlp = 6000, 512, 6, 64, [32, 16]
    feats = arch(2, N)
    xyz1 = feats[:, :3, :]
    g = torch.Generator(device="cuda").manual_seed(7)
    with world("reference"):
        x1v = xyz1.permute(0, 2, 1)
        xyz2 = refpn().index_points(x1v, refpn().farthest_point_sample(x1v, S)).permute(0, 2, 1)
    p1 = torch.randn(2, D1, N, device="cuda", generator=g)
    p2 = torch.randn(2, D2, S, device="cuda", generator=g)
    torch.manual_seed(0)
    ours = pn2.PointNetFeaturePropagation(D1 + D2, mlp).cuda().train()
    res = {}
    for name in ("reference", "b200"):
        a1, a2 = p1.clone().requires_grad_(True), p2.clone().requires_grad_(True)
        if name == "reference":
            with world("reference"):
                mod = _copy(ours, refpn().PointNetFeaturePropagation(D1 + D2, mlp).cuda()).train()
                out = mod(xyz1, xyz2, a1, a2)
        else:
            mod = ours
            out = mod(xyz1, xyz2, a1, a2)
        out.square().mean().backward()
        res[name] = {"out": out.detach(), "g_p1": a1.grad, "g_p2": a2.grad, **{n: q.grad for n, q in mod.named_parameters()}}
    for k, want in res["reference"].items():
        got = res["b200"][k]
        if k in ("out", "g_p1", "g_p2"):
            assert torch.equal(got, want), (k, float((got - want).abs().max()))
        else:       # cuDNN's weight-gradient kernels are not bit-reproducible run to run; the inputs to them are identical
            assert elementwise(got, want) < 1e-5, k


# ------------------------------------------------------------------------------------ the reference's own blocks.py on both operator sets
def test_real_blocks_transition_down_transformer_layer_transition_up():
    """``models/modules/cbl_point_transformer/blocks.py`` as shipped (TransitionDown :47-79, PointTransformerLayer :14-44,
    TransitionUp :82-111), imported once per operator set; same weights, training-mode BatchNorm, forward + backward."""
    name = "models.modules.cbl_point_transformer.blocks"
    xyz, _, _ = clouds.dental_arch(24000, 2)
    p = xyz.cuda()
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.randn(24000, 32, device="cuda", generator=g)
    o = torch.tensor([24000], dtype=torch.int32, device="cuda")
    outs, grads, state = {}, {}, None
    for ops in ("reference", "b200"):
        w = world(ops)
        with w:
            B = w.mod(name)
            torch.manual_seed(0)
            mods = torch.nn.ModuleDict({"td": B.TransitionDown(32, 64, 4, 24), "pt": B.PointTransformerLayer(64, 64, 8, 24),
                                        "tu": B.TransitionUp(64, 32), "lin": torch.nn.Linear(32, 32)}).cuda()
            if state is None:
                state = {k: v.clone() for k, v in mods.state_dict().items()}
            else:
                mods.load_state_dict(state)
            xin = x.clone().requires_grad_(True)
            p2, x2, o2 = mods["td"]([p, xin, o])
            x3 = mods["pt"]([p2, x2, o2])
            up = mods["tu"]([p, mods["lin"](xin), o], [p2, x3, o2])
            up.square().mean().backward()
            outs[ops] = {"p2": p2, "x2": x2, "o2": o2, "x3": x3, "up": up}
            grads[ops] = {"x": xin.grad.clone(), **{n: q.grad.clone() for n, q in mods.named_parameters() if q.grad is not None}}
    a, b = outs["b200"], outs["reference"]
    assert torch.equal(a["p2"], b["p2"]) and torch.equal(a["o2"], b["o2"])          # FPS indices identical
    for k in ("x2", "x3", "up"):
        assert elementwise(a[k], b[k]) < REL_TOL, k
    # backward: the gathers' scatter-adds follow torch's index_put order (csrc/csr.cu), everything else is the reference's
    # own torch code on bit-identical inputs -> every gradient bit-identical
    for k in ("x2", "x3", "up"):
        assert torch.equal(a[k], b[k]), k
    for k, want in grads["reference"].items():
        got = grads["b200"][k]
        assert torch.equal(got, want), (k, float((got - want).abs().max()), float(want.abs().max()))


@pytest.mark.parametrize("c,K,n", [(32, 36, 24000), (64, 24, 6000), (128, 24, 1500), (512, 24, 93)])
@pytest.mark.parametrize("train_bn", [True, False])
def test_fused_point_transformer_layer_vs_reference_layer(c, K, n, train_bn):
    """blocks.PointTransformerLayer (:14-44) under no_grad: the fused multi-pass kernel (csrc/pt_layer.cu) against the reference's own
    layer on the reference's operators, and against that layer evaluated in float64 with the same neighbour indices."""
    from toothgroupnetwork_b200 import blocks_fused, pointops
    name = "models.modules.cbl_point_transformer.blocks"
    p = clouds.dental_arch(n, 4)[0].cuda()
    g = torch.Generator(device="cuda").manual_seed(2)
    x = torch.randn(n, c, device="cuda", generator=g)
    o = torch.tensor([n], dtype=torch.int32, device="cuda")
    with world("reference"), torch.no_grad():
        Bm = world("reference").mod(name)
        torch.manual_seed(0)
        ref = Bm.PointTransformerLayer(c, c, 8, K).cuda().train(train_bn)
        g2 = torch.Generator().manual_seed(3)
        for b in (ref.linear_p[1], ref.linear_w[0], ref.linear_w[3]):      # non-trivial affine / running statistics
            b.weight.copy_(torch.rand(b.weight.shape, generator=g2) + 0.5)
            b.bias.copy_(torch.randn(b.bias.shape, generator=g2) * 0.1)
            b.running_mean.copy_(torch.randn(b.running_mean.shape, generator=g2) * 0.1)
            b.running_var.copy_(torch.rand(b.running_var.shape, generator=g2) + 0.5)
        state = {k: v.clone() for k, v in ref.state_dict().items()}
        want = ref([p, x, o])
        ref_state_after = {k: v.clone() for k, v in ref.state_dict().items()}
        # float64 truth: same layer, same neighbour indices (kNN on the float32 coordinates)
        ref.load_state_dict(state)
        po = world("reference").mod("external_libs.pointops.functions.pointops")
        saved = po.knnquery
        po.knnquery = lambda k, xyz, new_xyz, off, noff: saved(k, xyz.float().contiguous(), new_xyz.float().contiguous(), off, noff)
        try:
            truth = ref.double()([p.double(), x.double(), o])
        finally:
            po.knnquery = saved
            ref.float()
    with world("b200"), torch.no_grad():
        ours = world("b200").mod(name).PointTransformerLayer(c, c, 8, K).cuda().train(train_bn)
        ours.load_state_dict(state)
        assert blocks_fused.pt_layer_fusable(ours, p, x, o)
        launches = pn2.L.launch_count()
        got = ours([p, x, o])
        assert pn2.L.launch_count() - launches >= 2
    err, e_ours, e_ref = elementwise(got, want), elementwise(got, truth), elementwise(want, truth)
    assert err < REL_TOL or e_ours <= max(REL_TOL, 2.0 * e_ref), (err, e_ours, e_ref)
    if train_bn:
        for k, v in ref_state_after.items():
            if "running" in k:
                assert elementwise(ours.state_dict()[k], v) < 1e-4, k
            if "num_batches_tracked" in k:
                assert int(ours.state_dict()[k]) == int(v)


@pytest.mark.parametrize("train_bn", [True, False])
def test_fused_transition_down_vs_reference(train_bn):
    """blocks.TransitionDown (stride 4, :59-79) under no_grad on the tensor-core layer chain: same sampled points, features within 1e-4 /
    the float64 criterion."""
    name = "models.modules.cbl_point_transformer.blocks"
    p = torch.cat([clouds.dental_arch(6000, 5)[0], clouds.dental_arch(3000, 6)[0]]).cuda()
    g = torch.Generator(device="cuda").manual_seed(4)
    x = torch.randn(9000, 32, device="cuda", generator=g)
    o = torch.tensor([6000, 9000], dtype=torch.int32, device="cuda")
    with world("reference"), torch.no_grad():
        torch.manual_seed(0)
        ref = world("reference").mod(name).TransitionDown(32, 64, 4, 24).cuda().train(train_bn)
        state = {k: v.clone() for k, v in ref.state_dict().items()}
        p_ref, x_ref, o_ref = ref([p, x, o])
    with world("b200"), torch.no_grad():
        ours = world("b200").mod(name).TransitionDown(32, 64, 4, 24).cuda().train(train_bn)
        ours.load_state_dict(state)
        p_new, x_new, o_new = ours([p, x, o])
    assert torch.equal(p_new, p_ref) and torch.equal(o_new, o_ref)
    assert elementwise(x_new, x_ref) < REL_TOL


def test_farthest_point_sample_np_wrapper():
    """pointnet2_utils.farthest_point_sample_np (:103-118; unused by the reference, random start there): numpy in/out,
    deterministic start, same samples as the tensor API."""
    xyz = clouds.dental_arch(6000, 3)[0]
    got = pn2.farthest_point_sample_np(xyz.numpy()[None], 256)
    want = pn2.farthest_point_sample(xyz[None].cuda(), 256).cpu().numpy()
    assert got.dtype == np.int64 and np.array_equal(got, want)


# ------------------------------------------------------------------------------------ whole models (C2-model, C3, C4)
def _model_parity():
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "scripts"))
    import model_parity
    return model_parity


def test_pointnet_pp_model_eval_bn_logits_vs_reference():
    mp = _model_parity()
    feats, _ = mp.make_inputs(24000)
    res = mp.case_pp([world("reference"), world("b200")], feats, False, mp.Timer())
    assert res["indices_identical"]
    assert res["verdict"]["pass"], res["verdict"]


def test_pointnet_pp_model_train_bn_logits_vs_reference():
    mp = _model_parity()
    feats, _ = mp.make_inputs(24000)
    res = mp.case_pp([world("reference"), world("b200")], feats, True, mp.Timer())
    assert res["indices_identical"]
    assert res["verdict"]["pass"], res["verdict"]


def test_tgnet_fps_forward_backward_vs_reference():
    mp = _model_parity()
    feats, labels = mp.make_inputs(24000)
    res = mp.case_tgn([world("reference"), world("b200")], feats, labels, mp.Timer())
    assert res["indices_identical"]
    assert res["tensors"]["nn_crop_indexes"]["bitwise"]
    assert res["verdict"]["pass"], res["verdict"]
    assert res["grads"]["pass"], res["grads"]


def test_tgnet_inference_branch_clusters_and_crops_like_the_reference():
    """The label-free branch of GroupingNetworkModule.forward (grouping_network_module.py:58-73): predicted offsets are clustered
    (ops_utils.get_clustering_labels: DBSCAN + noise vote), the centroids pick the 3072-point crops, the second network runs on them.
    Random weights predict no clusters, so the first network is replaced in BOTH worlds by the same stand-in that 'predicts' the
    foreground mask and offsets of a nearly converged model; everything after it is the reference's code on either operator set:
    scikit-learn + KDTree on the host in one world, csrc/dbscan.cu + csrc/crop_knn.cu in the other."""
    import numpy as np
    mp = _model_parity()
    n = 24000
    xyz, normal, label = clouds.dental_arch(n, 2)
    lab = torch.where(label < 0, torch.zeros_like(label), label).long()
    cent = torch.stack([xyz[lab == c].mean(0) if bool((lab == c).any()) else torch.zeros(3) for c in range(int(lab.max()) + 1)])
    g = torch.Generator().manual_seed(3)
    offset = 0.93 * (cent[lab] - xyz) + 0.003 * torch.randn(n, 3, generator=g)
    stray = torch.rand(n, generator=g) < 0.03
    offset[stray] += 0.08 * torch.randn(int(stray.sum()), 3, generator=g)
    offset[lab == 0] = 0
    sem = torch.stack([(lab == 0).float(), (lab != 0).float()]).unsqueeze(0).cuda()          # (1, 2, n) "logits"
    offset = offset.t().contiguous().unsqueeze(0).cuda()                                     # (1, 3, n)
    feats = torch.cat([xyz, normal], 1).t().contiguous().unsqueeze(0).cuda()

    class Converged(torch.nn.Module):
        def forward(self, inputs):
            return sem, offset, None, None

    outs, state = {}, None
    for w in (world("reference"), world("b200")):
        with w, torch.no_grad():
            torch.manual_seed(0)
            module = w.mod("models.modules.grouping_network_module").GroupingNetworkModule({"model_parameter": dict(mp.TGN_PARAMS)}).cuda()
            if state is None:
                state = {k: v.clone() for k, v in module.state_dict().items()}
            module.load_state_dict(state)
            module.eval()
            module.first_ins_cent_model = Converged()
            if w.ops == "b200":
                assert w.mod("ops_utils").get_clustering_labels.__module__ == "toothgroupnetwork_b200.clustering"
            outs[w.ops] = module([feats])
    ref, new = outs["reference"], outs["b200"]
    assert len(ref["nn_crop_indexes"]) == len(new["nn_crop_indexes"]) == 1
    assert np.array_equal(np.asarray(ref["nn_crop_indexes"][0]), np.asarray(new["nn_crop_indexes"][0]))
    assert np.asarray(ref["nn_crop_indexes"][0]).shape[0] >= 10                               # the teeth were found
    assert torch.equal(ref["cropped_feature_ls"], new["cropped_feature_ls"])
    assert elementwise(new["sem_2"], ref["sem_2"]) < REL_TOL            # (the second network of tgnet_fps has no offset head)
