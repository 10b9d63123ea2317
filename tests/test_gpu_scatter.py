"""The gather family one launch at a time.

* Order-exact backwards (csrc/csr.cu): bit for bit against torch's own autograd of the reference's formulation on the same
  device -- ``x[idx]``, ``points[batch_indices, idx, :]``, pointops.interpolation's ``new_feat += feat[idx[:, i]] * w[:, i:i+1]``
  loop and ``torch.sum(index_points(p2, idx) * w.view(B, N, 3, 1), 2)``.  Gradients span six decades, and every case also
  checks that the same sums taken in reverse order differ from torch's somewhere, so the bitwise check cannot pass by luck.
* Atomic backwards (csrc/gather.cu): element-wise against float64, |got - S64| <= (d + 1) * 2^-24 * sum |t_i| (oracle/scatter.py).
* Forwards: bitwise against torch on the device or the C oracle, with c % 4 != 0, c == 1 and a base pointer one float off
  16-byte alignment (which must equal the aligned call bit for bit).
* Refusals raise TgnError."""
import numpy as np
import pytest
import torch

from oracle import oracle
from oracle import scatter as S
from toothgroupnetwork_b200 import _lib as L
from toothgroupnetwork_b200 import clouds, pointops, pointops_cuda
from toothgroupnetwork_b200 import pointnet2_utils as pn2

pytestmark = pytest.mark.gpu

WORST = {}          # entry point -> worst err / bound seen, printed at the end of the module


@pytest.fixture(scope="module", autouse=True)
def report_worst():
    yield
    for name, r in sorted(WORST.items()):
        print(f"\nworst err/bound {name}: {r:.3g}")


def check_bound(name, got, s: S.Scatter):
    got = got.detach().cpu().double().numpy().reshape(s.f64.shape)
    err = np.abs(got - s.f64)
    b = S.bound(s)
    assert np.all(err <= b), f"{name}: worst err/bound {float(np.max(err / np.maximum(b, 1e-300))):.3g}"
    nz = b > 0
    if nz.any():
        WORST[name] = max(WORST.get(name, 0.0), float(np.max(err[nz] / b[nz])))


def spread(shape, seed):
    g = np.random.default_rng(seed)
    return torch.from_numpy((g.standard_normal(shape) * 10.0 ** g.uniform(-3, 3, shape)).astype(np.float32))


def keys_with_degrees(n_rows, degrees, seed, hot=0):
    g = np.random.default_rng(seed)
    d = np.asarray([degrees[r % len(degrees)] for r in range(n_rows)])
    if hot:
        d[n_rows // 2] = hot
    keys = np.repeat(np.arange(n_rows), d)
    return torch.from_numpy(keys[g.permutation(keys.shape[0])].astype(np.int32))


def bits(t):
    return t.detach().contiguous().view(torch.int32)


def same_bits(a, b):
    return torch.equal(bits(a), bits(b))


def unaligned(t):
    """a contiguous copy of t whose base address is 4 bytes past a 16-byte boundary"""
    buf = torch.empty(t.numel() + 1, dtype=t.dtype, device="cuda")
    u = buf[1:].view(t.shape)
    u.copy_(t)
    assert u.data_ptr() % 16 == 4
    return u


@pytest.fixture
def atomics():
    pointops.set_deterministic_backward(False)
    yield
    pointops.set_deterministic_backward(True)


def torch_gather_grad(n_rows, keys, go):
    """grad of x[keys] by torch on CUDA, and the same sums in descending position"""
    x = torch.zeros(n_rows, go.shape[-1], device="cuda", requires_grad=True)
    x[keys.long()].backward(go)
    rev = torch.zeros(n_rows, go.shape[-1], device="cuda").index_put_((keys.long().flip(0),), go.flip(0), accumulate=True)
    return x.grad, rev


# ================================================================================================ order-exact backwards
C_EXACT = [1, 2, 3, 4, 31, 32, 33, 64, 131]


@pytest.mark.parametrize("n_rows", [1, 1023, 1024, 1025, 2049])
@pytest.mark.parametrize("c", C_EXACT)
def test_grouping_backward_bitwise_vs_torch(c, n_rows):
    """degrees 0, 1, 31, 32, 33, 64 and one row of 1 100; rows around the scan's 1024-row chunks"""
    keys = keys_with_degrees(n_rows, (0, 1, 31, 32, 33, 64), n_rows + c, hot=1100)
    go = spread((keys.shape[0], 1, c), c).cuda()
    x = torch.zeros(n_rows, c, device="cuda", requires_grad=True)
    out = pointops.grouping(x, keys.view(-1, 1).cuda())
    out.backward(go)
    want, rev = torch_gather_grad(n_rows, keys.cuda(), go.view(-1, c))
    assert same_bits(x.grad, want)
    assert not same_bits(rev, want)
    # the restatement's order is torch's (for c == 1 the order of torch's stride_1 kernel)
    s = S.gather_backward(go.cpu().numpy(), keys.numpy(), n_rows)
    assert np.array_equal(s.f32.view(np.int32), bits(want).cpu().numpy())
    check_bound("gather_backward_det", x.grad, s)


@pytest.mark.parametrize("c", [1, 4, 33])
def test_grouping_backward_bitwise_384000_rows(c):
    """375 chunks of the scan's carry; a hot row of 1 500"""
    n_rows = 384000
    keys = keys_with_degrees(n_rows, (0, 1, 2, 3, 33), 7, hot=1500).cuda()
    go = spread((keys.shape[0], c), 8).cuda()
    x = torch.zeros(n_rows, c, device="cuda", requires_grad=True)
    pointops.grouping(x, keys.view(-1, 1)).backward(go.view(-1, 1, c))
    want, rev = torch_gather_grad(n_rows, keys, go)
    assert same_bits(x.grad, want) and not same_bits(rev, want)


@pytest.mark.parametrize("K", [16, 36])
@pytest.mark.parametrize("c", [1, 3, 32])
def test_grouping_backward_bitwise_knn_indices(K, c):
    """kNN of a dental arch in itself: the index tensors a transformer level groups with"""
    xyz = clouds.dental_arch(24000, 3)[0].cuda()
    o = torch.tensor([24000], dtype=torch.int32, device="cuda")
    idx, _ = pointops.knn_packed(K, xyz, xyz, o, o)
    go = spread((24000, K, c), K + c).cuda()
    x = torch.zeros(24000, c, device="cuda", requires_grad=True)
    pointops.grouping(x, idx).backward(go)
    want, rev = torch_gather_grad(24000, idx.reshape(-1), go.view(-1, c))
    assert same_bits(x.grad, want) and not same_bits(rev, want)


def torch_index_points_grad(points_shape, idx, go):
    B = points_shape[0]
    p = torch.zeros(points_shape, device="cuda", requires_grad=True)
    bi = torch.arange(B, device="cuda").view(B, *([1] * (idx.dim() - 1))).expand_as(idx)
    p[bi, idx.long(), :].backward(go)
    flat = (idx.long() + torch.arange(B, device="cuda").view(B, *([1] * (idx.dim() - 1))) * points_shape[1]).reshape(-1)
    rev = torch.zeros(B * points_shape[1], points_shape[2], device="cuda").index_put_(
        (flat.flip(0),), go.reshape(-1, points_shape[2]).flip(0), accumulate=True)
    return p.grad, rev.view(points_shape)


@pytest.mark.parametrize("B", [1, 2, 16])
@pytest.mark.parametrize("c", [1, 3, 4, 33])
def test_index_points_backward_bitwise_synthetic(B, c):
    N, M = 1500, 4000
    g = torch.Generator().manual_seed(B * 100 + c)
    idx = torch.randint(0, N, (B, M), generator=g, dtype=torch.int32)
    idx[:, : M // 4] = 17                                            # a hot row in every cloud
    idx = idx.cuda()
    go = spread((B, M, c), B + c).cuda()
    p = torch.zeros(B, N, c, device="cuda", requires_grad=True)
    pn2.index_points(p, idx).backward(go)
    want, rev = torch_index_points_grad((B, N, c), idx, go)
    assert same_bits(p.grad, want) and not same_bits(rev, want)


@pytest.mark.parametrize("B", [1, 2, 16])
@pytest.mark.parametrize("c", [1, 3, 35])
def test_index_points_backward_bitwise_ball_query(B, c):
    """ball query r = 0.025, K = 64 on dental arches: the padding with the first hit makes very hot rows"""
    N, S_ = 24000, 512
    xyz = torch.stack([clouds.dental_arch(N, 40 + b)[0] for b in range(B)]).cuda()
    new_xyz = xyz[:, ::N // S_][:, :S_].contiguous()
    idx = pn2.query_ball_point(0.025, 64, xyz, new_xyz)
    assert int(torch.bincount(idx[0].reshape(-1)).max()) > 32
    go = spread((B, S_, 64, c), B + c).cuda()
    p = torch.zeros(B, N, c, device="cuda", requires_grad=True)
    pn2.index_points(p, idx).backward(go)
    want, rev = torch_index_points_grad((B, N, c), idx, go)
    assert same_bits(p.grad, want) and not same_bits(rev, want)


def torch_loop(feat, idx, w, go):
    """pointops.interpolation's torch loop (pointops.py:177-179) under autograd on CUDA; and the G_i summed in reverse order"""
    f = feat.clone().requires_grad_(True)
    new_feat = torch.zeros(idx.shape[0], feat.shape[1], device="cuda")
    for i in range(idx.shape[1]):
        new_feat += f[idx[:, i].long(), :] * w[:, i].unsqueeze(-1)
    new_feat.backward(go)
    other = None
    for i in range(idx.shape[1]):
        gi = torch.zeros_like(feat).index_put_((idx[:, i].long(),), go * w[:, i:i + 1], accumulate=True)
        other = gi if other is None else other + gi
    return new_feat.detach(), f.grad, other


def three_nn_case(n_coarse, k, seed):
    fine = clouds.dental_arch(24000, seed)[0]
    coarse = fine[torch.randperm(24000, generator=torch.Generator().manual_seed(seed))[:n_coarse]].contiguous()
    o, no = torch.tensor([n_coarse], dtype=torch.int32).cuda(), torch.tensor([24000], dtype=torch.int32).cuda()
    idx, d2 = pointops.knn_packed(k, coarse.cuda(), fine.cuda(), o, no)
    w = pointops._inverse_distance_weights(torch.sqrt(d2)).contiguous()
    return coarse.cuda(), fine.cuda(), o, no, idx, w


@pytest.mark.parametrize("n_coarse", [128, 512])
@pytest.mark.parametrize("k", [1, 3, 8])
@pytest.mark.parametrize("c", [1, 3, 32, 33])
def test_interpolation_loop_backward_bitwise(n_coarse, k, c):
    """k-NN from 24 000 points to 128 / 512: each coarse row gathers hundreds of contributions per index_put"""
    coarse, fine, o, no, idx, w = three_nn_case(n_coarse, k, 5)
    feat = spread((n_coarse, c), k + c).cuda()
    go = spread((24000, c), 2 * k + c).cuda()
    f = feat.clone().requires_grad_(True)
    out = pointops._WeightedGather.apply(f, idx, w, False)
    out.backward(go)
    want_out, want, other = torch_loop(feat, idx, w, go)
    assert same_bits(out, want_out)
    assert same_bits(f.grad, want)
    rev_out, rev, _ = torch_loop(feat, idx.flip(0), w.flip(0), go.flip(0))
    assert not same_bits(rev, want)
    if k > 1:
        assert not same_bits(other, want)
    s = S.weighted_backward(go.cpu().numpy(), idx.cpu().numpy(), w.cpu().numpy(), n_coarse, mode="loop")
    assert np.array_equal(s.f32.view(np.int32), bits(want).cpu().numpy())
    check_bound("weighted_gather_backward_det", f.grad, s)
    # the public function, weights and all
    f2 = feat.clone().requires_grad_(True)
    out2 = pointops.interpolation(coarse, fine, f2, o, no, k)
    out2.backward(go)
    assert same_bits(out2, want_out) and same_bits(f2.grad, want)


@pytest.mark.parametrize("k", [9, 12])
def test_interpolation_loop_backward_k_above_8_uses_atomics(k):
    coarse, fine, o, no, idx, w = three_nn_case(128, k, 6)
    feat = spread((128, 32), k).cuda().requires_grad_(True)
    go = spread((24000, 32), k + 1).cuda()
    pointops._WeightedGather.apply(feat, idx, w, False).backward(go)
    s = S.weighted_backward(go.cpu().numpy(), idx.cpu().numpy(), w.cpu().numpy(), 128)
    check_bound("interpolation_backward (k > 8)", feat.grad, s)
    with pytest.raises(L.TgnError):
        ws = pointops.csr_for(idx, 128)
        gi = torch.empty(128, 32, device="cuda")
        L.call("tgn_weighted_gather_backward_det", idx.numel(), 128, 32, k, 0, L.ptr(ws), L.ptr(go), L.ptr(w), L.ptr(gi), L.stream_ptr())


@pytest.mark.parametrize("B", [1, 2])
@pytest.mark.parametrize("n_coarse", [128, 512])
@pytest.mark.parametrize("c", [1, 3, 32, 33])
def test_three_interpolate_backward_bitwise(B, n_coarse, c):
    """torch.sum(index_points(points2, idx) * weight.view(B, N, 3, 1), dim=2) (pointnet2_utils.py:337-340)"""
    N = 24000
    xyz1 = torch.stack([clouds.dental_arch(N, 60 + b)[0] for b in range(B)]).cuda()
    xyz2 = xyz1[:, ::N // n_coarse][:, :n_coarse].contiguous()
    dist, idx = pn2.three_nn(xyz1, xyz2)
    p2 = spread((B, n_coarse, c), c + B).cuda()
    go = spread((B, N, c), c + B + 1).cuda()
    p = p2.clone().requires_grad_(True)
    out = pn2.three_interpolate(p, dist, idx)
    out.backward(go)
    rec = 1.0 / (dist + 1e-8)
    weight = rec / torch.sum(rec, dim=2, keepdim=True)
    q = p2.clone().requires_grad_(True)
    bi = torch.arange(B, device="cuda").view(B, 1, 1).expand(B, N, 3)
    want_out = torch.sum(q[bi, idx.long(), :] * weight.view(B, N, 3, 1), 2)
    want_out.backward(go)
    flat = (idx.long() + torch.arange(B, device="cuda").view(B, 1, 1) * n_coarse).reshape(-1)
    assert same_bits(p.grad, q.grad)
    if c > 1:       # with C = 1 torch reduces the three products as a contiguous row, in another order than the kernel's
        assert same_bits(out, want_out)
    f64, mag, d = S.weighted_forward(p2.view(-1, c).cpu().numpy(), flat.view(-1, 3).cpu().numpy(), weight.reshape(-1, 3).cpu().numpy())
    check_bound("weighted_gather (sum)", out.view(-1, c), S.Scatter(f64, mag, d))
    terms = (go.view(B, N, 1, c) * weight.view(B, N, 3, 1)).reshape(-1, c)
    rev = torch.zeros(B * n_coarse, c, device="cuda").index_put_((flat.flip(0),), terms.flip(0), accumulate=True)
    assert not same_bits(rev, q.grad.view(-1, c))
    s = S.weighted_backward(go.view(-1, c).cpu().numpy(), flat.view(-1, 3).cpu().numpy(), weight.reshape(-1, 3).cpu().numpy(),
                            B * n_coarse, mode="sum")
    assert np.array_equal(s.f32.view(np.int32), bits(q.grad).view(-1, c).cpu().numpy())


def test_empty_index_gives_zero_gradients():
    """M = 0: the inverse is empty and both backwards write zeros over whatever the buffers held"""
    lib = L.load()
    keys = torch.empty(0, dtype=torch.int32, device="cuda")
    for n_rows, c in ((1, 1), (37, 3), (1500, 32)):
        ws = torch.full((lib.tgn_csr_bytes(0, n_rows),), 0x7F, dtype=torch.uint8, device="cuda")
        L.call("tgn_csr_build", 0, n_rows, L.ptr(keys), L.ptr(ws), L.stream_ptr())
        go = torch.empty(0, c, device="cuda")
        gi = torch.full((n_rows, c), float("nan"), device="cuda")
        L.call("tgn_gather_backward_det", 0, n_rows, c, L.ptr(ws), L.ptr(go), L.ptr(gi), L.stream_ptr())
        assert same_bits(gi, torch.zeros_like(gi))
        for k, single in ((1, 0), (3, 0), (8, 0), (3, 1)):
            gi.fill_(float("nan"))
            L.call("tgn_weighted_gather_backward_det", 0, n_rows, c, k, single, L.ptr(ws), L.ptr(go), L.ptr(go), L.ptr(gi),
                   L.stream_ptr())
            assert same_bits(gi, torch.zeros_like(gi))
    # through autograd: an empty grouping / index_points / interpolation still gets its backward
    x = torch.ones(50, 3, device="cuda", requires_grad=True)
    out = pointops.grouping(x, torch.empty(0, 16, dtype=torch.int32, device="cuda"))
    (out.sum() + x.sum()).backward()
    assert torch.equal(x.grad, torch.ones_like(x))
    p = torch.ones(2, 50, 3, device="cuda", requires_grad=True)
    (pn2.index_points(p, torch.empty(2, 0, dtype=torch.int64, device="cuda")).sum() + p.sum()).backward()
    assert torch.equal(p.grad, torch.ones_like(p))
    f = torch.ones(50, 1, device="cuda", requires_grad=True)
    e = torch.empty(0, 3, device="cuda")
    (pointops._WeightedGather.apply(f, torch.empty(0, 3, dtype=torch.int32, device="cuda"), e, False).sum() + f.sum()).backward()
    assert torch.equal(f.grad, torch.ones_like(f))


def test_csr_cache_misses_after_an_in_place_change():
    n = 3000
    idx = torch.randint(0, n, (4000, 16), generator=torch.Generator().manual_seed(1), dtype=torch.int32).cuda()
    go = spread((4000, 16, 5), 2).cuda()
    x = torch.zeros(n, 5, device="cuda", requires_grad=True)
    pointops.grouping(x, idx).backward(go)
    assert same_bits(x.grad, torch_gather_grad(n, idx.reshape(-1), go.view(-1, 5))[0])
    idx.copy_(torch.randint(0, n // 2, (4000, 16), generator=torch.Generator().manual_seed(3), dtype=torch.int32).cuda())
    x.grad = None
    pointops.grouping(x, idx).backward(go)
    assert same_bits(x.grad, torch_gather_grad(n, idx.reshape(-1), go.view(-1, 5))[0])
    assert float(x.grad[n // 2:].abs().max()) == 0.0


# ===================================================================================================== atomic backwards
ATOMIC = [  # (c, w_c, nsample, n)
    (1, 1, 16, 3000), (3, 1, 1, 3000), (4, 4, 16, 3000), (6, 4, 64, 1500), (6, 6, 16, 3000), (32, 4, 16, 3000),
    (35, 1, 64, 1500), (35, 35, 16, 3000), (128, 4, 16, 1500), (128, 128, 1, 3000), (3, 4, 16, 3000),
    (32, 4, 16, 20000),     # n * c above 16 * SMs * 256: the grid-stride loop takes more than one step
]


def atomic_idx(n, ns, n2, seed):
    idx = torch.randint(0, n2, (n, ns), generator=torch.Generator().manual_seed(seed), dtype=torch.int32)
    idx[: n // 2, 0] = 11                                            # a hot row with n / 2 contributions
    return idx


@pytest.mark.parametrize("c,w_c,ns,n", ATOMIC)
def test_grouping_backward_atomic(c, w_c, ns, n, atomics):
    idx = atomic_idx(n, ns, 2000, c + ns)
    go = spread((n, ns, c), c).cuda()
    x = torch.zeros(2000, c, device="cuda", requires_grad=True)
    pointops.grouping(x, idx.cuda()).backward(go)
    check_bound("grouping_backward", x.grad, S.gather_backward(go.cpu().numpy(), idx.numpy(), 2000))


@pytest.mark.parametrize("k", [1, 3, 9])
@pytest.mark.parametrize("c,w_c,ns,n", ATOMIC[::2])
def test_interpolation_backward_atomic(c, w_c, ns, n, k):
    m = 700
    idx = atomic_idx(n, k, m, c + k)
    w = torch.rand(n, k, generator=torch.Generator().manual_seed(k)).cuda()
    go = spread((n, c), c + 1).cuda()
    gi = torch.zeros(m, c, device="cuda")
    pointops_cuda.interpolation_backward_cuda(n, c, k, go, idx.cuda(), w, gi)
    check_bound("interpolation_backward", gi, S.weighted_backward(go.cpu().numpy(), idx.numpy(), w.cpu().numpy(), m))
    f = torch.zeros(m, c, device="cuda", requires_grad=True)          # interpolation2's autograd takes the same kernel
    pointops._WeightedGather.apply(f, idx.cuda(), w, True).backward(go)
    check_bound("interpolation_backward", f.grad, S.weighted_backward(go.cpu().numpy(), idx.numpy(), w.cpu().numpy(), m))


@pytest.mark.parametrize("c,w_c,ns,n", ATOMIC)
def test_subtraction_backward(c, w_c, ns, n):
    n2 = 2000
    idx = atomic_idx(n, ns, n2, c + 2 * ns)
    go = spread((n, ns, c), c + 3).cuda()
    a = torch.zeros(n, c, device="cuda", requires_grad=True)
    b = torch.zeros(n2, c, device="cuda", requires_grad=True)
    pointops.subtraction(a, b, idx.cuda()).backward(go)
    g1, g2 = S.subtraction_backward(idx.numpy(), go.cpu().numpy(), n2)
    check_bound("subtraction_backward grad_in1", a.grad, g1)
    check_bound("subtraction_backward grad_in2", b.grad, g2)


@pytest.mark.parametrize("c,w_c,ns,n", ATOMIC)
def test_aggregation_backward(c, w_c, ns, n):
    idx = atomic_idx(n, ns, n, c + w_c)
    inp, pos, w = spread((n, c), 1), spread((n, ns, c), 2), spread((n, ns, w_c), 3)
    go = spread((n, c), 4)
    ti, tp, tw = (t.cuda().requires_grad_(True) for t in (inp, pos, w))
    pointops.aggregation(ti, tp, tw, idx.cuda()).backward(go.cuda())
    gi, gp, gw = S.aggregation_backward(inp.numpy(), pos.numpy(), w.numpy(), idx.numpy(), go.numpy())
    check_bound("aggregation_backward grad_input", ti.grad, gi)
    check_bound("aggregation_backward grad_weight", tw.grad, gw)
    assert np.array_equal(tp.grad.cpu().numpy().view(np.int32), gp.view(np.int32))


# ============================================================================================================ forwards
C_FWD = [1, 3, 4, 6, 32, 35]


@pytest.mark.parametrize("c", C_FWD)
def test_grouping_and_subtraction_forward_bitwise(c):
    n, ns = 3000, 16
    idx = atomic_idx(n, ns, n, c).cuda()
    a, b = spread((n, c), 1).cuda(), spread((n, c), 2).cuda()
    want_g = b[idx.long()]
    want_s = a.unsqueeze(1) - b[idx.long()]
    for bb, aa in ((b, a), (unaligned(b), unaligned(a))):
        assert same_bits(pointops.grouping(bb, idx), want_g)
        assert same_bits(pointops.subtraction(aa, bb, idx), want_s)
    out = unaligned(torch.zeros(n, ns, c, device="cuda"))
    pointops_cuda.grouping_forward_cuda(n, ns, c, b, idx, out)
    assert same_bits(out, want_g)
    out = unaligned(torch.zeros(n, ns, c, device="cuda"))
    pointops_cuda.subtraction_forward_cuda(n, ns, c, a, b, idx, out)
    assert same_bits(out, want_s)


@pytest.mark.parametrize("B", [1, 2, 16])
@pytest.mark.parametrize("c", C_FWD)
def test_gather_rows_forward_bitwise(B, c):
    N, M = 1000, 2500
    idx = torch.randint(0, N, (B, M), generator=torch.Generator().manual_seed(B + c), dtype=torch.int32).cuda()
    p = spread((B, N, c), c).cuda()
    bi = torch.arange(B, device="cuda").view(B, 1).expand(B, M)
    want = p[bi, idx.long(), :]
    assert same_bits(pn2.index_points(p, idx), want)
    for pp in (p, unaligned(p)):
        for out in (torch.empty(B, M, c, device="cuda"), unaligned(torch.empty(B, M, c, device="cuda"))):
            L.call("tgn_gather_rows", B, N, M, c, L.ptr(pp), L.ptr(idx), L.ptr(out), L.stream_ptr())
            assert same_bits(out, want)


@pytest.mark.parametrize("k", [1, 3, 8])
@pytest.mark.parametrize("c", C_FWD)
def test_interpolation_forward(k, c):
    m, n = 700, 3000
    idx = atomic_idx(n, k, m, c + k)
    inp, w = spread((m, c), 1), torch.rand(n, k, generator=torch.Generator().manual_seed(2))
    f64, mag, d = S.weighted_forward(inp.numpy(), idx.numpy(), w.numpy())
    fused_want = oracle.interpolation_forward(inp.numpy(), idx.numpy(), w.numpy())
    loop_want, _, _ = torch_loop(inp.cuda(), idx.cuda(), w.cuda(), torch.zeros(n, c, device="cuda"))
    for ii, ww in ((inp.cuda(), w.cuda()), (unaligned(inp.cuda()), unaligned(w.cuda()))):
        out = torch.zeros(n, c, device="cuda")
        pointops_cuda.interpolation_forward_cuda(n, c, k, ii, idx.cuda(), ww, out)
        assert np.array_equal(bits(out).cpu().numpy(), fused_want.view(np.int32))
        check_bound("interpolation_forward", out, S.Scatter(f64, mag, d))
        unf = pointops._WeightedGather.apply(ii, idx.cuda(), ww, False)
        assert same_bits(unf, loop_want)
        check_bound("weighted_gather (unfused)", unf, S.Scatter(f64, mag, d))


@pytest.mark.parametrize("c,w_c,ns,n", ATOMIC)
def test_aggregation_forward(c, w_c, ns, n):
    idx = atomic_idx(n, ns, n, c + w_c + 1)
    inp, pos, w = spread((n, c), 5), spread((n, ns, c), 6), spread((n, ns, w_c), 7)
    want = oracle.aggregation_forward(inp.numpy(), pos.numpy(), w.numpy(), idx.numpy())
    f64, mag, d = S.aggregation_forward(inp.numpy(), pos.numpy(), w.numpy(), idx.numpy())
    for ii, pp, ww in ((inp.cuda(), pos.cuda(), w.cuda()), (unaligned(inp.cuda()), unaligned(pos.cuda()), unaligned(w.cuda()))):
        out = pointops.aggregation(ii, pp, ww, idx.cuda())
        assert np.array_equal(bits(out).cpu().numpy(), want.view(np.int32))
        check_bound("aggregation_forward", out, S.Scatter(f64, mag, d))


# ============================================================================================================ refusals
def test_refusals():
    z = torch.zeros(64, device="cuda")
    zi = torch.zeros(64, dtype=torch.int32, device="cuda")
    for w_c in (0, -1):
        with pytest.raises(L.TgnError, match="w_c"):
            L.call("tgn_aggregation_forward", 4, 2, 4, w_c, L.ptr(z), L.ptr(z), L.ptr(z), L.ptr(zi), L.ptr(z), L.stream_ptr())
        with pytest.raises(L.TgnError, match="w_c"):
            L.call("tgn_aggregation_backward", 4, 2, 4, w_c, L.ptr(z), L.ptr(z), L.ptr(z), L.ptr(zi), L.ptr(z), L.ptr(z), L.ptr(z),
                   L.ptr(z), L.stream_ptr())
    ws = torch.zeros(L.load().tgn_csr_bytes(8, 4), dtype=torch.uint8, device="cuda")
    for k in (0, 9, 16):
        with pytest.raises(L.TgnError, match="k="):
            L.call("tgn_weighted_gather_backward_det", 8, 4, 2, k, 0, L.ptr(ws), L.ptr(z), L.ptr(z), L.ptr(z), L.stream_ptr())
    with pytest.raises(L.TgnError, match="B=65536"):
        L.call("tgn_gather_rows", 65536, 1, 1, 1, L.ptr(z), L.ptr(zi), L.ptr(z), L.stream_ptr())
