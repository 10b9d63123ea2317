"""Pins oracle/scatter.py -- the restatement of one launch of the gather family's backwards and forwards -- against float64
torch and against torch's own float32 autograd on the CPU, where index_put_(accumulate=True) adds sequentially in ascending
source position.  The CUDA order for c == 1 (torch's stride_1 kernel) is pinned here against a lane-by-lane restatement of
that kernel, and on the GPU against torch itself (tests/test_gpu_scatter.py)."""
import numpy as np
import pytest
import torch

from oracle import scatter as S


def spread(shape, seed):
    """randn * 10^U(-3, 3): magnitudes that make the summation order show in the bits"""
    g = np.random.default_rng(seed)
    return (g.standard_normal(shape) * 10.0 ** g.uniform(-3, 3, shape)).astype(np.float32)


def keys_with_degrees(n_rows, degrees, seed, hot=0):
    """a shuffled key vector in which row r occurs degrees[r % len(degrees)] times (plus one hot row of `hot` keys)"""
    g = np.random.default_rng(seed)
    d = np.asarray([degrees[r % len(degrees)] for r in range(n_rows)])
    if hot:
        d[n_rows // 2] = hot
    keys = np.repeat(np.arange(n_rows), d)
    return keys[g.permutation(keys.shape[0])].astype(np.int32)


def torch_gather_grad(x_shape, keys, go, dtype):
    x = torch.zeros(x_shape, dtype=dtype, requires_grad=True)
    x[torch.from_numpy(keys.astype(np.int64))].backward(torch.from_numpy(go).to(dtype))
    return x.grad.numpy()


def lane_by_lane_stride1(terms):
    """torch's indexing_backward_kernel_stride_1 for one row, lane by lane (float32)"""
    d = len(terms)
    passes = d // 32
    lanes = [np.float32(0.0)] * 32
    for i in range(passes):
        for L in range(32):
            lanes[L] = np.float32(lanes[L] + terms[32 * i + L])
    for off in (16, 8, 4, 2, 1):
        lanes = [np.float32(lanes[L] + lanes[L + off]) if L + off < 32 else np.float32(lanes[L] + lanes[L]) for L in range(32)]
    g = lanes[0]
    for j in range(passes * 32, d):
        g = np.float32(g + terms[j])
    return np.float32(np.float32(0.0) + g)


def test_inverse_is_a_stable_argsort_that_drops_out_of_range_keys():
    keys = np.array([3, 0, 3, -1, 5, 0, 3, 7, 2, 3], np.int32)      # 5 and 7 are >= n_rows, -1 is negative
    row_start, order = S.inverse(keys, 5)
    assert row_start.tolist() == [0, 2, 2, 3, 7, 7]                 # rows 1 and 4: d = 0
    assert order.tolist() == [1, 5, 8, 0, 2, 6, 9]


@pytest.mark.parametrize("c", [1, 3, 32, 33])
@pytest.mark.parametrize("degrees,hot", [((0, 1, 31, 32, 33, 64), 0), ((2, 0, 5), 1200)])
def test_gather_backward_against_torch(c, degrees, hot):
    n_rows = 70
    keys = keys_with_degrees(n_rows, degrees, 1, hot)
    go = spread((keys.shape[0], c), 2)
    s = S.gather_backward(go, keys, n_rows, order="seq")
    np.testing.assert_allclose(s.f64, torch_gather_grad((n_rows, c), keys, go, torch.float64), rtol=1e-13, atol=0)
    assert np.array_equal(s.mag, torch_gather_grad((n_rows, c), keys, np.abs(go), torch.float64))
    assert np.array_equal(s.d[:, 0], np.bincount(keys, minlength=n_rows))
    # float32, sequential in ascending position: torch's CPU index_add_ bit for bit, and its CPU autograd for rows narrower than
    # 31 elements (wider rows take another summation order in torch's CPU index_put)
    x = torch.zeros(n_rows, c).index_add_(0, torch.from_numpy(keys.astype(np.int64)), torch.from_numpy(go))
    assert np.array_equal(s.f32.view(np.int32), x.numpy().view(np.int32))
    if c < 31:
        assert np.array_equal(s.f32.view(np.int32), torch_gather_grad((n_rows, c), keys, go, torch.float32).view(np.int32))
    assert np.all(s.f32[s.d == 0] == 0)
    # the magnitude bound holds for sums in both directions, and the two directions differ somewhere
    rev = S.index_put_f32(go, keys, n_rows, order="rev")
    for got in (s.f32, rev):
        assert np.all(np.abs(got - s.f64) <= S.bound(s))
    assert not np.array_equal(rev, s.f32)


def test_out_of_range_keys_are_dropped():
    keys = keys_with_degrees(40, (3, 0, 40), 3)
    bad = keys.copy()
    g = np.random.default_rng(4)
    sel = g.choice(keys.shape[0], 25, replace=False)
    bad[sel[:10]] = -1 - g.integers(0, 5, 10)
    bad[sel[10:]] = 40 + g.integers(0, 5, 15)
    go = spread((keys.shape[0], 5), 5)
    keep = (bad >= 0) & (bad < 40)
    s = S.gather_backward(go, bad, 40, order="seq")
    assert np.array_equal(s.f32, torch_gather_grad((40, 5), bad[keep], go[keep], torch.float32))
    np.testing.assert_allclose(s.f64, torch_gather_grad((40, 5), bad[keep], go[keep], torch.float64), rtol=1e-13)
    assert np.array_equal(s.d[:, 0], np.bincount(bad[keep], minlength=40))
    assert np.array_equal(S.index_put_f32(go, bad, 40, "cuda"), S.index_put_f32(go[keep], bad[keep], 40, "cuda"))


@pytest.mark.parametrize("d", [0, 1, 5, 31, 32, 33, 63, 64, 65, 100, 1100])
def test_stride1_order_lane_by_lane(d):
    keys = np.zeros(d, np.int32)
    go = spread((d, 1), 10 + d)
    got = S.index_put_f32(go, keys, 2, "cuda")
    assert got[1, 0] == 0 and got.dtype == np.float32
    want = lane_by_lane_stride1(go[:, 0])
    assert got[0, 0].view(np.int32) == want.view(np.int32)
    seq = S.index_put_f32(go, keys, 2, "seq")
    if d < 32:
        assert got[0, 0].view(np.int32) == seq[0, 0].view(np.int32)


def test_stride1_order_differs_from_sequential_for_32_or_more():
    keys = keys_with_degrees(200, (32, 33, 64, 100), 11)
    go = spread((keys.shape[0], 1), 12)
    cuda, seq = S.index_put_f32(go, keys, 200, "cuda"), S.index_put_f32(go, keys, 200, "seq")
    assert not np.array_equal(cuda, seq)
    s = S.gather_backward(go, keys, 200)
    assert np.all(np.abs(cuda - s.f64) <= S.bound(s))


def loop_torch(feat, idx, w, go, dtype):
    """pointops.interpolation's forward as the reference writes it (pointops.py:177-179), under autograd"""
    f = torch.from_numpy(feat).to(dtype).requires_grad_(True)
    it, wt = torch.from_numpy(idx.astype(np.int64)), torch.from_numpy(w).to(dtype)
    new_feat = torch.zeros(idx.shape[0], feat.shape[1], dtype=dtype)
    for i in range(idx.shape[1]):
        new_feat += f[it[:, i], :] * wt[:, i].unsqueeze(-1)
    new_feat.backward(torch.from_numpy(go).to(dtype))
    return new_feat.detach().numpy(), f.grad.numpy()


def sum_torch(p2, idx, w, go, dtype):
    """three_interpolate as pointnet2_utils.py:340 writes it: torch.sum(index_points(points2, idx) * weight.view(B, N, 3, 1), 2)"""
    B, N, k = idx.shape
    p = torch.from_numpy(p2).to(dtype).requires_grad_(True)
    bi = torch.arange(B).view(B, 1, 1).expand(B, N, k)
    out = torch.sum(p[bi, torch.from_numpy(idx.astype(np.int64)), :] * torch.from_numpy(w).to(dtype).view(B, N, k, 1), 2)
    out.backward(torch.from_numpy(go).to(dtype))
    return out.detach().numpy(), p.grad.numpy()


@pytest.mark.parametrize("k", [1, 3, 8, 9])
@pytest.mark.parametrize("c", [1, 4, 17])
def test_weighted_loop_order_against_torch(k, c):
    m, n = 50, 400
    g = np.random.default_rng(20 + k)
    idx = g.integers(0, m, (n, k)).astype(np.int32)
    idx[: n // 2, 0] = 7                                                # a hot row
    feat, w, go = spread((m, c), 21), g.random((n, k)).astype(np.float32), spread((n, c), 22)
    s = S.weighted_backward(go, idx, w, m, mode="loop", order="seq")
    out32, grad32 = loop_torch(feat, idx, w, go, torch.float32)
    assert np.array_equal(s.f32.view(np.int32), grad32.view(np.int32))
    out64, grad64 = loop_torch(feat, idx, w, go, torch.float64)
    np.testing.assert_allclose(s.f64, grad64, rtol=1e-12, atol=1e-300)
    assert np.all(np.abs(s.f32 - s.f64) <= S.bound(s))
    f64, mag, d = S.weighted_forward(feat, idx, w)
    np.testing.assert_allclose(f64, out64, rtol=1e-12, atol=1e-300)
    assert np.all(np.abs(out32 - f64) <= (d + 1) * S.U32 * mag)
    if k > 1:       # the k results summed the other way round are not torch's
        other = None
        for i in range(k):
            gi = S.index_put_f32(go * w[:, i:i + 1], idx[:, i], m, "seq")
            other = gi if other is None else other + gi
        assert not np.array_equal(other, s.f32)


@pytest.mark.parametrize("c", [1, 5, 16])
def test_weighted_single_order_against_torch(c):
    B, S_, N = 2, 40, 300
    g = np.random.default_rng(30 + c)
    idx = g.integers(0, S_, (B, N, 3)).astype(np.int32)
    idx[0, :, 1] = 3                                                    # a hot row in cloud 0
    p2, w, go = spread((B, S_, c), 31), g.random((B, N, 3)).astype(np.float32), spread((B, N, c), 32)
    flat = (idx + (np.arange(B) * S_).reshape(B, 1, 1)).reshape(B * N, 3)
    s = S.weighted_backward(go.reshape(B * N, c), flat, w.reshape(B * N, 3), B * S_, mode="sum", order="seq")
    _, grad32 = sum_torch(p2, idx, w, go, torch.float32)
    assert np.array_equal(s.f32.view(np.int32), grad32.reshape(B * S_, c).view(np.int32))
    _, grad64 = sum_torch(p2, idx, w, go, torch.float64)
    np.testing.assert_allclose(s.f64, grad64.reshape(B * S_, c), rtol=1e-12, atol=1e-300)


@pytest.mark.parametrize("c", [1, 6])
def test_subtraction_backward_against_torch(c):
    n, n2, ns = 300, 90, 16
    g = np.random.default_rng(40)
    idx = g.integers(0, n2, (n, ns)).astype(np.int32)
    idx[:, 0] = 5
    go = spread((n, ns, c), 41)
    a = torch.zeros(n, c, dtype=torch.float64, requires_grad=True)
    b = torch.zeros(n2, c, dtype=torch.float64, requires_grad=True)
    (a.unsqueeze(1) - b[torch.from_numpy(idx.astype(np.int64))]).backward(torch.from_numpy(go).double())
    g1, g2 = S.subtraction_backward(idx, go, n2)
    np.testing.assert_allclose(g1.f64, a.grad.numpy(), rtol=1e-13, atol=1e-300)
    np.testing.assert_allclose(g2.f64, b.grad.numpy(), rtol=1e-13, atol=1e-300)
    assert np.all(g1.d == ns) and np.array_equal(g2.d[:, 0], np.bincount(idx.reshape(-1), minlength=n2))


@pytest.mark.parametrize("c,w_c", [(1, 1), (6, 1), (6, 4), (6, 6), (35, 4)])
def test_aggregation_against_torch(c, w_c):
    n, ns = 120, 16
    g = np.random.default_rng(50 + c + w_c)
    idx = g.integers(0, n, (n, ns)).astype(np.int32)
    idx[:, 3] = 9
    inp, pos, w, go = spread((n, c), 51), spread((n, ns, c), 52), spread((n, ns, w_c), 53), spread((n, c), 54)
    ti, tp, tw = (torch.from_numpy(a).double().requires_grad_(True) for a in (inp, pos, w))
    ch = torch.arange(c) % w_c
    out = ((ti[torch.from_numpy(idx.astype(np.int64))] + tp) * tw[:, :, ch]).sum(1)
    out.backward(torch.from_numpy(go).double())
    gi, gp, gw = S.aggregation_backward(inp, pos, w, idx, go)
    np.testing.assert_allclose(gi.f64, ti.grad.numpy(), rtol=1e-12, atol=1e-300)
    np.testing.assert_allclose(gw.f64, tw.grad.numpy(), rtol=1e-12, atol=1e-300)
    assert np.array_equal(gp, (torch.from_numpy(go)[:, None, :] * torch.from_numpy(w)[:, :, ch]).numpy())
    assert np.all(gw.d.sum(-1) == c)
    f64, mag, d = S.aggregation_forward(inp, pos, w, idx)
    np.testing.assert_allclose(f64, out.detach().numpy(), rtol=1e-12, atol=1e-300)
    assert np.all(mag >= np.abs(f64)) and np.all(d == ns)
