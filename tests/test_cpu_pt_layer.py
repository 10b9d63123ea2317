"""oracle/pt_layer.py, the float64 restatement of one tgn_pt_layer_forward launch, pinned on the CPU: against blocks.py:31-44
written out in float64 torch with the module's own BatchNorm1d (train and eval, non-default eps and momentum, the running
statistics it leaves), against oracle.point_transformer_layer on the reference's fixture layers, and the soundness of its
error bound for float32 evaluations of the data cases the GPU tests use."""
import numpy as np
import pytest
import torch

from oracle import oracle as O
from oracle import pt_layer
from test_gpu_blocks import GOLD, Layer, _state
from toothgroupnetwork_b200 import clouds

F64 = torch.float64
WORST = {}


def _knn(p, o, K):
    idx, _, _ = O.knnquery(K, p.numpy(), p.numpy(), o.numpy(), o.numpy())
    return torch.from_numpy(np.ascontiguousarray(idx))


def _crops(n_crops, per_crop, seed=0):
    """n_crops dental arches of per_crop points packed into one batch -> p, o"""
    p = torch.cat([clouds.dental_arch(per_crop, seed + k)[0] for k in range(n_crops)]).contiguous()
    return p, torch.arange(1, n_crops + 1, dtype=torch.int32) * per_crop


def _fields(layer, p, xq, xk, xv, idx, modes, update):
    lp0, bn_p, lp1 = layer.linear_p[0], layer.linear_p[1], layer.linear_p[3]
    bn_a, la, bn_b, lb = layer.linear_w[0], layer.linear_w[2], layer.linear_w[3], layer.linear_w[5]
    n, K = idx.shape
    f = {"n": n, "c": layer.out_planes, "K": K, "p": p, "xq": xq, "xk": xk, "xv": xv, "idx": idx,
         "p_w0": lp0.weight, "p_b0": lp0.bias, "p_w1": lp1.weight, "p_b1": lp1.bias, "a_w": la.weight, "a_b": la.bias,
         "b_w": lb.weight, "b_b": lb.bias, "bn_mode": modes, "update_running": int(update)}
    for tag, bn in (("p", bn_p), ("a", bn_a), ("b", bn_b)):
        f.update({tag + "_gamma": bn.weight, tag + "_beta": bn.bias, tag + "_rmean": bn.running_mean.clone(),
                  tag + "_rvar": bn.running_var.clone(), tag + "_eps": bn.eps, tag + "_momentum": bn.momentum})
    return {k: v.detach() if torch.is_tensor(v) else v for k, v in f.items()}


def _module_forward(layer, p, xq, xk, xv, idx):
    """blocks.py:31-44 in the module's dtype with index gathers in place of queryandgroup (float32 p - p_i, as queryandgroup
    computes it on float32 points) -> out, and the BatchNorm inputs t, w0, w1 as (n K, cn)"""
    n, K = idx.shape
    nbr = idx.long()
    p_r = (p[nbr] - p.unsqueeze(1)).to(xq.dtype)
    seen = {}
    for i, m in enumerate(layer.linear_p):
        if i == 1:
            seen["p"] = p_r.reshape(n * K, -1)
        p_r = m(p_r.transpose(1, 2).contiguous()).transpose(1, 2).contiguous() if i == 1 else m(p_r)
    w = xk[nbr] - xq.unsqueeze(1) + p_r
    for i, m in enumerate(layer.linear_w):
        if i % 3 == 0:
            seen["ab"[i // 3]] = w.reshape(n * K, -1)
        w = m(w.transpose(1, 2).contiguous()).transpose(1, 2).contiguous() if i % 3 == 0 else m(w)
    w = torch.softmax(w, dim=1)
    c = xv.shape[1]
    return ((xv[nbr] + p_r).view(n, K, 8, c // 8) * w.unsqueeze(2)).sum(1).view(n, c), seen


def _close(got, want, tol=1e-12):
    return float((got - want).abs().max()) <= tol * max(1.0, float(want.abs().max()))


@pytest.mark.parametrize("c,K,n_crops,per_crop", [(32, 16, 1, 400), (64, 7, 3, 150), (256, 24, 16, 12)])
@pytest.mark.parametrize("train", [True, False])
def test_restatement_matches_module_in_float64(c, K, n_crops, per_crop, train):
    torch.manual_seed(c + K)
    layer = Layer(c, K).double().train(train)
    g = torch.Generator().manual_seed(7)
    for i, bn in enumerate((layer.linear_p[1], layer.linear_w[0], layer.linear_w[3])):
        with torch.no_grad():
            bn.weight.copy_(torch.randn(bn.weight.shape, generator=g))
            bn.bias.copy_(torch.randn(bn.bias.shape, generator=g) * 0.1)
            bn.running_mean.copy_(torch.randn(bn.running_mean.shape, generator=g) * 0.1)
            bn.running_var.copy_(torch.rand(bn.running_var.shape, generator=g) + 0.5)
        bn.eps, bn.momentum = (2.0 ** -10, 2.0 ** -6, 1e-5)[i], (0.375, 1.0, 0.125)[i]   # float32-exact descriptor fields
    p, o = _crops(n_crops, per_crop)
    idx = _knn(p, o, K)
    x = torch.randn(p.shape[0], c, generator=g, dtype=F64)
    with torch.no_grad():
        xq, xk, xv = layer.linear_q(x), layer.linear_k(x), layer.linear_v(x)
        f = _fields(layer, p, xq, xk, xv, idx, [1 if train else 2] * 3, train)
        want, seen = _module_forward(layer, p, xq, xk, xv, idx)
    sums = pt_layer.batch_sums(passes=(0, 1, 2), **f)
    for tag, y in seen.items():
        assert _close(sums[tag][0], torch.cat([y.sum(0), (y * y).sum(0)])), tag
    if train:
        f.update({"stats_" + t: s for t, (s, _) in sums.items()})
    got, bound = pt_layer.output(**f)
    assert got.dtype == F64 and got.shape == want.shape and _close(got, want)
    assert bool((bound > 0).all())
    sel = [0, p.shape[0] // 2, p.shape[0] - 1]
    assert torch.equal(pt_layer.output(select=sel, **f)[0], got[sel])
    upd = pt_layer.running_update(**f)
    assert sorted(upd) == (["a", "b", "p"] if train else [])
    for tag, bn in zip("pab", (layer.linear_p[1], layer.linear_w[0], layer.linear_w[3])):
        if train:
            assert _close(upd[tag][0], bn.running_mean) and _close(upd[tag][1], bn.running_var), tag


@pytest.mark.parametrize("c", [32, 64])
@pytest.mark.parametrize("train", [True, False])
def test_restatement_matches_oracle_layer(c, train):
    fix = np.load(f"{GOLD}/ref_torch_blocks.npz")
    tag = f"ptl{c}"
    K = int(fix[tag + "_K"])
    state = _state(fix, tag)
    p, o, x = (torch.from_numpy(fix[k]) for k in ("p", "o", tag + "_x"))
    want = O.point_transformer_layer(p, x, o, state, K, 8, train, dtype=F64)
    layer = Layer(c, K)
    layer.load_state_dict(state)
    layer.double()
    with torch.no_grad():
        x64 = x.double()
        xq, xk, xv = layer.linear_q(x64), layer.linear_k(x64), layer.linear_v(x64)
    f = _fields(layer, p, xq, xk, xv, _knn(p, o, K), [1 if train else 2] * 3, False)
    got, _ = pt_layer.output(**f)
    # the oracle subtracts the float64 coordinates, the restatement the float32 ones (as the kernel and queryandgroup do)
    assert _close(got, want, 1e-5)


def _f32(f):
    return {k: v.float() if torch.is_tensor(v) and v.is_floating_point() else v for k, v in f.items()}


def _ratio(got, want, bound):
    return float(((got.double() - want).abs() / bound).max())


@pytest.mark.parametrize("kind", pt_layer.CASES)
@pytest.mark.parametrize("c,K,n_crops,per_crop", [(32, 36, 1, 1500), (64, 24, 16, 40), (512, 24, 16, 12)])
def test_bound_holds_for_float32_evaluation(kind, c, K, n_crops, per_crop):
    """the restatement evaluated in float32, conditioned on the float64 evaluation's sums, within the bound of every sum and
    every output element; at c = 512 every neighbourhood is padded (12 points per crop, K = 24)"""
    p, o = _crops(n_crops, per_crop, seed=c)
    f = pt_layer.make_case(c, K, p, _knn(p, o, K), kind, seed=c + K)
    s64 = pt_layer.batch_sums(**f)
    cond = {"stats_" + t: s for t, (s, _) in s64.items()}
    s32 = pt_layer.batch_sums(dtype=torch.float32, **_f32(f), **cond)
    worst = {}
    for tag, (s, b) in s64.items():
        worst["sums_" + tag] = _ratio(s32[tag][0], s, b)
    out, bound = pt_layer.output(**f, **cond)
    out32, _ = pt_layer.output(dtype=torch.float32, **_f32(f), **cond)
    assert out32.dtype == torch.float32
    worst["out"] = _ratio(out32, out, bound)
    for k, v in worst.items():
        WORST[k] = max(WORST.get(k, 0.0), v)
    print(kind, c, K, {k: f"{v:.3g}" for k, v in worst.items()}, "worst so far", {k: f"{v:.3g}" for k, v in WORST.items()})
    assert all(v <= 0.999 for v in worst.values()), worst


def test_conditioning_moves_the_output():
    """the sums handed to a mode-1 BatchNorm are what it normalises with: 1 % more Sigma^2 moves the output past its bound"""
    p, o = _crops(1, 600)
    f = pt_layer.make_case(64, 16, p, _knn(p, o, 16), "plain", seed=3)
    cond = {"stats_" + t: s for t, (s, _) in pt_layer.batch_sums(**f).items()}
    out, bound = pt_layer.output(**f, **cond)
    for tag, cn in (("p", 3), ("a", 64), ("b", 8)):
        moved = dict(cond)
        moved["stats_" + tag] = cond["stats_" + tag].clone()
        moved["stats_" + tag][cn:] *= 1.01
        assert _ratio(pt_layer.output(**f, **moved)[0], out, bound) > 10.0, tag
    assert torch.equal(pt_layer.output(**f)[0], out)                      # missing sums are the module's own
