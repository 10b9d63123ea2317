"""GPU: tgn_sa_group_mlp_max launched directly, one launch at a time, against its float64 restatement (oracle/sa_group.py).

Accuracy is element-wise against float64, |got - truth| <= sum_l kappa_l * mag, where mag is the oracle's magnitude pass (the
network on |x|, |W|, |b|, max over the neighbourhood) and kappa_l bounds layer l's relative error per product-and-sum:
* engine 1 (exact fp32 FMA): (C_max + 2) 2^-24 per layer;
* engines 2 and 5 (3xTF32): 2^-18 + (C_max + 2) 2^-23 per layer -- the dropped lo*lo term, the tensor core's tf32 truncation of
  the lo parts, and the fp32 accumulation;
* engine 3: the same for layer 0 (3xTF32) and 2^-14 + (C_max + 2) 2^-23 for each bf16x2-split layer.
Worst observed err / bound over the cases below, on an H100 80GB HBM3 at 700 W: engine 1 1.9e-2, engines 2 and 5 0.11, engine 3 6.9e-2.

The rest is bitwise: each cloud of a B-cloud launch equals a launch of that cloud alone (tiles_per_cloud of 1, 2 and many, more
tiles than persistent CTA slots, the bench shape), engine 0 equals the engine the header names, engine 5 equals engine 2, two
launches of an engine are equal, channels outside [out_c_offset, +C_last) keep a NaN sentinel's bits, and every refusal raises
TgnError and leaves ``out`` untouched."""
import ctypes

import pytest
import torch

from oracle import sa_group
from toothgroupnetwork_b200 import _lib as L
from toothgroupnetwork_b200 import clouds
from toothgroupnetwork_b200 import pointnet2_utils as pn2

pytestmark = pytest.mark.gpu

AUTO, FP32, TC, TCW, TC_HALF = 0, 1, 2, 3, 5
SENTINEL = 0x7FC0DEAD                 # a quiet NaN with a payload: its exact bits show a channel nobody wrote


def kappas(engine, channels):
    cmax, n = max(channels), len(channels) - 1
    if engine == FP32:
        return [(cmax + 2) * 2.0 ** -24] * n
    tf = 2.0 ** -18 + (cmax + 2) * 2.0 ** -23
    if engine in (TC, TC_HALF):
        return [tf] * n
    return [tf] + [2.0 ** -14 + (cmax + 2) * 2.0 ** -23] * (n - 1)


# ------------------------------------------------------------------------------------------------------------------ inputs
class Inputs:
    """CPU tensors of one launch and their device copies; gidx from the library's ball query, with a few j = N rows"""

    def __init__(self, B, N, S, K, D, seed, kind="arch", radius=None, empty_every=97):
        gen = torch.Generator().manual_seed(seed)
        if kind == "arch":
            f = torch.cat([clouds.arch_features(N, 7 * seed + b) for b in range(B)], 0).permute(0, 2, 1)
            xyz, normals = f[..., :3].contiguous(), f[..., 3:]
            extra = torch.randn(B, N, max(D - 3, 0), generator=gen) * torch.logspace(-3, 3, max(D - 3, 0))
            feats = torch.cat([normals, extra], -1)[..., :D].contiguous() if D >= 3 else None
            if 0 < D < 3:
                feats = (torch.randn(B, N, D, generator=gen) * torch.logspace(3, -3, D)).contiguous()
            r = radius if radius is not None else 0.016 * K ** 0.5 + 0.01
        else:                          # far from the origin: the centre subtraction cancels
            xyz = torch.rand(B, N, 3, generator=gen) * 0.5 + 50.0
            feats = (torch.randn(B, N, D, generator=gen) * torch.logspace(-3, 3, D)).contiguous() if D else None
            r = radius if radius is not None else 0.1
        cen = torch.stack([torch.randperm(N, generator=gen)[:S] for _ in range(B)])
        new_xyz = torch.gather(xyz, 1, cen.unsqueeze(-1).expand(-1, -1, 3)).contiguous()
        gidx = pn2._ball_query(r, K, xyz.cuda(), new_xyz.cuda(), False, None, 1).cpu()
        if empty_every:
            gidx.view(-1)[5::empty_every] = N
        self.B, self.N, self.S, self.K, self.D = B, N, S, K, D
        self.xyz, self.feats, self.new_xyz, self.gidx = xyz, feats, new_xyz, gidx
        self.dev = [None if t is None else t.cuda() for t in (xyz, feats, new_xyz, gidx)]

    def cloud(self, b):
        """the same inputs restricted to cloud b (device copies)"""
        one = Inputs.__new__(Inputs)
        one.B, one.N, one.S, one.K, one.D = 1, self.N, self.S, self.K, self.D
        one.dev = [None if t is None else t[b:b + 1].contiguous() for t in self.dev]
        return one


def make_net(channels, seed, zero_bias=True):
    """weights with every third row exactly representable in tf32 (lo = 0); a last-layer bias negative enough that some
    outputs are exactly 0 (every fourth channel) and others clipped on part of the neighbourhood"""
    gen = torch.Generator().manual_seed(seed)
    ws, bs = [], []
    for ci, co in zip(channels[:-1], channels[1:]):
        w = torch.randn(co, ci, generator=gen) / ci ** 0.5
        w[::3] = (w[::3].view(torch.int32) & ~0x1FFF).view(torch.float32)
        ws.append(w.contiguous())
        bs.append(torch.randn(co, generator=gen) * 0.1)
    if zero_bias:
        bs[-1][::4] = -1e4
        bs[-1][1::4] -= 0.5
    return ws, bs


def launch(inp, ws, bs, engine, xyz_first=1, out=None, c_off=0, channels=None, n_layers=None, feats="inputs"):
    xyz, f, new_xyz, gidx = inp.dev
    if feats != "inputs":
        f = feats
    channels = channels or [3 + inp.D] + [w.shape[0] for w in ws]
    if out is None:
        out = torch.full((inp.B, channels[-1], inp.S), float("nan"), device="cuda")
    wd = [w.cuda() for w in ws]
    bd = [b.cuda() for b in bs]
    chv = (ctypes.c_int * len(channels))(*channels)
    wp = (ctypes.c_void_p * max(len(wd), 1))(*[w.data_ptr() for w in wd])
    bp = (ctypes.c_void_p * max(len(bd), 1))(*[b.data_ptr() for b in bd])
    L.call("tgn_sa_group_mlp_max", inp.B, inp.N, inp.S, inp.K, inp.D, L.ptr(xyz), L.ptr(f), L.ptr(new_xyz), L.ptr(gidx),
           int(xyz_first), len(ws) if n_layers is None else n_layers, ctypes.cast(chv, ctypes.c_void_p),
           ctypes.cast(wp, ctypes.c_void_p), ctypes.cast(bp, ctypes.c_void_p), L.ptr(out), out.shape[1], int(c_off), int(engine),
           L.stream_ptr())
    torch.cuda.synchronize()
    return out


def truth_of(inp, ws, bs, xyz_first, select=None):
    ch = [3 + inp.D] + [w.shape[0] for w in ws]
    return sa_group.group_mlp_max(inp.B, inp.N, inp.S, inp.K, inp.D, inp.xyz, inp.feats, inp.new_xyz, inp.gidx, xyz_first, ch,
                                  ws, bs, select=select)


def check_bound(got, truth, mag, engine, channels, tag):
    bound = sum(kappas(engine, channels)) * mag
    err = (got.detach().double().cpu() - truth).abs()
    ratio = float((err / bound.clamp(min=1e-300)).max())
    print(f"SA_GROUP_ERR engine={engine} {tag} err/bound={ratio:.3e}")
    bad = ~(err <= bound)
    assert not bool(bad.any()), f"engine {engine} {tag}: {int(bad.sum())} elements outside the bound, worst err/bound {ratio:.3e}"


def run_engines(inp, ws, bs, xyz_first, engines, tag):
    truth, mag = truth_of(inp, ws, bs, xyz_first)
    ch = [3 + inp.D] + [w.shape[0] for w in ws]
    outs = {}
    for e in engines:
        got = launch(inp, ws, bs, e, xyz_first)
        check_bound(got, truth, mag, e, ch, tag)
        assert torch.equal(got, launch(inp, ws, bs, e, xyz_first)), f"engine {e}: two launches differ"
        outs[e] = got
    return outs, truth


# ------------------------------------------------------------------------------------------------- a. accuracy: engines 2 / 5
def _tc_cases():
    cases = []      # (B, N, S, K, D, xyz_first, widths, kind)
    for i, K in enumerate([1, 3, 7, 8, 9, 20, 32, 40, 64, 100, 127, 128]):
        cases.append((3 if i % 2 == 0 else 1, 2000, 2 * (128 // K) + 1, K, 6, i % 2, [32, 64], "arch" if i % 3 else "offset"))
    for i, (D, xf) in enumerate([(d, x) for d in (0, 1, 6, 13) for x in (1, 0)]):
        cases.append((1 + 2 * (i % 2), 2000, 77, 16, D, xf, [16, 32], "offset" if i % 3 == 0 else "arch"))
    for i, w in enumerate([[16, 24], [32, 32, 40], [48, 64], [64, 64], [17, 9], [33, 50]]):       # NP = 16 / 32 / 48 / 64, odd widths
        cases.append((3 if i % 2 else 1, 2000, 61, 32, 6, 1, w, "arch"))
    for i, w in enumerate([[1], [64], [128]]):                                                   # one layer
        cases.append((3, 2000, 50, 20, 13 if i == 1 else 6, i % 2, w, "arch"))
    for i, w in enumerate([[32, 65], [64, 128], [17, 33, 128]]):                                 # the hc = 1 slice of the last layer
        cases.append((1 + 2 * (i % 2), 2000, 45, 32, 6, 1 - i % 2, w, "offset" if i == 1 else "arch"))
    cases.append((3, 2000, 40, 32, 13, 1, [48, 48, 48, 48], "arch"))    # four layers ([64] * 4 does not fit: see the refusals)
    for K, S in [(32, 1), (32, 3), (32, 4), (32, 5), (32, 1001), (7, 1), (7, 17), (7, 18), (7, 19)]:   # S around gpt = 128 / K
        cases.append((3 if S % 2 else 1, 2000, S, K, 6, 1, [32, 32, 64], "arch"))
    return cases


@pytest.mark.parametrize("B,N,S,K,D,xyz_first,widths,kind", _tc_cases())
def test_tensor_core_engine_against_float64(B, N, S, K, D, xyz_first, widths, kind):
    inp = Inputs(B, N, S, K, D, seed=K * 31 + S + D, kind=kind)
    ws, bs = make_net([3 + D] + widths, seed=len(widths) * 100 + K)
    outs, truth = run_engines(inp, ws, bs, xyz_first, (TC, TC_HALF), f"B={B} S={S} K={K} D={D} xf={xyz_first} w={widths} {kind}")
    assert torch.equal(outs[TC_HALF], outs[TC])
    if widths[-1] > 1:
        assert bool((truth == 0).any()) and bool((truth > 0).any())


# --------------------------------------------------------------------------------------------------- a. accuracy: engine 3
TCW_CASES = [
    # (B, N, S, K, D, xyz_first, widths, kind)
    (3, 2000, 40, 16, 3, 1, [80, 128], "arch"),                 # NP = 80, full tiles; unit-scale features (normals)
    (1, 2000, 43, 16, 6, 0, [72, 96], "offset"),                # partial last tile of 3 neighbourhoods: 48 rows <= 64
    (3, 2000, 46, 16, 13, 1, [128, 64], "arch"),                # partial last tile of 6: 64 < 96 < 128 rows
    (1, 2000, 29, 32, 3, 1, [96, 96, 64], "arch"),              # NP = 96, last tile of one neighbourhood (32 rows)
    (3, 2000, 31, 32, 0, 0, [112, 33], "arch"),                 # NP = 112, last tile of 96 rows
    (1, 2000, 19, 64, 6, 1, [112, 128], "offset"),              # K = 64, last tile of 64 rows
    (3, 2000, 20, 64, 1, 0, [128, 64, 100], "arch"),
    (1, 2000, 9, 128, 3, 0, [96, 80, 64, 100], "arch"),         # four layers, K = 128
    (3, 2000, 12, 128, 13, 0, [65, 81, 128], "arch"),
    (3, 2000, 50, 32, 6, 1, [16, 32], "arch"),                  # narrow layers: four tile groups
]


@pytest.mark.parametrize("B,N,S,K,D,xyz_first,widths,kind", TCW_CASES)
def test_wide_engine_against_float64(B, N, S, K, D, xyz_first, widths, kind):
    inp = Inputs(B, N, S, K, D, seed=K * 17 + S + D, kind=kind)
    ws, bs = make_net([3 + D] + widths, seed=len(widths) * 10 + K + 3)
    run_engines(inp, ws, bs, xyz_first, (TCW,), f"B={B} S={S} K={K} D={D} xf={xyz_first} w={widths} {kind}")


# --------------------------------------------------------------------------------------------------- a. accuracy: engine 1
FP32_CASES = [
    (3, 2000, 300, 1, 6, 1, [32, 64], "arch"),
    (1, 2000, 77, 5, 13, 0, [17, 40], "offset"),
    (3, 2000, 20, 128, 6, 1, [64, 128], "arch"),
    (1, 2000, 20, 129, 6, 0, [32, 48], "arch"),                 # K > 128: two chunks merged with atomicMax
    (3, 2000, 15, 200, 0, 1, [64, 64, 64], "arch"),
    (1, 2000, 15, 256, 6, 1, [128], "offset"),
    (3, 2000, 10, 300, 13, 0, [40, 128], "arch"),
    (1, 2000, 40, 32, 125, 1, [128, 64], "arch"),               # input width 128
    (3, 2000, 40, 32, 125, 0, [128, 128, 128, 128], "arch"),    # weights do not fit next to the activations: staged per layer
]


@pytest.mark.parametrize("B,N,S,K,D,xyz_first,widths,kind", FP32_CASES)
def test_exact_fma_engine_against_float64(B, N, S, K, D, xyz_first, widths, kind):
    inp = Inputs(B, N, S, K, D, seed=K * 13 + S + D, kind=kind)
    ws, bs = make_net([3 + D] + widths, seed=len(widths) * 7 + K + 5)
    run_engines(inp, ws, bs, xyz_first, (FP32,), f"B={B} S={S} K={K} D={D} xf={xyz_first} w={widths} {kind}")


# ----------------------------------------------------------------------------------- b. batch and grid invariance, bitwise
INVARIANCE = [
    # (engine, B, N, S, K, widths)   tiles per cloud: 1, 2, many; B = 600 with one tile per cloud: more tiles than CTA slots
    (TC, 3, 600, 4, 32, [32, 32, 64]), (TC, 3, 600, 7, 32, [32, 32, 64]), (TC, 3, 600, 201, 32, [32, 32, 64]),
    (TC, 600, 400, 12, 10, [32, 32, 64]), (TC_HALF, 3, 600, 201, 20, [32, 64]), (TC_HALF, 600, 400, 4, 32, [32, 64]),
    (TCW, 3, 600, 8, 16, [128, 128]), (TCW, 3, 600, 11, 16, [128, 128]), (TCW, 3, 600, 203, 16, [96, 64]),
    (TCW, 600, 400, 2, 64, [128, 128]), (TCW, 600, 400, 8, 16, [32, 48]),
    (FP32, 3, 600, 8, 16, [32, 64]), (FP32, 3, 600, 201, 16, [64, 128]), (FP32, 600, 400, 8, 16, [32, 64]),
    (FP32, 3, 600, 40, 200, [32, 64]), (FP32, 3, 600, 30, 32, [128, 128, 128, 128]),
]


@pytest.mark.parametrize("engine,B,N,S,K,widths", INVARIANCE)
def test_each_cloud_equals_its_own_launch(engine, B, N, S, K, widths):
    D = 125 if widths == [128, 128, 128, 128] else 6
    inp = Inputs(B, N, S, K, D, seed=B + S + K, kind="offset" if B > 100 else "arch", radius=0.1 if B > 100 else None)
    ws, bs = make_net([3 + D] + widths, seed=S + K)
    full = launch(inp, ws, bs, engine)
    assert not bool(full.isnan().any())
    picks = range(B) if B <= 3 else sorted({0, B - 1, *torch.randperm(B, generator=torch.Generator().manual_seed(B))[:22].tolist()})
    for b in picks:
        assert torch.equal(full[b:b + 1], launch(inp.cloud(b), ws, bs, engine)), f"cloud {b}"


def test_bench_shape():
    """1056 clouds of 24 000 points, S = 1024, K = 32, D = 6, [32, 32, 64] on engine 2: sampled clouds equal their own launches,
    and 2 000 sampled neighbourhoods are within the float64 bound"""
    B, N, S, K, D, nd = 1056, 24000, 1024, 32, 6, 8
    base = torch.stack([clouds.arch_features(N, clouds.cloud_seed(0, j))[0] for j in range(nd)]).permute(0, 2, 1).cuda()
    g = torch.Generator(device="cuda").manual_seed(2024)
    pts = (base[torch.arange(B, device="cuda") % nd] + 1e-3 * torch.randn(B, N, 6, device="cuda", generator=g)).contiguous()
    inp = Inputs.__new__(Inputs)
    inp.B, inp.N, inp.S, inp.K, inp.D = B, N, S, K, D
    xyz, feats = pts[..., :3].contiguous(), pts            # the bench's features: [xyz; normal]
    new_xyz = xyz[:, :S].contiguous()
    gidx = pn2._ball_query(0.1, K, xyz, new_xyz, False, None, 1)
    inp.dev = [xyz, feats, new_xyz, gidx]
    ws, bs = make_net([3 + D, 32, 32, 64], seed=9)
    full = launch(inp, ws, bs, TC)
    assert not bool(full.isnan().any())
    sel_gen = torch.Generator().manual_seed(7)
    clouds_sel = sorted({0, B - 1, *torch.randperm(B, generator=sel_gen)[:6].tolist()})
    for b in clouds_sel:
        assert torch.equal(full[b:b + 1], launch(inp.cloud(b), ws, bs, TC)), f"cloud {b}"
    # float64 on 40 clouds x 50 neighbourhoods
    cl = torch.randperm(B, generator=sel_gen)[:40]
    sub = Inputs.__new__(Inputs)
    sub.B, sub.N, sub.S, sub.K, sub.D = len(cl), N, S, K, D
    sub.xyz, sub.feats, sub.new_xyz, sub.gidx = (t[cl.cuda()].cpu() for t in (xyz, feats, new_xyz, gidx))
    select = [(i, int(s)) for i in range(len(cl)) for s in torch.randperm(S, generator=sel_gen)[:50]]
    truth, mag = truth_of(sub, ws, bs, 1, select=select)
    got = torch.stack([full[int(cl[i]), :, s] for i, s in select])
    check_bound(got, truth, mag, TC, [3 + D, 32, 32, 64], "bench shape")


# ------------------------------------------------------------------------------------------- c. dispatcher and equivalences
@pytest.mark.parametrize("K,widths,named", [
    (32, [32, 32, 64], TC),               # fits the 3xTF32 engine
    (32, [128, 128], TCW),                # hidden width 128: the wide engine
    (32, [64, 64, 64, 64], TCW),          # every width <= 64, but four 64-wide layers do not fit engine 2's shared memory
    (24, [128, 128], FP32),               # K = 24: neither tensor-core engine
    (200, [32, 64], FP32),                # K > 128
])
def test_auto_equals_the_named_engine(K, widths, named):
    inp = Inputs(3, 2000, 60, K, 6, seed=K + len(widths))
    ws, bs = make_net([9] + widths, seed=K)
    auto = launch(inp, ws, bs, AUTO)
    assert torch.equal(auto, launch(inp, ws, bs, named))
    others = [e for e in (FP32, TC, TCW) if e != named]
    assert not any(torch.equal(auto, launch(inp, ws, bs, e)) for e in others if _supported(inp, ws, bs, e))


def _supported(inp, ws, bs, engine):
    try:
        launch(inp, ws, bs, engine)
        return True
    except L.TgnError:
        return False


# ----------------------------------------------------------------------------------------------------- d. output placement
def _sentinel(shape):
    return torch.full(shape, SENTINEL, dtype=torch.int32, device="cuda").view(torch.float32)


@pytest.mark.parametrize("engine,K,widths", [(TC, 32, [32, 32, 64]), (TC_HALF, 7, [32, 65]), (TCW, 16, [128, 128]),
                                             (FP32, 32, [64, 128]), (FP32, 200, [32, 48])])
def test_branch_writes_only_its_channels(engine, K, widths):
    inp = Inputs(3, 2000, 37, K, 6, seed=K + 1)
    ws, bs = make_net([9] + widths, seed=K + 2)
    want = launch(inp, ws, bs, engine)
    c, off, total = widths[-1], 5, widths[-1] + 12
    out = _sentinel((3, total, 37))
    out[:, off:off + c] = 1e30              # garbage in the branch's own slice: the K > 128 path must clear it first
    launch(inp, ws, bs, engine, out=out, c_off=off)
    assert torch.equal(out[:, off:off + c], want)
    bits = out.view(torch.int32)
    assert bool((bits[:, :off] == SENTINEL).all()) and bool((bits[:, off + c:] == SENTINEL).all())


@pytest.mark.parametrize("engines", [(TC, TC), (TC, FP32), (FP32, TCW)])
def test_two_branches_back_to_back(engines):
    """MSG: [feats | xyz_rel] branches of K = 16 and K = 200 / 32 written into one (B, C0 + C1 + 3, S) buffer"""
    S, D = 50, 6
    spec = [(16, 0.05, [16, 32]), (200 if engines[1] == FP32 else 32, 0.1, [32, 48] if engines[1] != TCW else [128, 40])]
    base = Inputs(2, 2000, S, 16, D, seed=3)
    out = _sentinel((2, 32 + spec[1][2][-1] + 3, S))
    wants, off = [], 0
    for e, (K, r, widths) in zip(engines, spec):
        inp = Inputs.__new__(Inputs)
        inp.B, inp.N, inp.S, inp.K, inp.D = 2, 2000, S, K, D
        inp.dev = list(base.dev)
        inp.dev[3] = pn2._ball_query(r, K, base.dev[0], base.dev[2], False, None, 1)
        ws, bs = make_net([3 + D] + widths, seed=K)
        wants.append((off, launch(inp, ws, bs, e, xyz_first=0)))
        launch(inp, ws, bs, e, xyz_first=0, out=out, c_off=off)
        off += widths[-1]
    for o, w in wants:
        assert torch.equal(out[:, o:o + w.shape[1]], w)
    assert bool((out.view(torch.int32)[:, off:] == SENTINEL).all())


# ---------------------------------------------------------------------------------------------------------- e. refusals
REFUSALS = [
    # (engine, K, D, channels, n_layers, feats_null, message)
    (-1, 32, 6, [9, 32], None, False, "unknown engine -1"),
    (4, 32, 6, [9, 32], None, False, "unknown engine 4"),
    (6, 32, 6, [9, 32], None, False, "unknown engine 6"),
    (TC, 32, 6, [9, 65, 32], None, False, "not supported by the tensor-core engine"),
    (TC, 32, 14, [17, 32], None, False, "not supported by the tensor-core engine"),
    (TC, 32, 6, [9, 64, 64, 64, 64], None, False, "not supported by the tensor-core engine"),    # > 220 KB of shared memory
    (TCW, 64, 6, [9, 128, 128, 100], None, False, "not supported by the wide tensor-core engine"),  # > 224 KB
    (TCW, 24, 6, [9, 128, 128], None, False, "not supported by the wide tensor-core engine"),
    (TCW, 32, 6, [9, 128], None, False, "not supported by the wide tensor-core engine"),
    (AUTO, 32, 6, [8, 32], None, False, "channels[0]=8 but 3+D=9"),
    (AUTO, 32, 6, [9, 0, 32], None, False, "layer width 0 outside"),
    (FP32, 32, 6, [9, 32, 129], None, False, "layer width 129 outside"),
    (AUTO, 32, 6, [9], 0, False, "1..4 layers supported, got 0"),
    (AUTO, 32, 6, [9, 16, 16, 16, 16, 16], 5, False, "1..4 layers supported, got 5"),
    (FP32, 32, 6, [9, 32], None, True, "feats missing for D=6"),
]


@pytest.mark.parametrize("engine,K,D,channels,n_layers,feats_null,message", REFUSALS)
def test_refusals_leave_out_untouched(engine, K, D, channels, n_layers, feats_null, message):
    inp = Inputs(1, 500, 20, K, D, seed=1)
    ws, bs = make_net(channels, seed=1, zero_bias=False)          # full-size weights, though no refused call reads them
    out = _sentinel((1, 40, 20))
    with pytest.raises(L.TgnError, match=message.replace("[", r"\[").replace("]", r"\]").replace("+", r"\+")):
        launch(inp, ws, bs, engine, out=out, channels=channels, n_layers=n_layers, feats=None if feats_null else "inputs")
    assert bool((out.view(torch.int32) == SENTINEL).all())
