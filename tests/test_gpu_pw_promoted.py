"""GPU: the promoted-accumulation form of the layer kernel (tgn_pw_layer_forward with accum = 1, csrc/pw_layer.cuh) one launch at a
time against a float64 product of the same operands (oracle/pw_chain.py builds them as the kernel does).

Element-wise bound.  Write S[c, r] = sum_k |w[c, k]| m[r, k], with m = |x| for an operand without input BatchNorm and
m = |x - mean| |scale| + |beta| with one (the magnitude before the activation, which only shrinks it).  Then

    |y - exact| <= kappa(P, K) S + 2^-23 |exact|,       kappa(P, K) = 2^-23 (6 P + ceil(K / 16 P) / 2 + 2)

* operands: each is split into three bf16 parts exactly; the dropped cross terms are below 2^-25 |w x| per product, and the
  input BatchNorm's fp32 arithmetic rounds three times, 2^-24 m each: 2 units of 2^-23 S cover both;
* one chunk is P K-steps of 6 MMAs into a fresh accumulator.  Each MMA truncates: up to one ulp of its running sum, which is at
  most 2^-23 of that chunk's share of S, so a chunk is off by at most 6 P 2^-23 of its share and all chunks by 6 P 2^-23 S;
* the chunks are added into the total with ceil(K / 16 P) round-to-nearest adds, each within half an ulp of the total (<= S);
* the epilogue adds bias and cloud_bias in fp32: 2^-23 |exact|.

Without promotion (accum = 0) the truncations of all 6 ceil(K / 16) MMAs land on one accumulator, always towards zero.  On
channels whose operands share a sign and have |mean| / std = 1000, the running sum grows steadily and the error approaches
6 ceil(K / 16) / 2 ulps, above kappa(P, K) S at K = 512 and 1 024 (measured on an H100: see test_promotion_separates_the_forms);
the promoted launch stays below it.

Also: K and rows off every tile multiple, modes 0 / 1 / 2, two segments and cloud_bias, group extrema with negative scales on
both extrema paths, LeakyReLU, input BatchNorm from batch sums and from running statistics, the widest cin the promoted form
takes, per-row independence (a slice launched alone is bitwise equal), and the refusals."""
import ctypes
import math

import pytest
import torch

from oracle import pw_chain
from toothgroupnetwork_b200 import _lib as L

pytestmark = pytest.mark.gpu
P = 1                                   # K-steps per promoted chunk (csrc/pw_mlp_promoted.cu, kPromoteSteps)
HALF_TILE = 64                          # rows per epilogue thread at 128-row tiles: groups that do not divide it need atomics
MAX_CIN_AFFINE = (227 * 1024 - 16 - 2 * (24 + 3 * 8) * 1024) // 16     # shared memory: two 48 KB stages + 16 B per input channel


def kappa(K):
    return 2.0 ** -23 * (6 * P + math.ceil(K / (16 * P)) / 2 + 2)


_INT = ("rows", "rows_per_batch", "cin", "cout", "mode", "N", "S", "K", "D", "xyz_first", "in_affine", "in_update_running", "edge_C",
        "in_act", "group", "precision", "accum")
_FLOAT = ("in_eps", "in_momentum", "in_act_slope")
_ARRAY = ("seg_channels", "seg_batch_stride", "seg_row_stride", "seg_chan_stride", "edge_stride")
_PTR = ("xyz", "feats", "new_xyz", "gidx", "in_stats", "in_gamma", "in_beta", "in_running_mean", "in_running_var", "bias",
        "cloud_bias", "edge_x")


def _packed(w):
    cout, cin = w.shape
    buf = torch.empty(L.load().tgn_pw_packed_bytes(cout, cin), dtype=torch.uint8, device="cuda")
    L.call("tgn_pw_pack_weights", cout, cin, L.ptr(w), L.ptr(buf), L.stream_ptr())
    return buf


def _descriptor(f):
    dev = {k: f[k].cuda() for k in _PTR if f.get(k) is not None}
    dev.update({f"seg_ptr{i}": t.cuda() for i, t in enumerate(f.get("seg_ptr", ()))})
    dev["w_packed"] = _packed(f["weight"].cuda())
    d = L.PwLayer()
    for k in _INT:
        if k in f:
            setattr(d, k, int(f[k]))
    for k in _FLOAT:
        if k in f:
            setattr(d, k, float(f[k]))
    for k in _ARRAY:
        for i, v in enumerate(f.get(k, ())):
            getattr(d, k)[i] = int(v)
    for k in _PTR:
        setattr(d, k, L.ptr(dev.get(k)))
    for i in range(len(f.get("seg_ptr", ()))):
        d.seg_ptr[i] = L.ptr(dev[f"seg_ptr{i}"])
    d.w_packed = L.ptr(dev["w_packed"])
    return d, dev


def _magnitude(f):
    """S (cout, rows) of the bound: sum_k |w| m over the operand the oracle builds"""
    x, ok = pw_chain._operand(f["rows"], f["cin"], f.get("mode", 0), f.get("rows_per_batch", 0), f.get("seg_ptr", ()),
                              f.get("seg_channels", (0, 0)), f.get("seg_batch_stride", (0, 0)), f.get("seg_row_stride", (0, 0)),
                              f.get("seg_chan_stride", (0, 0)), f.get("xyz"), f.get("feats"), f.get("new_xyz"), f.get("gidx"),
                              f.get("N", 0), f.get("S", 0), f.get("K", 0), f.get("D", 0), f.get("xyz_first", 0), f.get("edge_x"),
                              f.get("edge_stride", (0, 0, 0)), f.get("edge_C", 0))
    m = x.double().abs()
    if f.get("in_affine"):
        mean, scale, beta = pw_chain._bn_scale(f["in_affine"], f["cin"], f.get("in_stats"), float(f["rows"]), f.get("in_gamma"),
                                               f.get("in_beta"), f.get("in_eps", 1e-5), f.get("in_running_mean"), f.get("in_running_var"))
        h = (x.double() - mean).abs() * scale.abs() + beta.abs()
        m = torch.where(ok.unsqueeze(1), h, m)
    return f["weight"].double().abs() @ m.t()


def launch(f, accum):
    """one launch -> (y, ymax, ymin, stats) on the CPU; extrema merged with atomics when the group does not divide the half tile"""
    d, dev = _descriptor(f)
    d.accum = accum
    rows, cout, G = f["rows"], f["cout"], f.get("group", 0)
    y = torch.empty((cout, rows), dtype=torch.float32, device="cuda")
    stats = torch.zeros(2 * cout, dtype=torch.float64, device="cuda")
    d.y, d.stats = L.ptr(y), L.ptr(stats)
    ymax = ymin = None
    if G:
        ymax = torch.full((cout, rows // G), float("-inf"), device="cuda")
        ymin = torch.full((cout, rows // G), float("inf"), device="cuda")
        d.ymax, d.ymin, d.extrema_atomic = L.ptr(ymax), L.ptr(ymin), 1 if (HALF_TILE if accum else 128) % G else 0
    L.call("tgn_pw_layer_forward", ctypes.byref(d), L.stream_ptr())
    torch.cuda.synchronize()
    return y.cpu(), None if ymax is None else ymax.cpu(), None if ymin is None else ymin.cpu(), stats.cpu(), dev


def ratio(y, f):
    """max over the elements of |y - exact| / bound"""
    want = pw_chain.layer_forward(**f)["y"]
    bound = kappa(f["cin"]) * _magnitude(f) + 2.0 ** -23 * want.abs()
    return float(((y.double() - want).abs() / bound.clamp(min=1e-300)).max())


# ------------------------------------------------------------------------------------------------------------ case builders
def _weight(gen, cout, cin):
    return torch.randn(cout, cin, generator=gen) / cin ** 0.5


def _in_bn(gen, cin, rows, mode, slope=None):
    """input BatchNorm fields: gamma with negative and zero entries; batch sums of a (mean, var) per channel, or running statistics"""
    m = torch.randn(cin, generator=gen, dtype=torch.float64) * 0.5
    v = torch.rand(cin, generator=gen, dtype=torch.float64) + 0.2
    gamma = torch.randn(cin, generator=gen)
    gamma[::7] = 0.0
    f = {"in_affine": mode, "in_gamma": gamma, "in_beta": torch.randn(cin, generator=gen) * 0.2,
         "in_running_mean": torch.randn(cin, generator=gen) * 0.3, "in_running_var": torch.rand(cin, generator=gen) + 0.5,
         "in_eps": 1e-5, "in_momentum": 0.1}
    if mode == 1:
        f["in_stats"] = torch.cat([rows * m, rows * (v + m * m)])
    if slope is not None:
        f.update(in_act=1, in_act_slope=slope)
    return f


def _mode0(gen, B, n, cin, cout, segs="cf", cloud_bias=False, **extra):
    """segs: 'cf' one channel-first segment; 'fp' [channel-first (3 channels) | point-major]"""
    rows = B * n
    f = {"rows": rows, "cin": cin, "cout": cout, "mode": 0, "rows_per_batch": n, "weight": _weight(gen, cout, cin),
         "bias": torch.randn(cout, generator=gen) * 0.1}
    if segs == "cf":
        x = torch.randn(B, cin, n, generator=gen)
        f.update(seg_ptr=(x,), seg_channels=(cin, 0), seg_batch_stride=(cin * n, 0), seg_row_stride=(1, 0), seg_chan_stride=(n, 0))
    else:
        d1, d2 = 3, cin - 3
        skip, interp = torch.randn(B, d1, n, generator=gen), torch.randn(B, n, d2, generator=gen)
        f.update(seg_ptr=(skip, interp), seg_channels=(d1, d2), seg_batch_stride=(d1 * n, n * d2), seg_row_stride=(1, d2),
                 seg_chan_stride=(n, 1))
    if cloud_bias:
        f["cloud_bias"] = torch.randn(B, cout, generator=gen)
    f.update(extra)
    return f


def _mode1(gen, B, N, S, K, D, xyz_first, cout):
    xyz = torch.rand(B, N, 3, generator=gen)
    gidx = torch.randint(0, N, (B, S, K), generator=gen, dtype=torch.int32)
    gidx.view(-1)[3::37] = N                                                  # empty-ball entries: zero rows
    return {"rows": B * S * K, "cin": D + 3, "cout": cout, "mode": 1, "rows_per_batch": S * K, "xyz": xyz,
            "feats": torch.randn(B, N, D, generator=gen) if D else None, "new_xyz": xyz[:, :S].contiguous(), "gidx": gidx,
            "N": N, "S": S, "K": K, "D": D, "xyz_first": xyz_first, "weight": _weight(gen, cout, D + 3),
            "bias": torch.randn(cout, generator=gen) * 0.1, "group": K}


def _mode2(gen, in_mode, K=20):
    B, C, N, cout = 2, 17, 300, 70
    base = torch.randn(B, 2 * C + 1, N, generator=gen)
    x = base[:, 1::2]
    idx = torch.randint(0, N, (B, N, K), generator=gen, dtype=torch.int32)
    idx[0, 3, 1], idx[-1, N - 1, K - 1] = N, -1
    rows = B * N * K
    f = {"rows": rows, "cin": 2 * C, "cout": cout, "mode": 2, "rows_per_batch": N * K, "edge_x": base.reshape(-1)[1:],
         "edge_stride": x.stride(), "edge_C": C, "gidx": idx, "N": N, "K": K, "weight": _weight(gen, cout, 2 * C), "group": K}
    f.update(_in_bn(gen, 2 * C, rows, in_mode, slope=0.2))
    return f


def _offset(gen, cin, rows=1000, cout=200):
    """operands with |mean| / std = 1000 on every channel, of one sign per cloud channel: the running sums of half the output
    channels (non-negative weights) grow steadily through K, the others (signed weights) partly cancel"""
    mu = torch.rand(cin, generator=gen) + 0.5
    x = mu[:, None] * (1.0 + 1e-3 * torch.randn(cin, rows, generator=gen))
    w = torch.rand(cout, cin, generator=gen) / cin
    w[1::2] = torch.randn(cout // 2, cin, generator=gen) / cin ** 0.5
    return {"rows": rows, "cin": cin, "cout": cout, "mode": 0, "rows_per_batch": rows, "weight": w, "bias": None,
            "seg_ptr": (x.contiguous(),), "seg_channels": (cin, 0), "seg_batch_stride": (0, 0), "seg_row_stride": (1, 0),
            "seg_chan_stride": (rows, 0)}


@pytest.mark.parametrize("K", [512, 1024])
def test_promotion_separates_the_forms(K):
    """|mean| / std = 1000: the accum = 0 launch exceeds the bound, the promoted one meets it (measured on an H100, max error over
    bound: K = 512 accum 0 / 1 = 1.31 / 0.17, K = 1 024 = 1.10 / 0.13)"""
    f = _offset(torch.Generator().manual_seed(K), K)
    r0, r1 = ratio(launch(f, 0)[0], f), ratio(launch(f, 1)[0], f)
    print(f"K={K}: max |y - exact| / bound, accum 0: {r0:.3f}, accum 1: {r1:.3f}")
    assert r1 <= 1.0 < r0, (r0, r1)


CASES = {
    # mode 0: K not a multiple of 32 or 16 P, cin = 1, rows and cout off the 128 tiles, two segments, cloud_bias, input BatchNorm
    "m0_cin1_rows257_cout129": lambda g: _mode0(g, 1, 257, 1, 129),
    "m0_cin33_rows1000_cout1": lambda g: _mode0(g, 1, 1000, 33, 1),
    "m0_cin17_rows127_cout200_bn_running": lambda g: _mode0(g, 1, 127, 17, 200, **_in_bn(g, 17, 127, 2)),
    "m0_fp_cin67_rows3000_cloud_bias": lambda g: _mode0(g, 2, 1500, 67, 128, segs="fp", cloud_bias=True),
    "m0_cin1216_rows2001_bn_running_leaky_cloud_bias": lambda g: _mode0(g, 3, 667, 1216, 130, cloud_bias=True,
                                                                        **_in_bn(g, 1216, 2001, 2, slope=0.2)),
    "m0_cin530_rows999_bn_batch": lambda g: _mode0(g, 1, 999, 530, 64, **_in_bn(g, 530, 999, 1)),
    "m0_cin_max_rows300_bn_running": lambda g: _mode0(g, 1, 300, MAX_CIN_AFFINE, 64, **_in_bn(g, MAX_CIN_AFFINE, 300, 2)),
    # mode 1: group extrema on both paths (K = 32 divides the 64-row half tile, K = 20 and 128 need atomics), empty balls
    "m1_K20_D6": lambda g: _mode1(g, 2, 900, 33, 20, 6, 0, 129),
    "m1_K32_D61": lambda g: _mode1(g, 2, 700, 21, 32, 61, 1, 64),
    "m1_K128_D0": lambda g: _mode1(g, 2, 600, 5, 128, 0, 0, 128),
    # mode 2: EdgeConv operand, LeakyReLU after the input BatchNorm (batch sums / running statistics), negative scales
    "m2_bn_batch_leaky": lambda g: _mode2(g, 1),
    "m2_bn_running_leaky": lambda g: _mode2(g, 2),
    "m2_K16_bn_running_leaky": lambda g: _mode2(g, 2, K=16),
}


@pytest.mark.parametrize("case", list(CASES))
def test_launch_within_the_bound(case):
    f = CASES[case](torch.Generator().manual_seed(sum(map(ord, case))))
    y, ymax, ymin, stats, _ = launch(f, 1)
    assert ratio(y, f) <= 1.0, case
    G = f.get("group", 0)
    if G:
        gy = y.view(f["cout"], f["rows"] // G, G)
        assert torch.equal(ymax, gy.amax(2)) and torch.equal(ymin, gy.amin(2))
    # the fp64 sums are those of the launch's own y
    yd = y.double()
    c, n = yd.shape
    assert torch.allclose(stats[:c] / n, yd.mean(1), rtol=0, atol=1e-6 * float(yd.std(1).max()) + 1e-12)


def test_rows_are_independent():
    """rows 77 .. 376 of a launch, launched alone through an offset segment, are bitwise the same: no row's arithmetic depends on
    the tile it lands in"""
    gen = torch.Generator().manual_seed(5)
    f = _mode0(gen, 1, 1000, 300, 130, cloud_bias=True, **_in_bn(gen, 300, 1000, 2, slope=0.2))
    y_all = launch(f, 1)[0]
    lo, n = 77, 300
    x = f["seg_ptr"][0]
    g = dict(f, rows=n, rows_per_batch=n, seg_ptr=(x[:, :, lo:lo + n].contiguous(),), seg_batch_stride=(300 * n, 0),
             seg_chan_stride=(n, 0))
    y_part = launch(g, 1)[0]
    assert torch.equal(y_all[:, lo:lo + n].view(torch.int32), y_part.view(torch.int32))


def test_refusals():
    """an unknown accum, a group the half tile needs atomics for, and a cin past the shared memory: an error naming the problem,
    no launch, the output untouched"""
    gen = torch.Generator().manual_seed(3)
    y = torch.full((16, 64), 7.0, device="cuda")

    def refused(f, match, **fields):
        d, dev = _descriptor(f)
        d.y = L.ptr(y)
        for k, v in fields.items():
            setattr(d, k, v)
        before = L.launch_count()
        with pytest.raises(L.TgnError, match=match):
            L.call("tgn_pw_layer_forward", ctypes.byref(d), L.stream_ptr())
        torch.cuda.synchronize()
        assert L.launch_count() == before
        assert bool((y == 7.0).all())

    base = _mode0(gen, 1, 64, 8, 16)
    refused(base, "unknown accum 2", accum=2)
    refused(base, "unknown accum -1", accum=-1)
    g1 = _mode1(gen, 1, 50, 4, 128, 0, 1, 16)
    fill = torch.empty(16 * 4, device="cuda")
    refused(g1, "group 128 needs the atomic extrema path", accum=1, ymax=L.ptr(fill), ymin=L.ptr(fill), group=128, extrema_atomic=0)
    wide = _mode0(gen, 1, 64, MAX_CIN_AFFINE + 1, 16, **_in_bn(gen, MAX_CIN_AFFINE + 1, 64, 2))
    refused(wide, f"cin {MAX_CIN_AFFINE + 1} too wide", accum=1)
