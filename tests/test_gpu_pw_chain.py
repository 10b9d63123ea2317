"""GPU: the batch-statistics layer chain (csrc/pw_mlp.cu) one launch at a time against its float64 restatement
(oracle/pw_chain.py), and as modules in training mode against the float64 oracle.

Per tgn_pw_layer_forward launch:
* y element-wise within 5e-5 (5 % floor) at precision 3 for up to 16 K chunks of 32 (cin <= 512), a bound that grows with the
  number of chunks beyond that (the fp32 MMA accumulator collects six products per element per K step: 1.1e-4 measured at
  cin = 1536 on an H100); at precision 2, norm-wise within 1e-5 (include/tgn_b200.h: two bf16 parts per operand, ~1e-5);
* ymax / ymin equal to the max / min over groups of the kernel's own y, written by the same launch (values equal: a -0.0 / +0.0
  pair is the one difference torch.equal lets through);
* the fp64 sums against float64 sums of the kernel's own y: mean within 1e-6 std, variance within 1e-5 relative, on channels whose
  |mean| / std reaches 1000 as well;
* the running statistics the launch updates within 1e-6 relative.
tgn_pw_apply against float64 with negative, zero and positive BatchNorm scales, and the refusals of both entry points."""
import ctypes

import pytest
import torch
import torch.nn as nn

from oracle import oracle, pw_chain
from toothgroupnetwork_b200 import _lib as L
from toothgroupnetwork_b200 import clouds
from toothgroupnetwork_b200 import pointnet2_utils as pn2

pytestmark = pytest.mark.gpu
FLOOR = 0.05


def y_bound(precision, cin):
    """precision 3: element-wise, 5e-5 up to 16 K chunks and proportional to the chunk count above; precision 2: norm-wise"""
    return 1e-5 if precision == 2 else 5e-5 * max(1.0, (cin + 31) // 32 / 16)

_INT = ("rows", "rows_per_batch", "cin", "cout", "mode", "N", "S", "K", "D", "xyz_first", "in_affine", "in_update_running", "edge_C",
        "in_act", "group", "precision")
_FLOAT = ("in_eps", "in_momentum", "in_act_slope")
_ARRAY = ("seg_channels", "seg_batch_stride", "seg_row_stride", "seg_chan_stride", "edge_stride")
_PTR = ("xyz", "feats", "new_xyz", "gidx", "in_stats", "in_gamma", "in_beta", "in_running_mean", "in_running_var", "bias",
        "cloud_bias", "edge_x")


def elementwise(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float(((a - b).abs() / b.abs().clamp(min=FLOOR * float(b.abs().max()))).max())


def normwise(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / b.norm())


def _packed(w):
    cout, cin = w.shape
    buf = torch.empty(L.load().tgn_pw_packed_bytes(cout, cin), dtype=torch.uint8, device="cuda")
    L.call("tgn_pw_pack_weights", cout, cin, L.ptr(w), L.ptr(buf), L.stream_ptr())
    return buf


def _descriptor(f):
    """PwLayer from an oracle field dict (CPU tensors) -> (descriptor, the device copies it points to, by field name)"""
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


# ------------------------------------------------------------------------------------------------------------ case builders
def _weight(gen, cout, cin):
    return torch.randn(cout, cin, generator=gen) / cin ** 0.5


def _in_bn(gen, cin, rows, mode, slope=None, update=False):
    """input BatchNorm fields: gamma with negative and zero entries, batch sums of a (mean, var) per channel"""
    m = torch.randn(cin, generator=gen, dtype=torch.float64) * 0.5
    v = torch.rand(cin, generator=gen, dtype=torch.float64) + 0.2
    gamma = torch.randn(cin, generator=gen)
    gamma[::7] = 0.0
    f = {"in_affine": mode, "in_gamma": gamma, "in_beta": torch.randn(cin, generator=gen) * 0.2,
         "in_running_mean": torch.randn(cin, generator=gen) * 0.3, "in_running_var": torch.rand(cin, generator=gen) + 0.5,
         "in_eps": 1e-5, "in_momentum": 0.1}
    if mode == 1:
        f["in_stats"] = torch.cat([rows * m, rows * (v + m * m)])
        f["in_update_running"] = int(update)
    if slope is not None:
        f.update(in_act=1, in_act_slope=slope)
    return f


def _mode0(gen, B, n, cin, cout, segs="cf", cloud_bias=False, **extra):
    """segs: 'cf' one channel-first segment; 'fp' [skip channel-first (3 channels) | interpolated point-major];
    'fp_s1' [skip (64) | one coarse row per cloud read with row stride 0] (feature propagation with S == 1)"""
    rows = B * n
    f = {"rows": rows, "cin": cin, "cout": cout, "mode": 0, "rows_per_batch": n, "weight": _weight(gen, cout, cin),
         "bias": torch.randn(cout, generator=gen) * 0.1}
    if segs == "cf":
        x = torch.randn(B, cin, n, generator=gen)
        f.update(seg_ptr=(x,), seg_channels=(cin, 0), seg_batch_stride=(cin * n, 0), seg_row_stride=(1, 0), seg_chan_stride=(n, 0))
    else:
        d1 = 3 if segs == "fp" else 64
        d2 = cin - d1
        skip = torch.randn(B, d1, n, generator=gen)
        if segs == "fp":
            interp = torch.randn(B, n, d2, generator=gen)
            s2 = (n * d2, d2, 1)
        else:
            interp = torch.randn(B, 1, d2, generator=gen)
            s2 = (d2, 0, 1)
        f.update(seg_ptr=(skip, interp), seg_channels=(d1, d2), seg_batch_stride=(d1 * n, s2[0]), seg_row_stride=(1, s2[1]),
                 seg_chan_stride=(n, s2[2]))
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


def _offset(gen, rows, **extra):
    """channels 0, 4, 8, ..: bias 100, spread ~0.1 (|mean| / std ~ 1000); channels 1, 5, ..: bias 10, spread ~0.1 (~100)"""
    cin, cout = 32, 128
    f = _mode0(gen, 1, rows, cin, cout, **extra)
    w = f["weight"]
    w[0::4] *= 0.1 / w[0::4].norm(dim=1, keepdim=True)
    w[1::4] *= 0.1 / w[1::4].norm(dim=1, keepdim=True)
    f["bias"][0::4] = 100.0
    f["bias"][1::4] = 10.0
    return f


def _mode2(gen, in_mode):
    B, C, N, K, cout = 2, 17, 300, 20, 70
    base = torch.randn(B, 2 * C + 1, N, generator=gen)
    x = base[:, 1::2]
    idx = torch.randint(0, N, (B, N, K), generator=gen, dtype=torch.int32)
    idx[0, 3, 1], idx[-1, N - 1, K - 1] = N, -1
    rows = B * N * K
    f = {"rows": rows, "cin": 2 * C, "cout": cout, "mode": 2, "rows_per_batch": N * K, "edge_x": base.reshape(-1)[1:],
         "edge_stride": x.stride(), "edge_C": C, "gidx": idx, "N": N, "K": K, "weight": _weight(gen, cout, 2 * C), "group": K}
    f.update(_in_bn(gen, 2 * C, rows, in_mode, slope=0.2, update=True))
    return f


CASES = {
    # mode 0: channel-first and feature-propagation segments, row counts around the 256-row tile, K chunks and affine tables
    "m0_cin1_rows257": lambda g: _mode0(g, 1, 257, 1, 129),
    "m0_cin32_rpb85_rows255": lambda g: _mode0(g, 3, 85, 32, 1, cloud_bias=True),
    "m0_fp_cin67_rows3000_cloud_bias": lambda g: _mode0(g, 2, 1500, 67, 128, segs="fp", cloud_bias=True),
    "m0_fp_s1_cin320_rows1554": lambda g: _mode0(g, 2, 777, 320, 63, segs="fp_s1"),
    "m0_cin1536_rows256_bn_batch_leaky": lambda g: _mode0(g, 1, 256, 1536, 1024, **_in_bn(g, 1536, 256, 1, slope=0.2, update=True)),
    "m0_cin31_rows1_bn_running": lambda g: _mode0(g, 1, 1, 31, 1024, **_in_bn(g, 31, 1, 2)),
    "m0_cin33_rows1000_precision2_bn_running": lambda g: _mode0(g, 1, 1000, 33, 129, precision=2, **_in_bn(g, 33, 1000, 2)),
    "m0_cin320_rows3001_precision2_bn_batch": lambda g: _mode0(g, 1, 3001, 320, 128, precision=2,
                                                               **_in_bn(g, 320, 3001, 1, update=True)),
    "m0_cin3_rows5003_bn_batch": lambda g: _mode0(g, 1, 5003, 3, 1024, **_in_bn(g, 3, 5003, 1, update=True)),
    # channels whose |mean| / std is 100 and 1000
    "m0_offset_rows256": lambda g: _offset(g, 256),
    "m0_offset_rows2048": lambda g: _offset(g, 2048),
    "m0_offset_rows7001_precision2": lambda g: _offset(g, 7001, precision=2),
    # mode 1: both channel orders, K on both extrema paths, groups across the two 128-row halves and across CTAs
    "m1_K1_D6": lambda g: _mode1(g, 2, 500, 100, 1, 6, 0, 64),
    "m1_K16_D0": lambda g: _mode1(g, 2, 800, 40, 16, 0, 1, 64),
    "m1_K20_D6": lambda g: _mode1(g, 2, 900, 33, 20, 6, 0, 129),
    "m1_K24_D61": lambda g: _mode1(g, 2, 700, 21, 24, 61, 1, 64),
    "m1_K64_D6": lambda g: _mode1(g, 2, 600, 9, 64, 6, 1, 63),
    "m1_K128_D0": lambda g: _mode1(g, 2, 600, 5, 128, 0, 0, 128),
    "m1_K200_D6": lambda g: _mode1(g, 2, 900, 7, 200, 6, 0, 129),
    "m1_K256_D61": lambda g: _mode1(g, 1, 900, 3, 256, 61, 1, 1024),
    # mode 2: EdgeConv operand with an input BatchNorm and LeakyReLU
    "m2_bn_batch_leaky": lambda g: _mode2(g, 1),
    "m2_bn_running_leaky": lambda g: _mode2(g, 2),
}


def _stats_check(stats, y):
    """the kernel's sums against float64 sums of its own y: mean within 1e-6 std, variance within 1e-5 relative.  The floors are
    what float64 itself gives the sum / sum-of-squares form (its rounding of sum y^2 / n - mean^2)."""
    yd = y.double()
    n = yd.shape[1]
    c = yd.shape[0]
    mean, var = yd.mean(1), yd.var(1, unbiased=False)
    km = stats[:c] / n
    kv = stats[c:] / n - km * km
    eps64 = 2.0 ** -52
    dm = (km - mean).abs() / (1e-6 * var.sqrt() + 4 * eps64 * mean.abs() + 1e-300)
    dv = (kv - var).abs() / (1e-5 * var + 8 * eps64 * mean * mean + 1e-300)
    return float(dm.max()), float(dv.max())


@pytest.mark.parametrize("case", list(CASES))
def test_layer_launch_against_float64(case):
    f = CASES[case](torch.Generator().manual_seed(sum(map(ord, case))))
    d, dev = _descriptor(f)
    rows, cout, G = f["rows"], f["cout"], f.get("group", 0)
    y = torch.empty((cout, rows), dtype=torch.float32, device="cuda")
    stats = torch.zeros(2 * cout, dtype=torch.float64, device="cuda")
    d.y, d.stats = L.ptr(y), L.ptr(stats)
    if G:
        ymax = torch.full((cout, rows // G), float("-inf"), device="cuda")
        ymin = torch.full((cout, rows // G), float("inf"), device="cuda")
        d.ymax, d.ymin, d.extrema_atomic = L.ptr(ymax), L.ptr(ymin), 1 if 128 % G else 0
    L.call("tgn_pw_layer_forward", ctypes.byref(d), L.stream_ptr())
    torch.cuda.synchronize()
    want = pw_chain.layer_forward(**f)
    y = y.cpu()
    prec = f.get("precision", 3)
    err = elementwise(y, want["y"]) if prec == 3 else normwise(y, want["y"])
    assert err <= y_bound(prec, f["cin"]), (case, err)
    if G:
        gy = y.view(cout, rows // G, G)
        assert torch.equal(ymax.cpu(), gy.amax(2)) and torch.equal(ymin.cpu(), gy.amin(2))
    dm, dv = _stats_check(stats.cpu(), y)
    assert dm <= 1.0 and dv <= 1.0, (case, dm, dv)
    if f.get("in_update_running"):
        rm, rv = dev["in_running_mean"].cpu().double(), dev["in_running_var"].cpu().double()
        wm, wv = pw_chain.running_update(f["in_stats"], rows, f["in_momentum"], f["in_running_mean"], f["in_running_var"])
        assert elementwise(rm, wm) <= 1e-6 and elementwise(rv, wv) <= 1e-6



@pytest.mark.parametrize("affine", [1, 2])
@pytest.mark.parametrize("act", ["relu", "leaky", "none"])
@pytest.mark.parametrize("extrema", [True, False])
def test_apply_against_float64(affine, act, extrema):
    """BatchNorm (batch sums or running statistics) + activation into a channel slice of a (B, C_total, n) tensor; with extrema,
    the max where the scale is >= 0 and the min where it is negative (gamma has negative, zero and positive entries)"""
    gen = torch.Generator().manual_seed(31 + affine)
    C, B, n, c_total, c_off = 37, 3, 50, 45, 5
    rows = B * n
    src = torch.randn(C, rows, generator=gen) + 2.0
    ymin = src - torch.rand(C, rows, generator=gen) - 1.0
    gamma = torch.randn(C, generator=gen)
    gamma[::6] = 0.0
    m = torch.randn(C, generator=gen, dtype=torch.float64)
    v = torch.rand(C, generator=gen, dtype=torch.float64) + 0.3
    stat_rows = 4000
    f = {"rows": rows, "rows_per_batch": n, "channels": C, "out_channels": c_total, "out_c_offset": c_off,
         "relu": 1 if act == "relu" else 0, "act": 1 if act == "leaky" else 0, "act_slope": 0.2, "affine": affine,
         "stats": torch.cat([stat_rows * m, stat_rows * (v + m * m)]), "stat_rows": stat_rows, "gamma": gamma,
         "beta": torch.randn(C, generator=gen) * 0.3, "running_mean": torch.randn(C, generator=gen),
         "running_var": torch.rand(C, generator=gen) + 0.5, "eps": 1e-5, "momentum": 0.01, "update_running": 1}
    dev = {k: f[k].cuda() for k in ("stats", "gamma", "beta", "running_mean", "running_var")}
    out = torch.full((B, c_total, n), 7.0, device="cuda")
    s_dev, m_dev = src.cuda(), ymin.cuda()
    a = L.PwApply()
    for k in ("rows", "rows_per_batch", "channels", "out_channels", "out_c_offset", "relu", "affine", "update_running", "stat_rows",
              "act"):
        setattr(a, k, int(f[k]))
    a.eps, a.momentum, a.act_slope = 1e-5, 0.01, 0.2
    a.src, a.ymin, a.out = L.ptr(s_dev), L.ptr(m_dev) if extrema else None, L.ptr(out)
    for k, t in dev.items():
        setattr(a, k, L.ptr(t))
    L.call("tgn_pw_apply", ctypes.byref(a), L.stream_ptr())
    torch.cuda.synchronize()
    want = pw_chain.apply(src=src, ymin=ymin if extrema else None, **{k: v for k, v in f.items() if k not in ("rows",)})
    got = out.cpu()
    assert elementwise(got[:, c_off:c_off + C], want) <= 2e-6
    assert bool((got[:, :c_off] == 7.0).all()) and bool((got[:, c_off + C:] == 7.0).all())
    if affine == 1:
        wm, wv = pw_chain.running_update(f["stats"], stat_rows, 0.01, f["running_mean"], f["running_var"])
        assert elementwise(dev["running_mean"], wm) <= 1e-6 and elementwise(dev["running_var"], wv) <= 1e-6
    else:
        assert torch.equal(dev["running_mean"].cpu(), f["running_mean"]) and torch.equal(dev["running_var"].cpu(), f["running_var"])


def test_refusals():
    """tgn_pw_layer_forward / tgn_pw_apply refuse malformed descriptors with a message naming the problem, before any launch"""
    gen = torch.Generator().manual_seed(3)
    base = _mode0(gen, 1, 64, 8, 16)
    g1 = _mode1(gen, 1, 50, 4, 8, 0, 1, 16)
    e2 = _mode2(gen, 1)
    y = torch.empty(16 * 64, device="cuda")
    fill = torch.empty(16 * 64, device="cuda")

    def refused(f, match, **fields):
        d, dev = _descriptor(f)
        d.y = L.ptr(y)
        for k, v in fields.items():
            if k.startswith("seg_"):
                getattr(d, k[:-2])[int(k[-1])] = v
            else:
                setattr(d, k, v)
        with pytest.raises(L.TgnError, match=match):
            L.call("tgn_pw_layer_forward", ctypes.byref(d), L.stream_ptr())

    refused(base, "bad shape", rows=0)
    refused(base, "bad shape", cout=0)
    refused(base, "bad shape", w_packed=None)
    refused(base, "bad segments", seg_channels_0=7)
    refused(base, "bad segments", seg_ptr_0=None)
    refused(base, "bad segments", rows_per_batch=0)
    refused(base, "bad segments", cin=12, seg_channels_1=4)
    refused(g1, "bad gather arguments", cin=4)
    refused(g1, "bad gather arguments", K=0)
    refused(g1, "bad gather arguments", gidx=None)
    refused(e2, "edge-feature", rows=e2["rows"] - e2["K"])
    refused(e2, "edge-feature", cin=35)
    refused(base, "unknown mode 3", mode=3)
    refused(g1, "cloud_bias needs rows_per_batch", rows_per_batch=0, cloud_bias=L.ptr(fill))
    refused(base, "in_affine=1 needs in_stats", in_affine=1)
    refused(base, "in_affine=2 needs running statistics", in_affine=2)
    refused(g1, "bad extrema arguments", ymax=L.ptr(fill), ymin=None, group=8)
    refused(g1, "bad extrema arguments", ymax=L.ptr(fill), ymin=L.ptr(fill), group=6)
    refused(g1, "group 24 needs the atomic extrema path", ymax=L.ptr(fill), ymin=L.ptr(fill), group=24, rows=g1["rows"] * 3)
    refused(base, "cin 6000 too wide", cin=6000, seg_channels_0=6000, in_affine=2, in_running_mean=L.ptr(fill),
            in_running_var=L.ptr(fill))
    a = L.PwApply()
    a.rows, a.rows_per_batch, a.channels, a.src, a.out = 64, 64, 16, L.ptr(fill), L.ptr(y)
    for k, v, match in (("rows", 0, "bad arguments"), ("rows_per_batch", 0, "bad arguments"), ("src", None, "bad arguments"),
                        ("affine", 1, "affine=1 needs stats")):
        bad = L.PwApply.from_buffer_copy(a)
        setattr(bad, k, v)
        with pytest.raises(L.TgnError, match=match):
            L.call("tgn_pw_apply", ctypes.byref(bad), L.stream_ptr())


# ------------------------------------------------------------------------------------------------------------ chain level
@pytest.fixture
def _reference_on_cpu():
    """the oracle restates FPS / ball query / 3-NN on CPU tensors (index-order |p|^2 rounding)"""
    pn2.set_reference_device("cpu")
    yield
    pn2.set_reference_device("cuda")


def _params(convs, bns):
    return [oracle.MlpParams(c.weight.detach().cpu().reshape(c.weight.shape[0], -1), c.bias.detach().cpu(), b.weight.detach().cpu(),
                             b.bias.detach().cpu(), b.running_mean.detach().cpu(), b.running_var.detach().cpu(), b.eps)
            for c, b in zip(convs, bns)]


def _seed_bn(module, gen):
    """BatchNorm scales of both signs (a negative scale makes the set abstraction take the minimum over the neighbours)"""
    for m in module.modules():
        if isinstance(m, (nn.BatchNorm1d, nn.BatchNorm2d)):
            with torch.no_grad():
                m.weight.copy_(torch.randn(m.weight.shape, generator=gen))
                m.bias.copy_(torch.randn(m.bias.shape, generator=gen) * 0.1)


def _offset_conv(conv, gen):
    """every third output channel: weight x 0.002 and bias + 1 (|mean| / std ~ 1000 in front of its BatchNorm), the next ones
    x 0.02 and + 1 (~ 100)"""
    with torch.no_grad():
        conv.weight[0::3] *= 0.002
        conv.bias[0::3] += 1.0
        conv.weight[1::3] *= 0.02
        conv.bias[1::3] += 1.0


def rel_err(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).abs().max() / b.abs().max())


def _both(module, *inputs):
    """(library chain, torch's fp32 conv + BatchNorm of the same module), both in training mode without autograd"""
    with torch.no_grad():
        ours = module(*inputs)
        pn2.set_pw_enabled(False)
        try:
            ref32 = module(*inputs)
        finally:
            pn2.set_pw_enabled(True)
    return ours, ref32


def _points(B, N, seed):
    return torch.cat([clouds.arch_features(N, seed + b) for b in range(B)], 0)            # (B, 6, N)


SA_CHAINS = {
    # name: (npoint, radius, nsample, widths, group_all, N, seeded_scales, offset)
    "ssg_K24": (256, 0.1, 24, [32, 64], False, 4000, False, False),
    "ssg_K24_wide_negative": (200, 0.15, 24, [64, 160, 192], False, 3000, True, False),
    "group_all_N1000": (None, None, None, [64, 128, 256], True, 1000, True, False),
    "ssg_offset_channels": (256, 0.1, 32, [32, 48, 64], False, 4000, True, True),
}


@pytest.mark.parametrize("name", list(SA_CHAINS))
def test_set_abstraction_train_mode_against_float64(name, _reference_on_cpu):
    npoint, radius, nsample, widths, group_all, N, seeded, offset = SA_CHAINS[name]
    B = 2
    gen = torch.Generator().manual_seed(sum(map(ord, name)))
    torch.manual_seed(5)
    feats = _points(B, N, 40)
    sa = pn2.PointNetSetAbstraction(npoint, radius, nsample, 9, widths, group_all)
    if seeded:
        _seed_bn(sa, gen)
    if offset:
        _offset_conv(sa.mlp_convs[1], gen)
    sa = sa.cuda().train()
    (nx, ours), (_, ref32) = _both(sa, feats[:, :3].contiguous().cuda(), feats.cuda())
    wx, want = oracle.set_abstraction(feats[:, :3].contiguous(), feats, npoint, radius, nsample, _params(sa.mlp_convs, sa.mlp_bns),
                                      group_all=group_all, train_bn=True, dtype=torch.float64)
    if not group_all:
        assert torch.equal(nx.cpu(), wx)
    e_ours, e_32 = rel_err(ours, want), rel_err(ref32, want)
    assert e_ours <= max(1e-4, 2 * e_32), (name, e_ours, e_32)


def test_set_abstraction_msg_train_mode_against_float64(_reference_on_cpu):
    """two radii with K = 20 (atomic extrema) and 32, seeded negative scales"""
    B, N = 2, 3000
    gen = torch.Generator().manual_seed(17)
    feats = _points(B, N, 50)
    msg = pn2.PointNetSetAbstractionMsg(128, [0.1, 0.2], [20, 32], 6, [[32, 48], [32, 144]])
    _seed_bn(msg, gen)
    msg = msg.cuda().train()
    (nx, ours), (_, ref32) = _both(msg, feats[:, :3].contiguous().cuda(), feats.cuda())
    wx, want = oracle.set_abstraction_msg(feats[:, :3].contiguous(), feats, 128, [0.1, 0.2], [20, 32],
                                          [_params(c, b) for c, b in zip(msg.conv_blocks, msg.bn_blocks)], train_bn=True,
                                          dtype=torch.float64)
    assert torch.equal(nx.cpu(), wx)
    e_ours, e_32 = rel_err(ours, want), rel_err(ref32, want)
    assert e_ours <= max(1e-4, 2 * e_32), (e_ours, e_32)


@pytest.mark.parametrize("S,skip,widths,offset", [(300, 6, [160, 96], False), (1, 6, [128, 64], False), (500, 0, [64, 32], False),
                                                  (300, 6, [96, 64, 32], True)])
def test_feature_propagation_train_mode_against_float64(S, skip, widths, offset, _reference_on_cpu):
    """3-NN interpolation (or the S == 1 broadcast, row stride 0) + skip features, seeded negative scales"""
    B, N, D2 = 2, 2000, 48
    gen = torch.Generator().manual_seed(S + skip)
    fine = _points(B, N, 60)
    xyz1 = fine[:, :3].contiguous()
    xyz2 = xyz1[:, :, :S].contiguous() if S > 1 else torch.zeros(B, 3, 1)
    points1 = fine if skip else None
    points2 = torch.randn(B, D2, S, generator=gen)
    fp = pn2.PointNetFeaturePropagation(skip + D2, widths)
    _seed_bn(fp, gen)
    if offset:
        _offset_conv(fp.mlp_convs[0], gen)
    fp = fp.cuda().train()
    ours, ref32 = _both(fp, xyz1.cuda(), xyz2.cuda(), None if points1 is None else points1.cuda(), points2.cuda())
    want = oracle.feature_propagation(xyz1, xyz2, points1, points2, _params(fp.mlp_convs, fp.mlp_bns), train_bn=True,
                                      dtype=torch.float64)
    e_ours, e_32 = rel_err(ours, want), rel_err(ref32, want)
    assert e_ours <= max(1e-4, 2 * e_32), (e_ours, e_32)
