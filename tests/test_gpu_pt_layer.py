"""GPU: the fused point-transformer layer (csrc/pt_layer.cu) called through tgn_pt_layer_forward directly, one pass at a time,
against its float64 restatement (oracle/pt_layer.py).

* Per pass: bn_mode [1,2,2], [2,1,2] and [2,2,1] each run one statistics pass (and the output pass), [2,2,2] the output pass
  alone, [1,1,1] all four.  Every {sum, sumsq} the launch writes is within its bound of ``batch_sums`` conditioned on the
  launch's own earlier sums, and ``out`` within its element-wise bound of ``output`` conditioned on all of them, under both
  schedules (warp and CTA per query) and the default threshold on both sides.
* The running statistics of every mode-1 BatchNorm within 4 float32 ulps of torch's momentum update of the launch's sums;
  mode-2 BatchNorms, null running pointers and update_running = 0 leave the buffers bitwise unchanged.
* One launch per mode-1 BatchNorm, one for the output, one for the running update; out and the three stats ranges written
  where they belong and nowhere else; the refusals.
Shapes are the two networks' levels (one cloud of 24 000 points; 16 crops of 3 072 packed, whose deepest level has 12 points
per crop and K = 24, so every neighbourhood there is padded), the K edges 1..64 and the n edges of both grid-stride loops;
neighbourhoods come from pointops.knn_packed on dental arches."""
import contextlib
import ctypes

import pytest
import torch

from oracle import pt_layer
from toothgroupnetwork_b200 import _lib as L
from toothgroupnetwork_b200 import clouds, pointops

pytestmark = pytest.mark.gpu
MODES = ([1, 2, 2], [2, 1, 2], [2, 2, 1], [2, 2, 2], [1, 1, 1])
TAGS = ("p", "a", "b")
GUARD = 7
SELECT = 256
WORST = {}
_IN = ("p", "xq", "xk", "xv", "idx", "p_w0", "p_b0", "p_w1", "p_b1", "a_w", "a_b", "b_w", "b_b",
       "p_gamma", "p_beta", "a_gamma", "a_beta", "b_gamma", "b_beta")
_RUNNING = ("p_rmean", "p_rvar", "a_rmean", "a_rvar", "b_rmean", "b_rvar")
REQUIRED = ("p", "xq", "xk", "xv", "idx", "out", "p_w0", "p_b0", "p_w1", "p_b1", "a_w", "a_b", "b_w", "b_b",
            "stats_p", "stats_a", "stats_b")
WARP, CTA, DEFAULT = 0, 1 << 30, None


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


@contextlib.contextmanager
def _threshold(value):
    lib = L.load()
    old = lib.tgn_pt_layer_set_cta_threshold(1024)
    lib.tgn_pt_layer_set_cta_threshold(old if value is None else value)
    try:
        yield
    finally:
        lib.tgn_pt_layer_set_cta_threshold(old)


def _cloud(n, K, crops=1, seed=0):
    """a dental arch of n points, or `crops` arches of n / crops points packed, and its kNN (n, K) -> CPU tensors"""
    per = n // crops
    p = torch.cat([clouds.dental_arch(per, seed + k)[0] for k in range(crops)]).cuda().contiguous()
    o = (torch.arange(1, crops + 1, dtype=torch.int32) * per).cuda()
    idx, _ = pointops.knn_packed(K, p, p, o, o)
    return p.cpu(), idx.cpu()


def _case(c, K, n, crops=1, kind="hard"):
    p, idx = _cloud(n, K, crops, seed=c + K)
    return pt_layer.make_case(c, K, p, idx, kind, seed=n + K)


def _nan_bits(t):
    return t.view(torch.int64 if t.dtype == torch.float64 else torch.int32)


def _launch(f, modes, update=1, null=(), expect_ok=True):
    """one tgn_pt_layer_forward -> dict(out (n, c), stats {tag: sums}, running {field: tensor}, launches), having checked that
    out and the stats ranges were written where they belong and nowhere else"""
    n, c = f["n"], f["c"]
    cs = c // 8
    dev = {k: f[k].cuda().contiguous() for k in _IN if f.get(k) is not None}
    run = {k: f[k].cuda().clone() for k in _RUNNING}
    out_buf = torch.full((n * c + 2 * GUARD,), float("nan"), device="cuda")
    sizes = {"p": 6, "a": 2 * c, "b": 2 * cs}
    starts, at = {}, GUARD
    for t in TAGS:
        starts[t] = at
        at += sizes[t] + GUARD
    st_buf = torch.full((at,), float("nan"), dtype=torch.float64, device="cuda")
    for t in TAGS:
        st_buf[starts[t]:starts[t] + sizes[t]] = 0.0
    d = L.PtLayer()
    d.n, d.c, d.K = n, c, f["K"]
    ptrs = {k: L.ptr(v) for k, v in dev.items()}
    ptrs.update({k: L.ptr(v) for k, v in run.items()})
    ptrs["out"] = out_buf.data_ptr() + GUARD * 4
    ptrs.update({"stats_" + t: st_buf.data_ptr() + starts[t] * 8 for t in TAGS})
    for k, v in ptrs.items():
        setattr(d, k, None if k in null else v)
    for t in TAGS:
        setattr(d, t + "_eps", float(f[t + "_eps"]))
        setattr(d, t + "_momentum", float(f[t + "_momentum"]))
    for i in range(3):
        d.bn_mode[i] = int(modes[i])
    d.update_running = int(update)
    before_out, before_st, before_run = out_buf.clone(), st_buf.clone(), {k: v.clone() for k, v in run.items()}
    launches = L.launch_count()
    try:
        L.call("tgn_pt_layer_forward", ctypes.byref(d), L.stream_ptr())
    except L.TgnError:
        if expect_ok:
            raise
        torch.cuda.synchronize()
        assert L.launch_count() == launches
        assert torch.equal(_nan_bits(out_buf), _nan_bits(before_out)) and torch.equal(_nan_bits(st_buf), _nan_bits(before_st))
        assert all(torch.equal(run[k], before_run[k]) for k in run)
        return None
    torch.cuda.synchronize()
    assert expect_ok, "the launch was not refused"
    res = {"launches": L.launch_count() - launches, "running": {k: v.cpu() for k, v in run.items()},
           "before_running": {k: v.cpu() for k, v in before_run.items()}}
    nanb = _nan_bits(before_out)[0]
    assert bool((_nan_bits(out_buf[:GUARD]) == nanb).all() and (_nan_bits(out_buf[-GUARD:]) == nanb).all())
    if n > 0:
        res["out"] = out_buf[GUARD:GUARD + n * c].view(n, c).cpu()
        assert not bool(torch.isnan(res["out"]).any()), "an element of out was not written"
    stn = _nan_bits(before_st)[0]
    for t in TAGS:
        for a, b in ((starts[t] - GUARD, starts[t]), (starts[t] + sizes[t], starts[t] + sizes[t] + GUARD)):
            assert bool((_nan_bits(st_buf[a:b]) == stn).all()), f"stats guard next to {t}"
    res["stats"] = {t: st_buf[starts[t]:starts[t] + sizes[t]].cpu() for t in TAGS}
    for i, t in enumerate(TAGS):
        if modes[i] != 1 or n == 0:
            assert not bool(res["stats"][t].any()), f"stats_{t} written in mode {modes[i]}"
    return res


def _ratio(key, err, bound):
    assert bool((err <= bound).all()), (key, float((err - bound).max()))
    r = float((err / bound.clamp(min=1e-300)).max())
    WORST[key] = max(WORST.get(key, 0.0), r)
    return r


def _select(idx):
    """SELECT queries at random, plus the first, the last and one with a padded neighbourhood (a repeated index)"""
    n = idx.shape[0]
    if n <= SELECT:
        return list(range(n))
    sel = set(torch.randperm(n, generator=torch.Generator().manual_seed(n))[:SELECT].tolist()) | {0, n - 1}
    srt = idx.sort(1).values
    padded = torch.nonzero((srt[:, 1:] == srt[:, :-1]).any(1)).flatten()
    if padded.numel():
        sel.add(int(padded[-1]))
    return sorted(sel)


def _ulp(x):
    x = x.abs().float()
    return (torch.nextafter(x, torch.full_like(x, float("inf"))) - x).double()


def _check(f, modes, got, update=1, null=()):
    fm = dict(f, bn_mode=modes, update_running=update)
    cond = {"stats_" + t: got["stats"][t] for i, t in enumerate(TAGS) if modes[i] == 1}
    sums = pt_layer.batch_sums(**fm, **cond)
    for t, (s, b) in sums.items():
        _ratio("sums_" + t, (got["stats"][t] - s).abs(), b)
    sel = _select(f["idx"])
    want, bound = pt_layer.output(select=sel, **fm, **cond)
    _ratio("out", (got["out"][sel].double() - want).abs(), bound)
    assert got["launches"] == sum(m == 1 for m in modes) + 1 + int(update)
    fm.update({k: None for k in null})
    upd = pt_layer.running_update(**fm, **cond)
    for i, t in enumerate(TAGS):
        for j, k in enumerate((t + "_rmean", t + "_rvar")):
            if t in upd and k not in null:
                m = float(torch.tensor(f[t + "_momentum"], dtype=torch.float32))
                old = got["before_running"][k].double()
                batch = (upd[t][j] - (1 - m) * old) / m
                scale = (1 - m) * old.abs() + m * batch.abs()
                _ratio("running", (got["running"][k].double() - upd[t][j]).abs(), 4 * _ulp(scale))
            else:
                assert torch.equal(got["running"][k], got["before_running"][k]), k


def _all_modes(f, schedule):
    with _threshold(schedule):
        for modes in MODES:
            _check(f, modes, _launch(f, modes))


FIRST = [(32, 36, 24000), (64, 24, 6000), (128, 24, 1500), (256, 24, 375), (512, 24, 93)]
SECOND = [(32, 36, 49152), (64, 24, 12288), (128, 24, 3072), (256, 24, 768), (512, 24, 192)]


@pytest.mark.parametrize("schedule", [WARP, CTA], ids=["warp", "cta"])
@pytest.mark.parametrize("c,K,n", FIRST)
def test_first_network_levels(c, K, n, schedule):
    _all_modes(_case(c, K, n), schedule)


@pytest.mark.parametrize("schedule", [WARP, CTA], ids=["warp", "cta"])
@pytest.mark.parametrize("c,K,n", SECOND)
def test_second_network_levels_16_crops(c, K, n, schedule):
    f = _case(c, K, n, crops=16)
    if n // 16 < K:
        srt = f["idx"].sort(1).values
        assert bool((srt[:, 1:] == srt[:, :-1]).any(1).all())                 # every neighbourhood padded
    _all_modes(f, schedule)


@pytest.mark.parametrize("schedule", [WARP, CTA], ids=["warp", "cta"])
@pytest.mark.parametrize("K", [1, 2, 7, 8, 9, 33, 64])
@pytest.mark.parametrize("c,n", [(32, 1000), (512, 150)])
def test_k_edges(c, n, K, schedule):
    _all_modes(_case(c, K, n), schedule)


@pytest.mark.parametrize("schedule", [WARP, CTA], ids=["warp", "cta"])
@pytest.mark.parametrize("n", [1, 7, 8, 9, "8sm+1", "32sm+1"])
@pytest.mark.parametrize("c,K", [(32, 16), (512, 24)])
def test_n_edges(c, K, n, schedule):
    """n below a warp's 8 queries per CTA, a CTA's second query (grid 8 SMs) and a warp's second (grid 4 SMs x 8 warps)"""
    n = {"8sm+1": 8 * _sms() + 1, "32sm+1": 32 * _sms() + 1}.get(n, n)
    _all_modes(_case(c, K, n), schedule)


@pytest.mark.parametrize("c,K", [(32, 16), (512, 24)])
def test_default_threshold_on_both_sides(c, K):
    """1023 queries run one CTA each, 1024 one warp each: the default launch equals the forced schedule bit for bit"""
    for n, forced in ((1023, CTA), (1024, WARP)):
        f = _case(c, K, n)
        _all_modes(f, DEFAULT)
        with _threshold(DEFAULT):
            dflt = _launch(f, [2, 2, 2], update=0)["out"]
        with _threshold(forced):
            same = _launch(f, [2, 2, 2], update=0)["out"]
        with _threshold(WARP if forced == CTA else CTA):
            other = _launch(f, [2, 2, 2], update=0)["out"]
        assert torch.equal(dflt, same) and not torch.equal(dflt, other), n


@pytest.mark.parametrize("schedule", [WARP, CTA], ids=["warp", "cta"])
@pytest.mark.parametrize("kind", ["plain", "saturated", "uniform"])
@pytest.mark.parametrize("c,K,n,crops", [(32, 36, 6000, 1), (128, 24, 3072, 16), (512, 24, 192, 16)])
def test_softmax_cases(c, K, n, crops, kind, schedule):
    """near one-hot logits (x 100) and an exactly uniform softmax (b_w = 0), next to unit-scale data"""
    _all_modes(_case(c, K, n, crops, kind), schedule)


@pytest.mark.parametrize("schedule", [WARP, CTA], ids=["warp", "cta"])
def test_running_statistics_left_alone(schedule):
    """update_running = 0 and a BatchNorm with a null running pointer leave the buffers bitwise unchanged (the others update)"""
    f = _case(64, 24, 700)
    with _threshold(schedule):
        _check(f, [1, 1, 1], _launch(f, [1, 1, 1], update=0), update=0)
        for null in (("a_rmean",), ("b_rvar",), ("p_rmean", "p_rvar")):
            _check(f, [1, 1, 1], _launch(f, [1, 1, 1], null=null), null=null)


def test_refusals_launch_nothing():
    f = _case(32, 16, 200)
    for k in (0, 65):
        _launch(dict(f, K=k), [1, 1, 1], expect_ok=False)
    for c in (48, 1024):
        _launch(dict(f, c=c), [1, 1, 1], expect_ok=False)
    for k in REQUIRED:
        _launch(f, [1, 1, 1], null=(k,), expect_ok=False)
    got = _launch(dict(f, n=0), [1, 1, 1])
    assert got["launches"] == 0
    assert all(torch.equal(got["running"][k], got["before_running"][k]) for k in _RUNNING)


def test_report_worst_ratio():
    """runs last in the file: the worst err / bound of each check, which must stay at or below 1"""
    print("pt_layer worst err / bound:", {k: f"{v:.3g}" for k, v in sorted(WORST.items())})
    assert all(v <= 1.0 for v in WORST.values())
