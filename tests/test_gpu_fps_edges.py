"""FPS at every compiled kernel and at every edge of its dispatch, one tgn_furthestsampling launch at a time.

Each case checks idx AND the final running minima (tmp) bitwise against the C restatement of the reference kernel (and
against the reference kernel itself when oracle/_ref is built), with idx and tmp allocated inside sentinel guards that must
survive the launch, and records the launch under torch.profiler to assert which kernels ran: the case tables below name every
instantiation of the bucket, resident and streaming kernels (tests/test_cpu_fps_cases.py checks that against the sources), so
a case list that drifts away from the dispatch fails here rather than quietly testing another kernel."""
import functools
import re
from types import SimpleNamespace

import numpy as np
import pytest
import torch
from torch.profiler import ProfilerActivity, profile, schedule

from oracle import oracle, ref_cuda
from toothgroupnetwork_b200 import _lib as L
from toothgroupnetwork_b200 import clouds

from test_gpu_pointops import FPS_CASES, FPS_MODES, _pack, i32

pytestmark = pytest.mark.gpu
needs_ref = pytest.mark.skipif(not ref_cuda.available(), reason="oracle/_ref not built")
AGAINST = ["oracle", pytest.param("reference", marks=needs_ref)]

# fps_bucket.cu: points per bucket, largest cloud sorted in shared memory, bucket-table capacity
KBP, SMEM_SORT_MAX_N, MAX_BUCKETS = 64, 26624, 3600
MAX_POINTS = MAX_BUCKETS * KBP           # fps_bucket_max_points(): 230 400
# fps.cu kConfigs, in pick_config's order: (T, SLOTS, CS, G)
RESIDENT_CONFIGS = [
    (128, 4, 1, 1), (256, 4, 1, 1), (512, 4, 1, 1), (1024, 4, 1, 1), (1024, 8, 1, 1),
    (512, 4, 2, 1), (512, 8, 2, 1), (512, 12, 2, 1), (512, 16, 2, 1), (512, 24, 2, 1),
    (512, 4, 4, 1), (512, 8, 4, 1), (512, 12, 4, 1), (512, 16, 4, 1), (512, 24, 4, 1),
    (512, 4, 8, 1), (512, 8, 8, 1), (512, 12, 8, 1), (512, 16, 8, 1), (512, 24, 8, 1),
    (512, 4, 1, 2),
    (512, 4, 2, 2), (512, 8, 2, 2), (512, 12, 2, 2),
    (512, 4, 4, 2), (512, 8, 4, 2), (512, 12, 4, 2),
    (512, 8, 8, 2), (512, 12, 8, 2),
]
RESIDENT_MAX = max(t * s * cs for t, s, cs, _ in RESIDENT_CONFIGS)


def K3(mt, bpl):
    return f"fps_bucket_kernel3<{mt}, {bpl}>"


def K2(mt):
    return f"fps_bucket_kernel2<{mt}>"


def K1(mt):
    return f"fps_bucket_kernel<{mt}>"


def SORT(n_max):
    return "fps_bucket_sort_kernel<true>" if n_max <= SMEM_SORT_MAX_N else "fps_bucket_sort_kernel<false>"


def RES(c):
    return "fps_resident_kernel<%d, %d, %d, %d>" % tuple(c)


STREAM = "fps_stream_kernel"


# ------------------------------------------------------------------------------------------------------------ case tables
# A case: (id, clouds as (kind, n, seed, m), mode, kernels that must run -- None: the call must be refused).

# Every launch_main3<32 W, BPL> of fps_bucket_launch as (W, BPL, first n, last n) under mode -(80 + W): bpl = ceil(nbmax / 32 W)
# with nbmax = ceil(n / 64); 16 warps take bpl 3 on the 4-bucket kernel and 5 on the 6-bucket kernel.
V3_RANGES = [
    (32, 1, 1, 65536),
    (16, 1, 1, 32768), (16, 2, 32769, 65536), (16, 4, 65537, 131072), (16, 6, 131073, 196608), (16, 8, 196609, MAX_POINTS),
    (8, 1, 1, 16384), (8, 2, 16385, 32768), (8, 4, 32769, 65536),
    (4, 2, 1, 16384), (4, 3, 16385, 24576), (4, 4, 24577, 32768),
]
# More buckets per lane than a v3 shape holds: fps_bucket_kernel2 of the same width, (W, first n, last n).  Sixteen warps have
# no such fallback: kMaxBuckets = 3 600 caps bpl at 8, which launch_main3<512, 8> holds.
V3_FALLBACKS = [(4, 32769, MAX_POINTS), (8, 65537, MAX_POINTS), (32, 65537, MAX_POINTS)]
V2_WARPS = [2, 4, 8, 16, 32]          # mode -(40 + W): fps_bucket_kernel2<32 W>, any n up to MAX_POINTS
V1_WARPS = [1, 2, 4, 8, 16]           # mode -(10 + W): fps_bucket_kernel<32 W>
KINDS = ["arch", "cube", "dups"]


def _m(n):
    return min(n, 200 if n > 100000 else 400)


def _two_ends(first, last, alt=0):
    """The top of a range (the last lane's last bucket full) and an n = 1 (mod 64) inside it (one point in the last bucket): the
    first n of the range when it has a lower edge, otherwise just below the top or, for the full-range kernels, just past
    either side of the sort crossover."""
    if first > 1:
        return [last, first]
    if last == MAX_POINTS:
        return [last, SMEM_SORT_MAX_N + 1 if alt % 2 else SMEM_SORT_MAX_N - 63]
    return [last, last - 63]


def instantiation_cases():
    cases, i = [], 0
    for w, bpl, first, last in V3_RANGES:
        for n in _two_ends(first, last):
            cases.append((f"v3_{32 * w}x{bpl}_n{n}", [(KINDS[i % 3], n, 100 + i, _m(n))], -(80 + w), (SORT(n), K3(32 * w, bpl))))
            i += 1
    for w, first, last in V3_FALLBACKS:
        for n in _two_ends(first, last):
            cases.append((f"v3_fallback_{32 * w}_n{n}", [(KINDS[i % 3], n, 100 + i, _m(n))], -(80 + w), (SORT(n), K2(32 * w))))
            i += 1
    for w in V2_WARPS:
        for n in _two_ends(1, MAX_POINTS, i):
            cases.append((f"v2_{32 * w}_n{n}", [(KINDS[i % 3], n, 100 + i, _m(n))], -(40 + w), (SORT(n), K2(32 * w))))
            i += 1
    for w in V1_WARPS:
        for n in _two_ends(1, MAX_POINTS, i):
            cases.append((f"v1_{32 * w}_n{n}", [(KINDS[i % 3], n, 100 + i, _m(n))], -(10 + w), (SORT(n), K1(32 * w))))
            i += 1
    # mode -2 / -3: the bucket kernel below the auto crossover, shape by batch size
    cases.append(("mode-2_n2000", [("arch", 2000, 150, 500)], -2, (SORT(2000), K3(512, 1))))
    cases.append(("mode-3_n3000", [("dups", 3000, 151, 500)], -3, (SORT(3000), K2(512))))
    return cases


# The global-memory sort with tiny clouds in the batch: one point, a single partial bucket, exactly one bucket, one point past
# it; m = 0 (a repeated new_offset), m = n and m > n.
RAGGED_GLOBAL = [("arch", 40000, 200, 300), ("cube", 1, 201, 5), ("cube", 2, 202, 0), ("cube", 63, 203, 63), ("dups", 64, 204, 64),
                 ("cube", 65, 205, 30), ("arch", 700, 206, 100)]
SORT_CASES = [
    ("sort_smem_last", [("arch", SMEM_SORT_MAX_N, 210, 400)], 0, (SORT(SMEM_SORT_MAX_N), K3(512, 1))),
    ("sort_global_first", [("arch", SMEM_SORT_MAX_N + 1, 211, 400)], 0, (SORT(SMEM_SORT_MAX_N + 1), K3(512, 1))),
    ("ragged_global_auto", RAGGED_GLOBAL, 0, (SORT(40000), K3(512, 2))),
    ("ragged_global_v1_128", RAGGED_GLOBAL, -14, (SORT(40000), K1(128))),
    ("ragged_global_v2_128", RAGGED_GLOBAL, -44, (SORT(40000), K2(128))),
    ("ragged_global_v3_1024", RAGGED_GLOBAL, -112, (SORT(40000), K3(1024, 1))),
    ("ragged_global_v3_128_fallback", RAGGED_GLOBAL, -84, (SORT(40000), K2(128))),
]

# Auto mode on both sides of each crossover.  The widening cases need at least 8 and 32 SMs.
CROSSOVER_CASES = [
    ("auto_4096_resident_cs4", [("arch", 4096, 220, 512)], 0, (RES((512, 4, 4, 1)),)),
    ("auto_4097_bucket", [("arch", 4097, 221, 512)], 0, (SORT(4097), K3(512, 1))),
    ("auto_3072x16_resident_cs2", [("arch", 3072, 230 + i, 256) for i in range(16)], 0, (RES((512, 4, 2, 1)),)),
    ("auto_230400_bucket", [("arch", MAX_POINTS, 222, 200)], 0, (SORT(MAX_POINTS), K3(512, 8))),
    ("auto_230401_stream", [("arch", MAX_POINTS + 1, 223, 200)], 0, (STREAM,)),
]


def _ties_batch(n_max, seed):
    """a duplicated-vertex cloud with more samples than unique points, the n_max cloud, an all-identical cloud"""
    nd = (n_max - 101) // 2 * 2
    return [("dups", nd, seed, nd // 2 + 10), ("cube", n_max, seed + 1, n_max // 4), ("same", n_max // 3, seed + 2, 20),
            ("dups", 40, seed + 3, 60)]


# The reference's tie order depends on BS = opt_n_threads(n_max); ties in clouds smaller than n_max.
TIE_CASES = [(f"ties_resident_{n}", _ties_batch(n, 240 + n), 0, (RES(c),))
             for n, c in [(511, (256, 4, 1, 1)), (512, (512, 4, 1, 1)), (513, (512, 4, 1, 1)), (1023, (512, 4, 1, 1)),
                          (1024, (1024, 4, 1, 1))]]
TIES_BUCKET = [("dups", 20000, 250, 2000), ("arch", 30000, 251, 500), ("same", 3000, 252, 50), ("dups", 9001, 253, 5000)]
TIES_SMEM = [("arch", 20000, 254, 400), ("dups", 12000, 255, 6100), ("same", 700, 256, 30)]
ALL_TIES = [("dups", 10000, 257, 6000)]       # 5 000 unique points twice: from sample 5 000 on, every maximum is a tie at t = 0
for _mode, _main in [(0, K3(512, 1)), (-14, K1(128)), (-44, K2(128))]:
    TIE_CASES += [(f"ties_bucket_global_{_mode}", TIES_BUCKET, _mode, (SORT(30000), _main)),
                  (f"ties_bucket_smem_{_mode}", TIES_SMEM, _mode, (SORT(20000), _main)),
                  (f"all_ties_{_mode}", ALL_TIES, _mode, (SORT(10000), _main))]

# The bucket boxes are inflated by 4e-6 max|coord|: far from the origin, a tiny extent, two degenerate axes.
PRUNING_CASES = []
for _mode, _main in [(0, K3(512, 1)), (-14, K1(128)), (-44, K2(128))]:
    PRUNING_CASES += [(f"{k}_{_mode}", [(k, n, 260 + j, 512)], _mode, (SORT(n), _main))
                      for j, (k, n) in enumerate([("far100", 24000), ("far1000", 24000), ("tiny", 24000), ("line", 30000)])]


def _pick_config(n_max, cs, g):
    """fps.cu pick_config: the first kConfigs entry of cluster size cs and g clouds in flight that holds n_max points"""
    bs = oracle.opt_n_threads(n_max)
    for c in RESIDENT_CONFIGS:
        t, s, ccs, cg = c
        if ccs == cs and cg == g and t * ccs >= bs and (t * ccs // bs) * s >= -(-n_max // bs):
            return c
    return None


@functools.lru_cache(maxsize=None)
def resident_tops():
    """{kConfigs entry: the largest n_max that pick_config gives it under its own (CS, G)}.  Within a run of n of one block size
    the entries of a (CS, G) group hold growing prefixes, so an entry's last n in a run is its capacity or the run's end."""
    runs = []                                   # [first n, last n, BS]
    for n in range(1, RESIDENT_MAX + 2):
        bs = oracle.opt_n_threads(n)
        if runs and runs[-1][2] == bs:
            runs[-1][1] = n
        else:
            runs.append([n, n, bs])
    tops = {}
    for c in RESIDENT_CONFIGS:
        t, s, cs, g = c
        for first, last, bs in runs:
            if t * cs < bs:
                continue
            n = min(last, (t * cs // bs) * s * bs)
            if n >= first and _pick_config(n, cs, g) == c:
                tops[c] = max(tops.get(c, 0), n)
    return tops


def resident_cases():
    """Every kConfigs entry under its forced mode 100 G + CS at the largest n_max it takes (every slot of the last residue
    full) and one past it, which moves to the next entry or is refused.  Two clouds in flight: three clouds, one pair and
    one alone, the middle one smaller."""
    cases = []
    for i, c in enumerate(RESIDENT_CONFIGS):
        t, s, cs, g = c
        mode = 100 * g + cs if g > 1 else cs
        top = resident_tops()[c]
        for n in (top, top + 1):
            nxt = _pick_config(n, cs, g)
            spec = [(KINDS[i % 3], n, 300 + i, min(n, 256))]
            if g > 1:
                spec += [("dups", max(2, n // 3), 400 + i, min(n // 3, 200)), ("arch", n, 500 + i, min(n, 256))]
            cases.append((f"resident_{t}x{s}_cs{cs}_g{g}_n{n}", spec, mode, None if nxt is None else (RES(nxt),)))
    return cases


ALL_CASES = instantiation_cases() + SORT_CASES + CROSSOVER_CASES + TIE_CASES + PRUNING_CASES + resident_cases()


def asserted_kernels():
    """every kernel name some case of this file requires to run"""
    names = {k for case in ALL_CASES if case[3] for k in case[3]}
    for n, _, _, main in BATCH_CASES:
        names |= {SORT(n), main}
    return names


# ------------------------------------------------------------------------------------------------------------ helpers
@functools.lru_cache(maxsize=64)
def _cloud(kind, n, seed):
    if kind == "arch":
        return clouds.dental_arch(n, seed)[0]
    if kind == "cube":
        return clouds.cube(n, seed)
    if kind == "dups":
        return clouds.with_duplicates(clouds.dental_arch((n + 1) // 2, seed)[0], seed)[:n].contiguous()
    if kind == "same":
        return torch.tensor([0.25, -0.5, 0.125]).expand(n, 3).contiguous()
    unit = clouds.cube(n, seed) * 0.5
    if kind == "far100":
        return unit + torch.tensor([100.0, -100.0, 100.0])
    if kind == "far1000":
        return unit + 1000.0
    if kind == "tiny":
        return unit * 1e-4
    if kind == "line":
        return clouds.cube(n, seed) * torch.tensor([1.0, 0.0, 0.0]) + torch.tensor([0.0, 0.3, -0.7])
    raise ValueError(kind)


def _batch(spec):
    xyz, offset, new_offset = _pack([_cloud(k, n, s) for k, n, s, _ in spec], [m for *_, m in spec])
    return xyz, offset, new_offset


GUARD = 512
IDX_SENTINEL = 0x7A5A5A5A                     # no index
TMP_SENTINEL = 0x7FA5A5A5                     # a NaN payload: no running minimum has these bits
TMP_INIT = int(np.float32(1e10).view(np.int32))
_KERNEL = re.compile(r"fps_\w+(<[^<>()]*>)?")


def _record(fn):
    """fn() under torch.profiler -> the names of the fps kernels it launched"""
    with profile(activities=[ProfilerActivity.CUDA], schedule=schedule(wait=0, warmup=1, active=1, repeat=1)) as prof:
        torch.ones(1, device="cuda").add_(1)
        torch.cuda.synchronize()
        prof.step()
        fn()
        torch.cuda.synchronize()
        prof.step()
    return {_KERNEL.search(e.key).group(0) for e in prof.key_averages() if _KERNEL.search(e.key)}


# torch.profiler's kernel records of one short session now and then come back incomplete (a kernel of the launch missing,
# never a kernel that did not run).  When a recorded launch lacks an expected kernel it is launched again on fresh buffers
# under a new session, up to this many times in all, and the kernels of all sessions are compared; an unexpected kernel in
# any session still fails the case.
RECORD_ATTEMPTS = 5


def _guarded(n, fill, sentinel):
    buf = torch.full((n + 2 * GUARD,), sentinel, dtype=torch.int32, device="cuda")
    buf[GUARD:GUARD + n] = fill
    return buf


def _run(xyz, offset, new_offset, mode, with_tmp=True, n_max=None, record=True, expect=()):
    """One tgn_furthestsampling launch on the current stream with idx and tmp inside sentinel guards.  Returns idx, the final
    tmp (as int32 bits), the fps kernels the profiler saw, the library's launch count delta and the error of a refused call;
    asserts the guards."""
    sizes = np.diff(np.concatenate([[0], offset]))
    n_max = int(sizes.max()) if n_max is None else n_max
    x, o, no = xyz.cuda().contiguous(), i32(offset), i32(new_offset)
    m, n = int(new_offset[-1]), xyz.shape[0]
    ibuf = _guarded(m, 0, IDX_SENTINEL)
    tbuf = _guarded(n, TMP_INIT, TMP_SENTINEL) if with_tmp else None
    torch.cuda.synchronize()
    before, err = L.launch_count(), []

    def call(ib, tb):
        try:
            L.call("tgn_furthestsampling", len(offset), int(n_max), L.ptr(x), L.ptr(o), L.ptr(no),
                   tb[GUARD:].data_ptr() if with_tmp else None, ib[GUARD:].data_ptr(), int(mode), L.stream_ptr())
        except L.TgnError as e:
            err.append(e)
        torch.cuda.synchronize()

    names = _record(lambda: call(ibuf, tbuf)) if record else call(ibuf, tbuf)
    launches = L.launch_count() - before
    for _ in range(RECORD_ATTEMPTS - 1):
        if not record or set(expect) <= names:
            break
        names |= _record(lambda: call(_guarded(m, 0, IDX_SENTINEL), _guarded(n, TMP_INIT, TMP_SENTINEL) if with_tmp else None))
    ib = ibuf.cpu().numpy()
    assert (ib[:GUARD] == IDX_SENTINEL).all() and (ib[GUARD + m:] == IDX_SENTINEL).all(), "idx guard overwritten"
    tb = None
    if with_tmp:
        tb = tbuf.cpu().numpy()
        assert (tb[:GUARD] == TMP_SENTINEL).all() and (tb[GUARD + n:] == TMP_SENTINEL).all(), "tmp guard overwritten"
        tb = tb[GUARD:GUARD + n]
    assert torch.equal(x.cpu(), xyz), "xyz written"
    return SimpleNamespace(idx=ib[GUARD:GUARD + m], tmp=tb, names=names, launches=launches, err=err[0] if err else None)


def _want(xyz, offset, new_offset, against):
    """(idx, tmp bits, idx slots to compare) of the oracle or of the reference kernel.  The reference kernel writes
    idx[start_m] = start_n for a cloud with m = 0 as well, racing with the next cloud's first sample: that slot is not compared."""
    m = int(new_offset[-1])
    keep = np.ones(m, bool)
    if against == "oracle":
        idx, tmp = oracle.furthestsampling(xyz.numpy(), offset, new_offset, return_tmp=True)
        return idx, tmp.view(np.int32), keep
    sizes_m = np.diff(np.concatenate([[0], new_offset]))
    assert sizes_m[-1] > 0, "the reference kernel writes past idx for a last cloud with m = 0"
    for c in np.nonzero(sizes_m == 0)[0]:
        keep[int(new_offset[c])] = False
    n_max = int(np.diff(np.concatenate([[0], offset])).max())
    idx, tmp = ref_cuda.furthestsampling(xyz.cuda(), i32(offset), i32(new_offset), n_max, m)
    return idx.cpu().numpy(), tmp.cpu().numpy().view(np.int32), keep


def _assert_refused(run, message):
    assert run.err is not None and message in str(run.err), run.err
    assert run.launches == 0 and not run.names, (run.launches, run.names)
    assert (run.idx == 0).all(), "idx written by a refused call"
    assert run.tmp is None or (run.tmp == TMP_INIT).all(), "tmp written by a refused call"


# ------------------------------------------------------------------------------------------------------------ tests
@pytest.mark.parametrize("against", AGAINST)
@pytest.mark.parametrize("case", ALL_CASES, ids=[c[0] for c in ALL_CASES])
def test_fps_edge_case(case, against):
    name, spec, mode, kernels = case
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    if name.startswith("auto_3072x16") and sms < 32 or name.startswith("auto_4096") and sms < 8:
        pytest.skip("the cluster widening of this case needs more SMs")
    xyz, offset, new_offset = _batch(spec)
    run = _run(xyz, offset, new_offset, mode, expect=kernels or ())
    if kernels is None:
        _assert_refused(run, f"no resident kernel of shape {mode}")
        return
    assert run.err is None, run.err
    assert run.names == set(kernels), run.names
    want_idx, want_tmp, keep = _want(xyz, offset, new_offset, against)
    assert np.array_equal(run.idx[keep], want_idx[keep])
    assert np.array_equal(run.tmp, want_tmp)


# Auto mode at the batch-size shape switch, (n, k, forced mode it must equal, main kernel, clouds): b = (sms, sms + 1, 2 sms,
# 2 sms + 1, 4 sms, 4 sms + 1)[k].  24 000 points: the register-table kernel up to 4 clouds per SM, then 4 warps per cloud;
# 40 000: 8 clouds per SM do not fit (fits(8) fails), so 8 warps; 70 000: nbmax > 1 024 keeps the register tables to one cloud
# per SM, and neither 4 nor 8 clouds per SM fit, so 16 warps.
BATCH_CASES = []
for _k in range(6):
    BATCH_CASES.append((24000, _k, -96 if _k < 5 else -14, K3(512, 1) if _k < 5 else K1(128)))
    BATCH_CASES.append((40000, _k, -96 if _k < 5 else -18, K3(512, 2) if _k < 5 else K1(256)))
    BATCH_CASES.append((70000, _k, -96 if _k < 1 else -26, K3(512, 4) if _k < 1 else K1(512)))


@pytest.mark.parametrize("n,k,forced,main", BATCH_CASES, ids=[f"n{c[0]}_b{c[1]}" for c in BATCH_CASES])
def test_auto_batch_shape(n, k, forced, main):
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    b = [sms, sms + 1, 2 * sms, 2 * sms + 1, 4 * sms, 4 * sms + 1][k]
    m = 128
    base = [clouds.dental_arch(n, 600 + s)[0] for s in range(6)]
    base += [clouds.with_duplicates(clouds.dental_arch(n // 2, 610 + s)[0], 610 + s) for s in range(2)]
    cl = [base[j % len(base)] for j in range(b)]
    xyz = torch.cat(cl, 0)
    offset = (np.arange(1, b + 1) * n).astype(np.int32)
    new_offset = (np.arange(1, b + 1) * m).astype(np.int32)
    auto = _run(xyz, offset, new_offset, 0, expect={SORT(n), main})
    assert auto.err is None, auto.err
    assert auto.names == {SORT(n), main}, auto.names
    ref = _run(xyz, offset, new_offset, forced, record=False)
    assert ref.err is None, ref.err
    assert np.array_equal(auto.idx, ref.idx) and np.array_equal(auto.tmp, ref.tmp)
    rng = np.random.default_rng(k)
    for j in sorted(rng.choice(b, 4, replace=False).tolist()) + [6, 7]:
        w_idx, w_tmp = oracle.furthestsampling(cl[j].numpy(), np.array([n], np.int32), np.array([m], np.int32), return_tmp=True)
        assert np.array_equal(auto.idx[j * m:(j + 1) * m] - j * n, w_idx), f"cloud {j}"
        assert np.array_equal(auto.tmp[j * n:(j + 1) * n], w_tmp.view(np.int32)), f"cloud {j}"


@pytest.mark.parametrize("n", [RESIDENT_MAX, RESIDENT_MAX + 1])
def test_auto_tmp_crossover_through_fps_packed(n):
    """pointops.fps_packed passes a tmp buffer from n_max > 98 304 on; the bucket kernel runs either way."""
    from toothgroupnetwork_b200 import pointops
    assert pointops._RESIDENT_FPS_MAX_POINTS == RESIDENT_MAX
    xyz = _cloud("arch", n, 700)
    x, o, no, got = xyz.cuda(), i32([n]), i32([256]), []
    names = set()
    for _ in range(RECORD_ATTEMPTS):
        names |= _record(lambda: got.append(pointops.fps_packed(x, o, no, n, 256, 0)))
        if {SORT(n), K3(512, 4)} <= names:
            break
    got = got[0]
    assert names == {SORT(n), K3(512, 4)}, names
    assert np.array_equal(got.cpu().numpy(), oracle.furthestsampling(xyz.numpy(), [n], [256]))


_ORACLE = {}


@pytest.mark.parametrize("name,build,ms", FPS_CASES, ids=[c[0] for c in FPS_CASES])
@pytest.mark.parametrize("mode", FPS_MODES)
def test_tmp_for_every_mode(name, build, ms, mode):
    """The final running minima of every mode bitwise; then without tmp (every mode but the streaming kernel's): the same idx,
    nothing written."""
    xyz, offset, new_offset = _pack(build(), ms)
    run = _run(xyz, offset, new_offset, mode, record=False)
    if run.err is not None and mode > 0 and "no resident kernel of shape" in str(run.err):
        pytest.skip("cluster size not applicable to this cloud size")
    assert run.err is None, run.err
    if name not in _ORACLE:
        _ORACLE[name] = _want(xyz, offset, new_offset, "oracle")[:2]
    want_idx, want_tmp = _ORACLE[name]
    assert np.array_equal(run.idx, want_idx)
    assert np.array_equal(run.tmp, want_tmp)
    if mode != -1:
        bare = _run(xyz, offset, new_offset, mode, with_tmp=False, record=False)
        assert bare.err is None, bare.err
        assert np.array_equal(bare.idx, want_idx)


UNKNOWN = "unknown mode"
REFUSALS = ([(md, 24000, True, UNKNOWN) for md in [-4, -10, -27, -40, -113, -200] + list(range(-80, -72))]
            + [(-13, 24000, True, "no shape of 3 warps"), (-41, 24000, True, "no shape of 1 warps"),
               (-43, 24000, True, "no shape of 3 warps"), (-81, 24000, True, "no shape of 1 warps"),
               (-82, 24000, True, "no shape of 2 warps"), (-83, 24000, True, "no shape of 3 warps"),
               (3, 24000, True, "no resident kernel of shape 3"), (100, 24000, True, "no resident kernel of shape 100"),
               (301, 24000, True, "no resident kernel of shape 301"), (8, RESIDENT_MAX + 1, True, "no resident kernel of shape 8"),
               (-1, 24000, False, "needs a tmp buffer"), (0, MAX_POINTS + 1, False, "no tmp buffer was given")]
            + [(md, MAX_POINTS + 1, True, "exceeds the bucket kernel")
               for md in (-2, -3, -11, -12, -14, -18, -26, -42, -44, -48, -56, -72, -84, -88, -96, -112)])


@pytest.mark.parametrize("mode,n,with_tmp,message", REFUSALS, ids=[f"mode{r[0]}_n{r[1]}{'' if r[2] else '_no_tmp'}" for r in REFUSALS])
def test_refusal_launches_nothing(mode, n, with_tmp, message):
    """A refused call returns an error with the reason, launches nothing and leaves idx and tmp as they were."""
    xyz, offset, new_offset = _batch([("arch", n, 800, 64), ("cube", 500, 801, 64)])
    _assert_refused(_run(xyz, offset, new_offset, mode, with_tmp=with_tmp), message)
