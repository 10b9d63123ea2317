"""The FPS edge-case tables of test_gpu_fps_edges.py against the CUDA sources they test, without a GPU: every kernel
instantiation the dispatch can launch has a case whose profiler assertion names it, the bucket-kernel cases sit where the
dispatch's if-chain sends them, and the constants the ranges are computed from are the sources' own."""
import os
import re

import test_gpu_fps_edges as E
from toothgroupnetwork_b200 import pointops

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "toothgroupnetwork_b200", "csrc")


def _src(name):
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


def _constant(src, name):
    return int(re.search(rf"constexpr int {name} = (\d+);", src).group(1))


def _v3_chain(src):
    """fps_bucket_launch's v3 if-chain in order: (warps, largest bpl, MT, BPL)"""
    return [tuple(map(int, g)) for g in re.findall(
        r"warps == (\d+) && bpl <= (\d+)\) rc = launch_main3<(\d+), (\d+)>\(", src)]


def _instantiations():
    bucket, fps = _src("fps_bucket.cu"), _src("fps.cu")
    names = {E.K3(int(a), int(b)) for a, b in re.findall(r"launch_main3<(\d+), (\d+)>\(", bucket)}
    names |= {E.K2(int(a)) for a in re.findall(r"launch_main2<(\d+)>\(", bucket)}
    names |= {E.K1(int(a)) for a in re.findall(r"launch_main<(\d+)>\(", bucket)}
    names |= {f"fps_bucket_sort_kernel<{v}>" for v in re.findall(r"fps_bucket_sort_kernel<(true|false)><<<", bucket)}
    names |= {E.RES(tuple(map(int, g))) for g in re.findall(r"TGN_FPS_CASE\((\d+), (\d+), (\d+), (\d+)\)", fps)}
    if re.search(r"fps_stream_kernel<<<", fps):
        names.add(E.STREAM)
    return names


def _k_configs():
    fps = _src("fps.cu")
    table = re.search(r"kConfigs\[\] = \{(.*?)\n\};", fps, re.S).group(1)
    return [tuple(map(int, g)) for g in re.findall(r"\{(\d+), (\d+), (\d+), (\d+)\}", table)]


def test_every_instantiation_has_a_case():
    names = _instantiations()
    assert len([k for k in names if k.startswith("fps_bucket_kernel3<")]) == 12
    assert len([k for k in names if k.startswith("fps_resident_kernel<")]) == len(_k_configs())
    missing = names - E.asserted_kernels()
    assert not missing, f"kernels without a case in test_gpu_fps_edges.py: {sorted(missing)}"
    unknown = E.asserted_kernels() - names
    assert not unknown, f"cases expect kernels the sources do not launch: {sorted(unknown)}"


def test_constants_match_the_sources():
    bucket = _src("fps_bucket.cu")
    assert _constant(bucket, "kBP") == E.KBP
    assert _constant(bucket, "kSmemSortMaxN") == E.SMEM_SORT_MAX_N
    assert _constant(bucket, "kMaxBuckets") == E.MAX_BUCKETS
    assert _k_configs() == E.RESIDENT_CONFIGS
    dispatched = [tuple(map(int, g)) for g in re.findall(r"TGN_FPS_CASE\((\d+), (\d+), (\d+), (\d+)\)", _src("fps.cu"))]
    assert sorted(dispatched) == sorted(E.RESIDENT_CONFIGS)
    assert pointops._RESIDENT_FPS_MAX_POINTS == max(t * s * cs for t, s, cs, _ in _k_configs()) == E.RESIDENT_MAX


def test_bucket_ranges_follow_the_dispatch():
    """Restate fps_bucket_launch's choice for every forced bucket case: the v3 if-chain parsed from the source, its fallback to
    fps_bucket_kernel2 of the same width, the sort variant by kSmemSortMaxN.  Each instantiation has a case at the top of its
    range and one with a single point in the last bucket."""
    chain = _v3_chain(_src("fps_bucket.cu"))
    assert len(chain) == 12
    for w, bpl, first, last in E.V3_RANGES:
        assert (w, bpl) in [(c[0], c[3]) for c in chain]
        assert last == min(E.MAX_POINTS, 2048 * w * bpl)
    tops, ones = set(), set()
    for name, spec, mode, kernels in E.instantiation_cases():
        if mode in (-2, -3):
            continue
        n = max(c[1] for c in spec)
        nbmax = -(-n // E.KBP)
        w = -mode - (10 if mode >= -26 else 40 if mode >= -72 else 80)
        if mode >= -26:
            main = E.K1(32 * w)
        elif mode >= -72:
            main = E.K2(32 * w)
        else:
            bpl = -(-nbmax // (32 * w))
            hit = [c for c in chain if c[0] == w and bpl <= c[1]]
            main = E.K3(hit[0][2], hit[0][3]) if hit else E.K2(32 * w)
        assert kernels == (E.SORT(n), main), name
        assert n <= E.MAX_BUCKETS * E.KBP
        (ones if n % E.KBP == 1 else tops).add(main)
    assert {k for k in E.asserted_kernels() if k.startswith("fps_bucket_kernel")} <= tops & ones


def test_every_resident_config_is_reachable_at_its_capacity():
    """pick_config gives every kConfigs entry some n_max under its forced mode, and one point past the largest moves to the
    next entry of the same (CS, G) or is refused."""
    tops = E.resident_tops()
    for i, c in enumerate(E.RESIDENT_CONFIGS):
        assert c in tops, f"{c} is never picked"
        t, s, cs, g = c
        assert tops[c] <= t * cs * s
        later = [d for d in E.RESIDENT_CONFIGS[i + 1:] if d[2:] == c[2:]]
        assert E._pick_config(tops[c] + 1, cs, g) == (later[0] if later else None), c
    assert tops[(128, 4, 1, 1)] == 255
    assert max(tops.values()) == E.RESIDENT_MAX


def test_refusals_cover_the_unknown_modes():
    """fps_dispatch refuses negative modes outside 0..-3, -11..-26, -41..-72 and -81..-112; the GPU refusal cases sample
    every gap of that set."""
    assert re.search(r"mode >= -3 \|\| \(mode <= -11 && mode >= -26\) \|\| \(mode <= -41 && mode >= -72\) \|\| "
                     r"\(mode <= -81 && mode >= -112\)", _src("fps.cu"))
    sampled = {r[0] for r in E.REFUSALS if r[3] == E.UNKNOWN}
    for lo, hi in [(-10, -4), (-40, -27), (-80, -73), (-200, -113)]:
        assert sampled & set(range(lo, hi + 1)), (lo, hi)
