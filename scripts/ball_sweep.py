"""Ball query: per-kernel times at the bench shape, then tile vs grid vs auto over radii / sizes (ms per call).

    python scripts/ball_sweep.py [B]

Prints the card name and power limit first: every time below belongs to them.
"""
import re
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, ".")
from toothgroupnetwork_b200 import clouds, pointnet2_utils as pn2


def timeit(f, n=5):
    for _ in range(2): f()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n): f()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def kernel_ms(f, n=10):
    """Mean device time per call of each kernel f launches, by kernel name (torch.profiler, CUDA activity)."""
    f(); torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(n): f()
        torch.cuda.synchronize()
    out = {}
    for ev in prof.key_averages():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        m = re.search(r"(\w+_kernel)\b", ev.key)
        name = m.group(1) if m else ev.key[:40]
        out[name] = out.get(name, 0.0) + ev.device_time_total / 1e3 / n
    return out


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def bench_shape(B=1056, N=24000, S=1024, r=0.1, K=32):
    """The bench's batch: 8 distinct 24k-point arches tiled, queries from FPS, as bench.py builds them."""
    base = [clouds.arch_features(N, clouds.cloud_seed(0, j))[0][:3].t().contiguous() for j in range(8)]
    xyz = torch.stack([base[j % 8] for j in range(B)]).cuda().contiguous()
    fps = pn2._fps_batched(xyz, S)
    new = pn2._take_rows(xyz.view(-1, 3), fps).view(B, S, 3)
    print(f"bench shape B={B} N={N} S={S} r={r} K={K}", flush=True)
    for name, path in (("tile", pn2.BALL_TILE), ("grid", pn2.BALL_GRID), ("auto", pn2.BALL_AUTO)):
        f = lambda: pn2._ball_query(r, K, xyz, new, False, path, 1)
        t = timeit(f, 10)
        ks = ", ".join(f"{k} {v:.3f}" for k, v in sorted(kernel_ms(f).items(), key=lambda kv: -kv[1]))
        print(f"  {name}: {t:.3f} ms per call; kernels (ms): {ks}", flush=True)


def sweep(B):
    for N, S in ((24000, 1024), (16384, 1024), (65536, 2048)):
        base = [clouds.dental_arch(N, s)[0] for s in range(4)]
        xyz = torch.stack([base[i % 4] for i in range(B if N < 60000 else B // 4)]).cuda().contiguous()
        sel = torch.randperm(N, generator=torch.Generator().manual_seed(1))[:S].cuda()
        new = xyz[:, sel].contiguous()
        for K in (16, 32, 64):
            for r in (0.025, 0.05, 0.075, 0.1, 0.15, 0.2, 0.4):
                t_tile = timeit(lambda: pn2._ball_query(r, K, xyz, new, False, pn2.BALL_TILE))
                t_grid = timeit(lambda: pn2._ball_query(r, K, xyz, new, False, pn2.BALL_GRID))
                t_auto = timeit(lambda: pn2._ball_query(r, K, xyz, new, False, pn2.BALL_AUTO))
                build = kernel_ms(lambda: pn2._ball_query(r, K, xyz, new, False, pn2.BALL_GRID), 3).get("bq_grid_build_kernel", float("nan"))
                print(f"N={N} S={S} K={K} r={r}: tile {t_tile:.3f} grid {t_grid:.3f} (build {build:.3f}) auto {t_auto:.3f} ms",
                      flush=True)


if __name__ == "__main__":
    print(card(), flush=True)
    bench_shape()
    sweep(int(sys.argv[1]) if len(sys.argv) > 1 else 296)
