"""The group-MLP stage of bench.py on its own: ``pn2.sa_group_mlp_max`` (gather -> 9->[32,32,64] -> max over K) at the
bench shape (B = 1056 clouds, S = 1024, K = 32), on the split-fp16 tensor-core engine in full-size (TC) and half-size
(TC_HALF) CTAs and on the exact-fp32 CUDA-core engine.  ``gidx`` and ``new_xyz`` come from the real FPS + ball query
on bench.py's own clouds and module.

Each engine is warmed up, then timed with CUDA events over --windows windows of --launches back-to-back launches;
the median window is reported as ms per launch, with useful TFLOP/s (2 * rows * sum C_l * C_l+1), issued FP16
TFLOP/s (the split-fp16 engine's padded MMAs, no tile falling back to 3xTF32) and that rate as a fraction of the H100 SXM
data-sheet dense FP16 peak (989 TFLOP/s at 700 W).  The card's name, power limit and max SM clock are read in the same run.

    python scripts/sa_mlp_bench.py [--clouds B] [--windows 7] [--launches 20]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (the workload's constants, clouds and module)
from toothgroupnetwork_b200 import pointnet2_utils as pn2  # noqa: E402

F16_PEAK_TFLOPS = 989.0           # H100 SXM data sheet, dense FP16, 700 W


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        name, power, clock = (x.strip() for x in out[torch.cuda.current_device()].split(","))
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:             # the timings stand without it; say so instead of guessing
        return {"name": torch.cuda.get_device_name(), "power_limit": f"unknown ({e!r})"[:80], "max_sm_clock": "unknown"}


def issued_f16_macs_per_row(channels):
    """FP16 MACs the tensor engine issues per grouped row, every split-fp16 term included.  Every layer runs transposed
    (weights on M, the tile's rows on N).  The inner layers run on 64 weight rows at K = C_0 rounded up to 16, then the
    previous width rounded up to 16; at inner widths up to 32 the rows pack W_hi and W_lo' of a channel (two MMAs per K-step),
    wider ones hold one channel per row (three).  The last layer runs in 64-channel slices, three MMAs per K-step."""
    L = len(channels) - 1
    np_ = max([16] + [(c + 15) // 16 * 16 for c in channels[1:L]])
    kpad = [(channels[0] + 15) // 16 * 16] + [(c + 15) // 16 * 16 for c in channels[1:L]]
    inner = sum(k * 64 * (2 if np_ <= 32 else 3) for k in kpad[:L - 1])
    return inner + kpad[L - 1] * 64 * 3 * ((channels[L] + 63) // 64)


def time_engine(fn, windows, launches):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(windows):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(launches):
            fn()
        e1.record()
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1) / launches)
    return float(np.median(ms)), ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clouds", type=int, default=1056)
    ap.add_argument("--windows", type=int, default=7)
    ap.add_argument("--launches", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("sa_mlp_bench.py needs a CUDA device")
    assert args.windows >= 5 and args.launches >= 20, "at least 5 windows of 20 launches"
    dev = torch.device("cuda", 0)
    B, S, K = args.clouds, bench.NPOINT, bench.NSAMPLE
    sa = bench.build_module(dev)
    feats = bench.make_clouds(0, B).to(dev)
    xyz = feats[:, :3].contiguous()
    folded = sa._folded.update(sa.mlp_convs, sa.mlp_bns)
    with torch.no_grad():
        xyz_t, feats_t = pn2.transpose_last2(xyz), pn2.transpose_last2(feats)
        fps = pn2._fps_batched(xyz_t, S)
        new_xyz_t = pn2._take_rows(xyz_t.view(-1, 3), fps).view(B, S, 3)
        gidx = pn2._ball_query(bench.RADIUS, K, xyz_t, new_xyz_t, False, None, 1)
    torch.cuda.synchronize()

    channels = [9] + list(bench.MLP)
    rows = B * S * K
    useful = 2.0 * rows * sum(a * b for a, b in zip(channels[:-1], channels[1:]))
    issued = 2.0 * rows * issued_f16_macs_per_row(channels)
    outs, result = {}, {"card": card(), "shape": {"B": B, "S": S, "K": K, "channels": channels}, "engines": {}}
    for name, engine in (("TC", pn2.ENGINE_TC), ("TC_HALF", pn2.ENGINE_TC_HALF), ("FP32", pn2.ENGINE_FP32)):
        out = torch.empty((B, channels[-1], S), device=dev)
        fn = lambda: pn2.sa_group_mlp_max(xyz_t, feats_t, new_xyz_t, gidx, True, folded, out, 0, engine=engine)  # noqa: E731
        med, ms = time_engine(fn, args.windows, args.launches)
        outs[name] = out
        rec = {"ms": med, "windows_ms": [round(m, 4) for m in ms], "useful_tflops": useful / (med * 1e-3) / 1e12}
        if name != "FP32":
            rec["issued_f16_tflops"] = issued / (med * 1e-3) / 1e12
            rec["frac_of_f16_peak"] = rec["issued_f16_tflops"] / F16_PEAK_TFLOPS
        result["engines"][name] = rec
    ref = outs["FP32"].double()
    floor = 0.05 * float(ref.abs().max())
    for name in ("TC", "TC_HALF"):
        result["engines"][name]["elementwise_rel_vs_fp32"] = float(((outs[name].double() - ref).abs() / ref.abs().clamp(min=floor)).max())

    c = result["card"]
    print(f"# {c['name']}, power limit {c['power_limit']}, max SM clock {c['max_sm_clock']}; B={B} S={S} K={K} {channels}")
    print(f"# useful {useful / 1e9:.1f} GFLOP, issued split-fp16 {issued / 1e9:.1f} GFLOP per launch")
    print("| engine | ms (median) | useful TFLOP/s | issued FP16 TFLOP/s | of 989 |")
    print("|---|---|---|---|---|")
    for name, rec in result["engines"].items():
        print(f"| {name} | {rec['ms']:.3f} | {rec['useful_tflops']:.1f} | {rec.get('issued_f16_tflops', float('nan')):.1f} | "
              f"{rec.get('frac_of_f16_peak', float('nan')):.3f} |")
    print(json.dumps(result))


if __name__ == "__main__":
    main()
