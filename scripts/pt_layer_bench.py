"""Fused PointTransformerLayer forward (csrc/pt_layer.cu) per level of the tgnet_fps encoder: warp-per-query against CTA-per-query
schedule, and the reference's unfused torch code on this package's operators, train-mode BatchNorm, no_grad.

The boundary network's c = 16 level (tgnet_bdl: 24 000 points, or 16 crops of 3 072) has one schedule (two queries per warp), so its
rows time the fused layer against the unfused code only: five alternating rounds of each, the median reported."""
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from test_gpu_blocks import Layer  # noqa: E402

from toothgroupnetwork_b200 import _lib as L  # noqa: E402
from toothgroupnetwork_b200 import blocks_fused, clouds, pointops  # noqa: E402


def unfused(layer, p, x, o):
    """blocks.py:31-44 written out (what runs when the fused path is off), on this package's queryandgroup"""
    x_q, x_k, x_v = layer.linear_q(x), layer.linear_k(x), layer.linear_v(x)
    x_k = pointops.queryandgroup(layer.nsample, p, p, x_k, None, o, o, use_xyz=True)
    x_v = pointops.queryandgroup(layer.nsample, p, p, x_v, None, o, o, use_xyz=False)
    p_r, x_k = x_k[:, :, 0:3], x_k[:, :, 3:]
    for i, m in enumerate(layer.linear_p):
        p_r = m(p_r.transpose(1, 2).contiguous()).transpose(1, 2).contiguous() if i == 1 else m(p_r)
    w = x_k - x_q.unsqueeze(1) + p_r
    for i, m in enumerate(layer.linear_w):
        w = m(w.transpose(1, 2).contiguous()).transpose(1, 2).contiguous() if i % 3 == 0 else m(w)
    w = torch.softmax(w, dim=1)
    n, K, c = x_v.shape
    return ((x_v + p_r).view(n, K, 8, c // 8) * w.unsqueeze(2)).sum(1).view(n, c)


def time_ms(fn, reps=20):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def c16_row(K, n):
    """fused against unfused at c = 16, alternated within one process so that both see the same clocks and neighbours"""
    layer = Layer(16, K).cuda().train()
    p = clouds.dental_arch(n, 1)[0].cuda().contiguous()
    x = torch.randn(n, 16, device="cuda")
    o = torch.tensor([n], dtype=torch.int32, device="cuda")
    fused, ref = [], []
    with torch.no_grad():
        for _ in range(5):
            fused.append(time_ms(lambda: blocks_fused.pt_layer_forward(layer, [p, x, o]), reps=100))
            ref.append(time_ms(lambda: unfused(layer, p, x, o), reps=20))
    return {"c": 16, "K": K, "n": n, "default_ms": statistics.median(fused), "unfused_torch_ms": statistics.median(ref),
            "default_ms_rounds": fused, "unfused_torch_ms_rounds": ref}


def main():
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print(json.dumps({"device": torch.cuda.get_device_name(0), "name_power_limit_max_sm_clock": card}))
    rows = []
    lib = L.load()
    for K, n in ((36, 24000), (36, 49152)):
        rows.append(c16_row(K, n))
        print(json.dumps(rows[-1]))
    for c, K, n in ((32, 36, 24000), (64, 24, 6000), (128, 24, 1500), (256, 24, 375), (512, 24, 93), (32, 36, 49152), (64, 24, 12288), (128, 24, 3072)):
        layer = Layer(c, K).cuda().train()
        p = clouds.dental_arch(n, 1)[0].cuda().contiguous()
        x = torch.randn(n, c, device="cuda")
        o = torch.tensor([n], dtype=torch.int32, device="cuda")
        row = {"c": c, "K": K, "n": n}
        with torch.no_grad():
            for name, thr in (("warp_per_query_ms", 0), ("cta_per_query_ms", 1 << 30)):
                old = lib.tgn_pt_layer_set_cta_threshold(thr)
                row[name] = time_ms(lambda: blocks_fused.pt_layer_forward(layer, [p, x, o]))
                lib.tgn_pt_layer_set_cta_threshold(old)
            row["default_ms"] = time_ms(lambda: blocks_fused.pt_layer_forward(layer, [p, x, o]))
            row["unfused_torch_ms"] = time_ms(lambda: unfused(layer, p, x, o), reps=5)
        rows.append(row)
        print(json.dumps(row))
    with open(os.path.join(ROOT, "gpurun_out", "r2_pt_layer_bench.json"), "w") as f:
        json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
