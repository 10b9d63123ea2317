"""No-grad forwards of the point-transformer network (cbl_point_transformer_module.PointTransformerSeg) run eagerly and replayed as
CUDA graphs (``dropin.accelerate_graphs``, toothgroupnetwork_b200/graphs.py), with the fused layers, TransitionDowns, decoder,
heads and blocks on in both (``accelerate``, ``accelerate_decoder``, ``accelerate_transformer_blocks``):

* tgnet's first network at 1 x 24 000 points and on the 16 x 3 072 crop batch, and the boundary network at 1 x 24 000,
  train-mode BatchNorm (what the inference pipelines run), random weights;
* the default block width (``BLOCK_FUSED_MAX_C`` = 32) and the fused-everywhere variant (512), each eager and graphed;
* eager and graphed forwards alternate (the first one rotating), a host clock around each forward ending in
  ``torch.cuda.synchronize()``: median, min, max and the interquartile range over the repetitions;
* the graph's capture and instantiate time, and the memory of its private pool (the allocator's segments of that pool);
* a separate ``torch.profiler`` run counts the CUDA kernels of one eager forward and one replay and their device time.

The card's name and power limit are read in the same run.  Needs the reference's model files staged by ``build()``.

    python scripts/graph_forward_bench.py [--reps 30] [--out PATH.json]
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from boundary_bench import card  # noqa: E402
from oracle import ref_models  # noqa: E402
from pt_block_bench import BOUNDARY, FIRST  # noqa: E402
from toothgroupnetwork_b200 import blocks_fused, clouds, graphs  # noqa: E402

CPM = "models.modules.cbl_point_transformer.cbl_point_transformer_module"
BLOCKS, HEADS = "models.modules.cbl_point_transformer.blocks", "models.modules.cbl_point_transformer.heads"
WIDTHS = (32, 512)


def world(graphed: bool):
    w = ref_models.World("b200")
    blocks_fused.accelerate_decoder(w.mod(BLOCKS), w.mod(HEADS))
    blocks_fused.accelerate_blocks(w.mod(BLOCKS))
    if graphed:
        graphs.accelerate(w.mod(CPM))
    return w


def pool_bytes(g) -> int:
    pool = tuple(g.pool())
    return sum(s["total_size"] for s in torch.cuda.memory_snapshot() if tuple(s.get("segment_pool_id", ())) == pool)


def timed(w, model, x) -> float:
    with w, torch.no_grad():
        t0 = time.perf_counter()
        model([x])
        torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def stats(ts) -> dict:
    q1, med, q3 = np.percentile(ts, [25, 50, 75])
    return {"median_ms": float(med), "min_ms": float(np.min(ts)), "max_ms": float(np.max(ts)), "iqr_ms": float(q3 - q1)}


def profile(w, model, x) -> dict:
    with w, torch.no_grad(), torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        model([x])
        torch.cuda.synchronize()
    kernels = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    return {"kernels": len(kernels), "kernel_ms": sum(e.device_time for e in kernels) / 1e3}


def run_case(worlds, B, N, params, reps):
    torch.manual_seed(0)
    models = {}
    for tag, w in worlds.items():
        with w:
            models[tag] = w.mod(CPM).get_model(c=6, k=17, **params)
    models["graphed"].load_state_dict(models["eager"].state_dict())
    for m in models.values():
        m.cuda().train()
    p = torch.stack([clouds.dental_arch(N, b)[0] for b in range(B)]).cuda()
    x = torch.cat([p, torch.nn.functional.normalize(torch.randn_like(p), dim=-1)], -1).permute(0, 2, 1).contiguous()
    res = {}
    for width in WIDTHS:
        blocks_fused.BLOCK_FUSED_MAX_C = width
        g = models["graphed"]
        before = dict(graphs.counters)
        for _ in range(3):                                                           # warm-up, capture, first replay
            timed(worlds["graphed"], g, x)
            timed(worlds["eager"], models["eager"], x)
        entries = [e for e in graphs.graph_entries(g).values() if e.graph is not None]
        assert dict(graphs.counters)["capture"] == before.get("capture", 0) + 1 and len(entries) == 1, "no graph was captured"
        e = entries[-1]
        with worlds["graphed"], torch.no_grad():
            got = g([x])
        with worlds["eager"], torch.no_grad():
            want = models["eager"]([x])
        times = {"eager": [], "graphed": []}
        for r in range(reps):
            for tag in (("eager", "graphed") if r % 2 == 0 else ("graphed", "eager")):
                times[tag].append(timed(worlds[tag], models[tag], x))
        out = {tag: stats(ts) for tag, ts in times.items()}
        out["graphed_minus_eager_median_ms"] = out["graphed"]["median_ms"] - out["eager"]["median_ms"]
        out["capture_ms"], out["instantiate_ms"] = e.capture_s * 1e3, e.instantiate_s * 1e3
        out["graph_pool_MiB"] = pool_bytes(e.graph) / 2 ** 20
        out["cls_max_rel_diff_graphed_vs_eager"] = float(((got[0] - want[0]).abs() / want[0].abs().clamp(min=0.05 * float(want[0].abs().max()))).max())
        out["profiler"] = {tag: profile(worlds[tag], models[tag], x) for tag in ("eager", "graphed")}
        res[f"fused_blocks_up_to_c{width}"] = out
        graphs.release_graphs(g)
    blocks_fused.BLOCK_FUSED_MAX_C = WIDTHS[0]
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    worlds = {"eager": world(False), "graphed": world(True)}
    report = {"card": card(), "reps": a.reps,
              "first_network_1x24000": run_case(worlds, 1, 24000, FIRST, a.reps),
              "crop_batch_16x3072": run_case(worlds, 16, 3072, FIRST, a.reps),
              "boundary_network_1x24000": run_case(worlds, 1, 24000, BOUNDARY, a.reps)}
    text = json.dumps(report, indent=1)
    print(text)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
