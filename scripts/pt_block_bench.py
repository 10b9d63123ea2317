"""No-grad forwards of the point-transformer network (cbl_point_transformer_module.PointTransformerSeg) with and without the fused
PointTransformerBlock (``blocks_fused.accelerate_blocks``, i.e. ``dropin.accelerate_transformer_blocks``), the fused block taken up
to 16, 32 or 512 channels (``blocks_fused.BLOCK_FUSED_MAX_C``), so that the width it is selected by rests on a measurement; the
fused layers, TransitionDowns, TransitionUps and heads (``accelerate`` + ``accelerate_decoder``) are on in every variant:

* tgnet's first network at 1 x 24 000 points and on the 16 x 3 072 crop batch, and the boundary network (planes [16, 32],
  stride [1, 1], nsample [36, 24]) at 1 x 24 000, train-mode BatchNorm (what the inference pipelines run), random weights;
* the variants alternate (the first one rotating), CUDA events around each forward, median and min over the repetitions;
  forward hooks with CUDA events give the time of the PointTransformerBlocks inside a forward, per width;
* a separate ``torch.profiler`` run counts the CUDA kernels of one forward of each variant and their device time.

The card's name and power limit are read in the same run.  Needs the reference's model files staged by ``build()``.

    python scripts/pt_block_bench.py [--reps 20] [--out PATH.json]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from boundary_bench import card  # noqa: E402
from oracle import ref_models  # noqa: E402
from toothgroupnetwork_b200 import blocks_fused, clouds  # noqa: E402

FIRST = {"stride": [1, 4, 4, 4, 4], "nsample": [36, 24, 24, 24, 24], "blocks": [2, 3, 4, 6, 3], "block_num": 5,
         "planes": [32, 64, 128, 256, 512]}
BOUNDARY = {"stride": [1, 1], "nsample": [36, 24], "blocks": [2, 3], "block_num": 2, "planes": [16, 32]}


# the variants: the class's previous forward (0), and the fused block up to each of these widths (BLOCK_FUSED_MAX_C)
WIDTHS = (0, 16, 32, 512)


class Variants:
    """swap PointTransformerBlock.forward between the class's previous forward and the fused wrapper, and set the widest block
    the wrapper fuses"""

    def __init__(self, blocks, heads):
        self.blocks = blocks
        blocks_fused.accelerate(blocks)
        blocks_fused.accelerate_decoder(blocks, heads)
        self.orig = blocks.PointTransformerBlock.forward
        blocks_fused.accelerate_blocks(blocks)
        self.fused = blocks.PointTransformerBlock.forward
        self.default = blocks_fused.BLOCK_FUSED_MAX_C

    def use(self, max_c: int):
        self.blocks.PointTransformerBlock.forward = self.fused if max_c else self.orig
        blocks_fused.BLOCK_FUSED_MAX_C = max_c or self.default


def section_hooks(model, acc):
    """CUDA events around every PointTransformerBlock call -> acc[width], a list of (start, end) events"""
    handles = []
    for _, m in model.named_modules():
        if type(m).__name__ != "PointTransformerBlock":
            continue

        def pre(mod, args):
            e = torch.cuda.Event(enable_timing=True)
            e.record()
            mod._tgn_ev = e

        def post(mod, args, out):
            e = torch.cuda.Event(enable_timing=True)
            e.record()
            acc.setdefault(mod.linear1.out_features, []).append((mod._tgn_ev, e))

        handles += [m.register_forward_pre_hook(pre), m.register_forward_hook(post)]
    return handles


def _tag(max_c):
    return "unfused_blocks" if max_c == 0 else f"fused_blocks_up_to_c{max_c}"


def run_case(w, variants, B, N, params, reps):
    cpm = w.mod("models.modules.cbl_point_transformer.cbl_point_transformer_module")
    torch.manual_seed(0)
    model = cpm.get_model(c=6, k=17, **params).cuda().train()
    state = {k: v.clone() for k, v in model.state_dict().items()}
    p = torch.stack([clouds.dental_arch(N, b)[0] for b in range(B)]).cuda()           # (B, N, 3)
    x = torch.cat([p, torch.nn.functional.normalize(torch.randn_like(p), dim=-1)], -1).permute(0, 2, 1).contiguous()
    res = {}
    outs = {}
    for v in WIDTHS:                                                                  # warm-up, and the outputs compared
        variants.use(v)
        with torch.no_grad():
            for _ in range(2):
                model.load_state_dict(state)
                o = model([x])
        outs[v] = o[0].double()                                                  # cls_results, (B, k, N)
    ref = outs[0]
    res["cls_max_rel_diff_vs_unfused"] = {_tag(v): float(((outs[v] - ref).abs() / ref.abs().clamp(min=0.05 * float(ref.abs().max()))).max())
                                          for v in WIDTHS[1:]}
    times = {v: [] for v in WIDTHS}
    sections = {v: {} for v in WIDTHS}
    for r in range(reps):
        order = WIDTHS[r % len(WIDTHS):] + WIDTHS[:r % len(WIDTHS)]                  # rotate which variant runs first
        for v in order:
            variants.use(v)
            model.load_state_dict(state)
            acc = {}
            hs = section_hooks(model, acc)
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            with torch.no_grad():
                a.record()
                model([x])
                b.record()
            b.synchronize()
            for h in hs:
                h.remove()
            times[v].append(a.elapsed_time(b))
            for c, evs in acc.items():
                sections[v].setdefault(c, []).append(sum(s.elapsed_time(e) for s, e in evs))
    for v in WIDTHS:
        res[_tag(v)] = {"forward_ms_median": float(np.median(times[v])), "forward_ms_min": float(np.min(times[v])),
                        "blocks_ms_median": float(np.median([sum(t) for t in zip(*sections[v].values())])),
                        "blocks_ms_median_by_width": {c: float(np.median(t)) for c, t in sorted(sections[v].items())}}
    for v in WIDTHS:
        variants.use(v)
        model.load_state_dict(state)
        with torch.no_grad(), torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            model([x])
            torch.cuda.synchronize()
        kernels = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
        res[_tag(v)]["profiler_kernels"] = len(kernels)
        res[_tag(v)]["profiler_kernel_ms"] = sum(e.device_time for e in kernels) / 1e3
    variants.use(variants.default)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    w = ref_models.World("b200")
    with w:
        variants = Variants(w.mod("models.modules.cbl_point_transformer.blocks"), w.mod("models.modules.cbl_point_transformer.heads"))
        report = {"card": card(), "reps": a.reps,
                  "first_network_1x24000": run_case(w, variants, 1, 24000, FIRST, a.reps),
                  "crop_batch_16x3072": run_case(w, variants, 16, 3072, FIRST, a.reps),
                  "boundary_network_1x24000": run_case(w, variants, 1, 24000, BOUNDARY, a.reps)}
    text = json.dumps(report, indent=1)
    print(text)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
