"""No-grad forwards of the point-transformer network (cbl_point_transformer_module.PointTransformerSeg, tgnet's planes) with the
fused blocks only (``blocks_fused.accelerate``) and with the fused decoder and heads added (``blocks_fused.accelerate_decoder``):

* the first network at 1 x 24 000 points and the same network on the 16 x 3 072 crop batch, train-mode BatchNorm (what the
  inference pipelines run), random weights;
* the two variants alternate, CUDA events around each forward, median over the repetitions; forward hooks with CUDA events give
  the time of the decoder's TransitionUps and of the heads inside a forward;
* a separate ``torch.profiler`` run counts the CUDA kernels of one forward of each variant and their device time.

The card's name and power limit are read in the same run.  Needs the reference's model files staged by ``build()``.

    python scripts/pt_decoder_bench.py [--reps 20] [--out PATH.json]
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

PARAMS = {"stride": [1, 4, 4, 4, 4], "nsample": [36, 24, 24, 24, 24], "blocks": [2, 3, 4, 6, 3], "block_num": 5,
          "planes": [32, 64, 128, 256, 512]}


class Variants:
    """swap TransitionUp.forward / MultiHead.forward between the reference's and the fused wrappers"""

    def __init__(self, blocks, heads):
        self.blocks, self.heads = blocks, heads
        self.orig = (blocks.TransitionUp.forward, heads.MultiHead.forward)
        blocks_fused.accelerate_decoder(blocks, heads)
        self.fused = (blocks.TransitionUp.forward, heads.MultiHead.forward)

    def use(self, fused: bool):
        self.blocks.TransitionUp.forward, self.heads.MultiHead.forward = self.fused if fused else self.orig


def section_hooks(model, acc):
    """CUDA events around every TransitionUp and head call -> acc["decoder"], acc["heads"] lists of (start, end) events"""
    handles = []
    mods = [(n, m) for n, m in model.named_modules() if type(m).__name__ in ("TransitionUp", "MultiHead")]
    for name, m in mods:
        key = "decoder" if type(m).__name__ == "TransitionUp" else "heads"

        def pre(mod, args, key=key):
            e = torch.cuda.Event(enable_timing=True)
            e.record()
            mod._tgn_ev = e

        def post(mod, args, out, key=key):
            e = torch.cuda.Event(enable_timing=True)
            e.record()
            acc.setdefault(key, []).append((mod._tgn_ev, e))

        handles += [m.register_forward_pre_hook(pre), m.register_forward_hook(post)]
    return handles


def run_case(w, variants, B, N, reps):
    cpm = w.mod("models.modules.cbl_point_transformer.cbl_point_transformer_module")
    torch.manual_seed(0)
    model = cpm.get_model(c=6, k=17, **PARAMS).cuda().train()
    state = {k: v.clone() for k, v in model.state_dict().items()}
    p = torch.stack([clouds.dental_arch(N, b)[0] for b in range(B)]).cuda()           # (B, N, 3)
    x = torch.cat([p, torch.nn.functional.normalize(torch.randn_like(p), dim=-1)], -1).permute(0, 2, 1).contiguous()
    res = {}
    outs = {}
    for fused in (False, True):                                                       # warm-up, and the outputs compared
        variants.use(fused)
        model.load_state_dict(state)
        with torch.no_grad():
            for _ in range(2):
                model.load_state_dict(state)
                o = model([x])
        outs[fused] = o[0].double()                                              # cls_results, (B, k, N)
    ref = outs[False]
    res["cls_max_rel_diff"] = float(((outs[True] - ref).abs() / ref.abs().clamp(min=0.05 * float(ref.abs().max()))).max())
    times = {False: [], True: []}
    sections = {False: {"decoder": [], "heads": []}, True: {"decoder": [], "heads": []}}
    for r in range(reps):
        for fused in ((False, True) if r % 2 == 0 else (True, False)):
            variants.use(fused)
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
            times[fused].append(a.elapsed_time(b))
            for key in ("decoder", "heads"):
                sections[fused][key].append(sum(s.elapsed_time(e) for s, e in acc.get(key, [])))
    for fused, tag in ((False, "blocks_only"), (True, "blocks_and_decoder")):
        res[tag] = {"forward_ms_median": float(np.median(times[fused])), "forward_ms_min": float(np.min(times[fused])),
                    "decoder_ms_median": float(np.median(sections[fused]["decoder"])),
                    "heads_ms_median": float(np.median(sections[fused]["heads"]))}
    for fused, tag in ((False, "blocks_only"), (True, "blocks_and_decoder")):
        variants.use(fused)
        model.load_state_dict(state)
        with torch.no_grad(), torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            model([x])
            torch.cuda.synchronize()
        kernels = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
        res[tag]["profiler_kernels"] = len(kernels)
        res[tag]["profiler_kernel_ms"] = sum(e.device_time for e in kernels) / 1e3
    variants.use(True)
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
                  "first_network_1x24000": run_case(w, variants, 1, 24000, a.reps),
                  "crop_batch_16x3072": run_case(w, variants, 16, 3072, a.reps)}
    text = json.dumps(report, indent=1)
    print(text)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
