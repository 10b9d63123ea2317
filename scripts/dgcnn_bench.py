#!/usr/bin/env python
"""DGCNN's feature-space kNN on the GPU against the reference's (models/modules/dgcnn.py:4-10), in one run (DESIGN §3.11).

* per call, at B = 1, N = 24 000, k = 20: C = 6 on the permute(0, 2, 1) view the sem pipeline passes, and C = 64 contiguous as the
  later layers pass it.  Median of CUDA-event windows after a warm-up, the growth of max_memory_allocated over one call, the
  kernel's FP32 rate (2*B*N^2*C FLOP over its time) as a share of the 67 TFLOP/s data-sheet figure, and the outputs compared
  bitwise;
* a whole DGCnnModule forward, no-grad with batch-statistics BatchNorm as the sem pipeline runs it, and one training step
  (forward, cross-entropy, backward), each with and without the drop-in: times, peak memory, cls_pred / loss / gradients bitwise;
* under "fused_forward" (DESIGN §3.12), for batch-statistics and eval-mode BatchNorm: the no-grad forward of the reference, with the
  kNN drop-in only, and fused (``accelerate_forward``), timed in the same windows in turn; the peak-memory growth of each; the
  share of points whose argmax(cls_pred) differs from the reference's; the rows whose layer-2 / layer-3 neighbour sets differ.

The reference's model file comes from the staged snapshot (oracle.ref_models).  Prints one JSON object with the card's name and
power limit, and also writes it to the file given by --out.
"""
import argparse
import importlib.util
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_models  # noqa: E402
from toothgroupnetwork_b200 import _lib as L  # noqa: E402
from toothgroupnetwork_b200 import clouds, dgcnn, dropin  # noqa: E402

FP32_PEAK = 67e12


def timed(fn, warmup, windows, reps):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(windows):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(reps):
            fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b) / reps)
    times.sort()
    return {"median_ms": times[len(times) // 2], "min_ms": times[0], "max_ms": times[-1]}


def peak_growth(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    out = fn()
    torch.cuda.synchronize()
    return out, torch.cuda.max_memory_allocated() - base


def load_reference_dgcnn(name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ref_models.reference_root(), "models", "modules", "dgcnn.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def bits_equal(a, b):
    return bool(torch.equal(a.view(torch.int32), b.view(torch.int32)))


def timed_in_turn(fns, warmup, windows, reps):
    """median / min / max ms per call of each fn, the windows of the fns alternating"""
    for fn in fns.values():
        for _ in range(warmup):
            fn()
    torch.cuda.synchronize()
    times = {tag: [] for tag in fns}
    for _ in range(windows):
        for tag, fn in fns.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(reps):
                fn()
            b.record()
            b.synchronize()
            times[tag].append(a.elapsed_time(b) / reps)
    out = {}
    for tag, t in times.items():
        t.sort()
        out[tag] = {"median_ms": t[len(t) // 2], "min_ms": t[0], "max_ms": t[-1]}
    return out


def fused_forward_rows(a, ref_mod, knn_mod, x6):
    fused_mod = load_reference_dgcnn("ref_dgcnn_bench_c")
    dropin.accelerate_dgcnn_forward(fused_mod)
    torch.backends.cudnn.deterministic = False
    rows = {}
    for bn_mode in ("batch_statistics", "eval"):          # eval mode is refused by dgcnn.fusable: the "fused" model runs the reference
        torch.manual_seed(0)
        base = ref_mod.DGCnnModule(None).cuda().train()
        if bn_mode == "eval":                         # running statistics = the batch statistics of one pass, as after training
            for name in ("bn1", "bn2", "bn3", "bn4", "bn5", "bn6", "bn7", "bn8"):
                getattr(base, name).momentum = 1.0
            with torch.no_grad():
                base([x6])
            for name in ("bn1", "bn2", "bn3", "bn4", "bn5", "bn6", "bn7", "bn8"):
                getattr(base, name).momentum = 0.1
        models = {}
        for tag, mod in (("reference", ref_mod), ("knn_only", knn_mod), ("fused", fused_mod)):
            m = mod.DGCnnModule(None).cuda()
            m.load_state_dict(base.state_dict())
            models[tag] = m.train() if bn_mode == "batch_statistics" else m.eval()

        def forward(tag):
            with torch.no_grad():
                torch.manual_seed(1)
                return models[tag]([x6])["cls_pred"]

        row = {}
        preds = {}
        for tag in models:
            forward(tag)
            preds[tag], row[f"{tag}_peak_growth_bytes"] = peak_growth(lambda: forward(tag))
        before = L.launch_count()
        forward("fused")
        row["fused_launches"] = L.launch_count() - before
        row["times"] = timed_in_turn({tag: (lambda t=tag: forward(t)) for tag in models}, 2, a.windows, 3)
        row["fused_speedup_over_knn_only"] = row["times"]["knn_only"]["median_ms"] / row["times"]["fused"]["median_ms"]
        row["fused_speedup_over_reference"] = row["times"]["reference"]["median_ms"] / row["times"]["fused"]["median_ms"]
        row["argmax_differs_fraction"] = float((preds["fused"].argmax(1) != preds["reference"].argmax(1)).float().mean())
        saved = torch.backends.cudnn.allow_tf32
        torch.backends.cudnn.allow_tf32 = False
        try:
            ref_fp32 = forward("reference")
        finally:
            torch.backends.cudnn.allow_tf32 = saved
        row["argmax_differs_fraction_vs_reference_without_tf32"] = float((preds["fused"].argmax(1) != ref_fp32.argmax(1)).float().mean())
        row["argmax_differs_fraction_reference_tf32_vs_fp32"] = float((preds["reference"].argmax(1) != ref_fp32.argmax(1)).float().mean())
        # neighbour sets of layers 2 and 3: the reference's own search on its features against the kernel's on the fused ones
        ref_idx, new_idx = [], []
        original = ref_mod.knn
        ref_mod.knn = lambda v, k: ref_idx.append(original(v, k)) or ref_idx[-1]
        try:
            forward("reference")
        finally:
            ref_mod.knn = original
        with torch.no_grad():
            torch.manual_seed(1)
            dgcnn.forward(models["fused"], [x6], knn=lambda v, k: new_idx.append(dgcnn.knn_features(v, k)) or new_idx[-1])
        row["neighbour_rows_differing"] = [int((u.sort(-1)[0] != w.sort(-1)[0]).any(-1).sum()) for u, w in zip(ref_idx, new_idx)]
        rows[bn_mode] = row
    return rows


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=24000)
    ap.add_argument("--k", type=int, default=20)
    ap.add_argument("--windows", type=int, default=7)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "dgcnn_bench.py measures on a CUDA device"
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    out = {"gpu": q.stdout.strip(), "torch": torch.__version__, "n": a.n, "k": a.k, "calls": {}, "model": {}}
    ref_mod, new_mod = load_reference_dgcnn("ref_dgcnn_bench_a"), load_reference_dgcnn("ref_dgcnn_bench_b")
    dropin.accelerate_dgcnn(new_mod)
    feats = clouds.arch_features(a.n).cuda()                                 # (1, 6, N)
    x6 = feats.transpose(1, 2).contiguous().permute(0, 2, 1)                 # inference_pipeline_sem.py:30
    g = torch.Generator().manual_seed(17)
    x64 = torch.nn.functional.leaky_relu(torch.einsum("oc,bcn->bon", torch.randn(64, 6, generator=g) * 2.0, feats.cpu())
                                         + 0.1 * torch.randn(1, 64, a.n, generator=g), 0.2).cuda()

    for name, x in (("C6_permuted", x6), ("C64_contiguous", x64)):
        C = x.shape[1]
        row = {}
        want, row["reference_peak_growth_bytes"] = peak_growth(lambda: ref_mod.knn(x, a.k))
        got, row["kernel_peak_growth_bytes"] = peak_growth(lambda: dgcnn.knn_features(x, a.k))
        before = L.launch_count()
        dropped = new_mod.knn(x, a.k)
        row["dropin_ran_kernel"] = L.launch_count() == before + 1
        row["indices_equal"] = bool(torch.equal(got, want)) and bool(torch.equal(dropped, want))
        row["reference"] = timed(lambda: ref_mod.knn(x, a.k), 3, a.windows, a.reps)
        row["kernel"] = timed(lambda: dgcnn.knn_features(x, a.k), 3, a.windows, a.reps)
        row["speedup"] = row["reference"]["median_ms"] / row["kernel"]["median_ms"]
        flop = 2.0 * x.shape[0] * a.n * a.n * C
        row["kernel_fp32_tflops"] = flop / (row["kernel"]["median_ms"] * 1e-3) / 1e12
        row["kernel_share_of_fp32_peak"] = flop / (row["kernel"]["median_ms"] * 1e-3) / FP32_PEAK
        out["calls"][name] = row

    torch.backends.cudnn.benchmark = False
    torch.backends.cudnn.deterministic = True
    labels = torch.randint(0, 17, (1, a.n), generator=torch.Generator().manual_seed(9)).cuda()
    models = {}
    for tag, mod in (("reference", ref_mod), ("dropin", new_mod)):
        torch.manual_seed(0)
        models[tag] = mod.DGCnnModule(None).cuda().train()

    def forward(tag):
        with torch.no_grad():
            torch.manual_seed(1)
            return models[tag]([x6])["cls_pred"]

    def step(tag):
        m = models[tag]
        m.zero_grad(set_to_none=True)
        torch.manual_seed(1)
        pred = m([x6])["cls_pred"]
        loss = torch.nn.functional.cross_entropy(pred, labels)
        loss.backward()
        return pred.detach(), loss.detach(), [p.grad for p in m.parameters() if p.grad is not None]

    preds, steps = {}, {}
    torch.use_deterministic_algorithms(True, warn_only=True)     # the gather's backward in a fixed order, so gradients compare
    for tag in models:
        preds[tag], fpeak = peak_growth(lambda: forward(tag))
        steps[tag], speak = peak_growth(lambda: step(tag))
        out["model"][tag] = {"forward_no_grad": timed(lambda: forward(tag), 2, 5, 3), "forward_peak_growth_bytes": fpeak,
                             "train_step": timed(lambda: step(tag), 2, 5, 2), "train_step_peak_growth_bytes": speak}
    torch.use_deterministic_algorithms(False)
    out["model"]["cls_pred_bitwise_equal"] = bits_equal(preds["reference"], preds["dropin"])
    (p0, l0, g0), (p1, l1, g1) = steps["reference"], steps["dropin"]
    out["model"]["train_step_bitwise_equal"] = bits_equal(p0, p1) and bits_equal(l0, l1) and len(g0) == len(g1) and all(
        bits_equal(u, v) for u, v in zip(g0, g1))
    for key in ("forward_no_grad", "train_step"):
        out["model"][f"{key}_speedup"] = out["model"]["reference"][key]["median_ms"] / out["model"]["dropin"][key]["median_ms"]

    out["fused_forward"] = fused_forward_rows(a, ref_mod, new_mod, x6)

    if a.out:
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
