#!/usr/bin/env python
"""PointNet's no-grad forward (models/modules/pointnet.py, get_model) on the GPU: the reference's and the fused one (DESIGN §3.15).

At (B, N) = (1, 24 000) and (2, 24 000), on the permute(0, 2, 1) view of (B, N, 6) arches the sem pipeline passes, with
batch-statistics BatchNorm (train mode, as the sem pipeline runs the model), three forwards are timed in turn in the same
CUDA-event windows after a warm-up:

* ``reference_default`` -- the reference's forward with torch's defaults (cuDNN convolutions in TF32);
* ``reference_fp32``    -- the same with ``torch.backends.cudnn.allow_tf32 = False``;
* ``fused``             -- ``toothgroupnetwork_b200.pointnet.forward`` (``dropin.accelerate_pointnet_forward``).

For each it also reports the peak-memory growth of one forward, the element-wise distance of its log-probabilities and
trans_feat to the float64 evaluation of the same module (|a - b| / max(|b|, 0.05 max|b|)), and the share of points whose argmax
differs from the reference's fp32 run.  The fused forward runs conv4 as the module's own cuDNN convolution, in TF32 under
torch's defaults, so its distance is also reported with TF32 off.  The reference's model files come from the staged snapshot
(oracle.ref_models).  Prints one JSON object with the card's name, power limit and max SM clock read in the same run, and also
writes it to --out.
"""
import argparse
import copy
import importlib.util
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_models  # noqa: E402
from toothgroupnetwork_b200 import clouds, dropin, pointnet  # noqa: E402


def load_reference_pointnet(name):
    root = ref_models.reference_root()
    if root is None:
        raise SystemExit("reference snapshot not staged (oracle/_ref/reference_py.tgz): run __graft_entry__.build() first")
    spec = importlib.util.spec_from_file_location(name + "_utils", os.path.join(root, "external_libs", "pointnet2_utils", "pointnet_utils.py"))
    utils = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(utils)
    sys.modules["external_libs.pointnet2_utils.pointnet_utils"] = utils
    try:
        spec = importlib.util.spec_from_file_location(name, os.path.join(root, "models", "modules", "pointnet.py"))
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
    finally:
        sys.modules.pop("external_libs.pointnet2_utils.pointnet_utils", None)
    return mod


def elementwise(a, b):
    a, b = a.detach().double(), b.detach().double()
    return float(((a - b).abs() / b.abs().clamp(min=0.05 * float(b.abs().max()))).max())


def peak_growth(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    out = fn()
    torch.cuda.synchronize()
    return out, torch.cuda.max_memory_allocated() - base


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=24000)
    ap.add_argument("--batches", type=int, nargs="+", default=[1, 2])
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--windows", type=int, default=9)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("pointnet_bench.py needs a GPU")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    out = {"gpu": q.stdout.strip(), "torch": torch.__version__, "n": a.n, "windows": a.windows, "reps": a.reps, "runs": {}}
    ref_mod, new_mod = load_reference_pointnet("ref_pointnet_bench_a"), load_reference_pointnet("ref_pointnet_bench_b")
    dropin.accelerate_pointnet_forward(new_mod)
    default_tf32 = torch.backends.cudnn.allow_tf32

    for B in a.batches:
        f = torch.cat([clouds.arch_features(a.n, b) for b in range(B)])
        x = f.transpose(1, 2).contiguous().cuda().permute(0, 2, 1)         # inference_pipeline_sem.py:29-31
        torch.manual_seed(0)
        mref = ref_mod.get_model().cuda().train()
        mnew = new_mod.get_model().cuda().train()
        mnew.load_state_dict(mref.state_dict())
        m64 = copy.deepcopy(mref).double()

        def ref_default():
            torch.backends.cudnn.allow_tf32 = default_tf32
            return mref([x])

        def ref_fp32():
            torch.backends.cudnn.allow_tf32 = False
            try:
                return mref([x])
            finally:
                torch.backends.cudnn.allow_tf32 = default_tf32

        def fused():
            return mnew([x])

        legs = {"reference_default": ref_default, "reference_fp32": ref_fp32, "fused": fused}
        row = {}
        with torch.no_grad():
            assert pointnet.fusable(mnew, [x])
            want64 = m64([x.double()])
            results = {}
            for name, fn in legs.items():
                res, grew = peak_growth(fn)
                results[name] = res
                row[name] = {"peak_growth_mb": grew / 2 ** 20, "dist_f64_log_softmax": elementwise(res[0], want64[0]),
                             "dist_f64_trans_feat": elementwise(res[1], want64[1])}
            # the fused forward runs the module's own conv4 through cuDNN, in TF32 under torch's defaults: its distance without TF32
            torch.backends.cudnn.allow_tf32 = False
            row["fused"]["dist_f64_log_softmax_conv4_fp32"] = elementwise(fused()[0], want64[0])
            torch.backends.cudnn.allow_tf32 = default_tf32
            cls32 = results["reference_fp32"][0].argmax(1)
            for name in legs:
                row[name]["argmax_differs_from_reference_fp32"] = float((results[name][0].argmax(1) != cls32).float().mean())
            del results, want64
            for _ in range(a.warmup):
                for fn in legs.values():
                    fn()
            torch.cuda.synchronize()
            times = {name: [] for name in legs}
            for _ in range(a.windows):
                for name, fn in legs.items():
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for _ in range(a.reps):
                        fn()
                    e1.record()
                    e1.synchronize()
                    times[name].append(e0.elapsed_time(e1) / a.reps)
        for name, t in times.items():
            t.sort()
            row[name].update(median_ms=t[len(t) // 2], min_ms=t[0], max_ms=t[-1])
        row["speedup_vs_reference_default"] = row["reference_default"]["median_ms"] / row["fused"]["median_ms"]
        row["speedup_vs_reference_fp32"] = row["reference_fp32"]["median_ms"] / row["fused"]["median_ms"]
        out["runs"][f"B{B}_N{a.n}"] = row
        del mref, mnew, m64
        torch.cuda.empty_cache()

    line = json.dumps(out)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
