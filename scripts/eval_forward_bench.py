#!/usr/bin/env python
"""Eval-mode (running-statistics BatchNorm) no-grad forwards of DGCNN and PointNet: the reference's forward against the fused one
with promoted accumulation (``accelerate_*_forward(..., running_stats=True)``, DESIGN §3.12 / §3.15), in one run.

* per model at (B, N) = (1, 24 000) and (2, 24 000), running statistics from one train-mode pass over other seeded clouds (per-cloud
  offsets survive the running-mean subtraction): the reference's forward with cuDNN's default TF32 and with TF32 off, and the fused
  forward, timed in alternating CUDA-event windows (median, min, max); the peak-memory growth of each; each output's element-wise
  distance to the float64 evaluation of the reference module (DGCNN: every side on the neighbours of the TF32-off run; the fused
  forward with TF32 off for the module's own last convolution, cls_conv / conv4); the share of points whose argmax differs from
  the TF32-off run's (DGCNN: each side with its own neighbours; the fused forward with cuDNN's default, TF32 on);
* the deepest layer of each model alone (DGCNN conv8, PointNet head conv2: one ``tgn_pw_layer_forward`` with an eval-mode input
  BatchNorm) with accum = 0 and accum = 1 in alternating windows: the cost of the promoted form's 128-row tiles.

The reference's model files come from the staged snapshot (oracle.ref_models).  Prints one JSON object with the card's name and
power limit, and also writes it to the file given by --out.
"""
import argparse
import copy
import ctypes
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
from toothgroupnetwork_b200 import clouds, dgcnn, dropin, pointnet  # noqa: E402
from toothgroupnetwork_b200 import pointnet2_utils as pn2  # noqa: E402

FLOOR = 0.05


def elementwise(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float(((a - b).abs() / b.abs().clamp(min=FLOOR * float(b.abs().max()))).max())


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


def peak_growth(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    out = fn()
    torch.cuda.synchronize()
    return out, torch.cuda.max_memory_allocated() - base


def load_dgcnn(name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ref_models.reference_root(), "models", "modules", "dgcnn.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def load_pointnet(name):
    root = ref_models.reference_root()
    spec = importlib.util.spec_from_file_location(name + "_utils", os.path.join(root, "external_libs", "pointnet2_utils", "pointnet_utils.py"))
    utils = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(utils)
    key = "external_libs.pointnet2_utils.pointnet_utils"
    saved = sys.modules.get(key)
    sys.modules[key] = utils
    try:
        spec = importlib.util.spec_from_file_location(name, os.path.join(root, "models", "modules", "pointnet.py"))
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
    finally:
        if saved is None:
            sys.modules.pop(key, None)
        else:
            sys.modules[key] = saved
    return mod


def inputs(B, N, seed=0):
    f = torch.cat([clouds.arch_features(N, seed + b) for b in range(B)]).cuda()
    return f.transpose(1, 2).contiguous().permute(0, 2, 1)


def make(model, mod, B, N):
    """seeded module in eval mode, negative-scale BatchNorm affines, running statistics of one pass over other clouds"""
    torch.manual_seed(0)
    m = (mod.DGCnnModule(None) if model == "dgcnn" else mod.get_model()).cuda()
    bns = [getattr(m, f"bn{i}") for i in range(1, 9)] if model == "dgcnn" else pointnet._bns(m)
    g = torch.Generator().manual_seed(1)
    with torch.no_grad():
        for bn in bns:
            bn.weight.copy_(torch.rand(bn.num_features, generator=g) * 3.0 - 1.0)
            bn.bias.copy_(torch.rand(bn.num_features, generator=g) * 0.4 - 0.2)
            bn.momentum = 1.0
        m.train()
        m([inputs(B, N, seed=100)])
    for bn in bns:
        bn.momentum = 0.1
    return m.eval()


def first(out):
    return out["cls_pred"] if isinstance(out, dict) else out[0]


def model_rows(model, B, N, a):
    load = load_dgcnn if model == "dgcnn" else load_pointnet
    ref_mod, fused_mod = load(f"ref_{model}_evb_a"), load(f"ref_{model}_evb_b")
    (dropin.accelerate_dgcnn_forward if model == "dgcnn" else dropin.accelerate_pointnet_forward)(fused_mod, running_stats=True)
    x = inputs(B, N)
    base = make(model, ref_mod, B, N)
    mref = base
    mnew = (fused_mod.DGCnnModule(None) if model == "dgcnn" else fused_mod.get_model()).cuda()
    mnew.load_state_dict(base.state_dict())
    mnew.eval()
    mod_of = {"reference_tf32": ref_mod, "reference_fp32": ref_mod, "fused": fused_mod}
    models = {"reference_tf32": mref, "reference_fp32": mref, "fused": mnew}

    def run(tag, knn=None):
        torch.backends.cudnn.allow_tf32 = tag != "reference_fp32"
        mod = mod_of[tag]
        if model == "dgcnn" and knn is not None:
            saved, mod.knn = mod.knn, knn
        try:
            with torch.no_grad():
                return first(models[tag]([x]))
        finally:
            if model == "dgcnn" and knn is not None:
                mod.knn = saved
            torch.backends.cudnn.allow_tf32 = True

    row = {"B": B, "N": N}
    preds = {}
    for tag in models:
        run(tag)
        preds[tag], row[f"{tag}_peak_growth_bytes"] = peak_growth(lambda: run(tag))
    before = L.launch_count()
    run("fused")
    row["fused_launches"] = L.launch_count() - before
    row["times"] = timed_in_turn({tag: (lambda t=tag: run(t)) for tag in models}, 2, a.windows, a.reps)
    row["fused_speedup_over_reference_tf32"] = row["times"]["reference_tf32"]["median_ms"] / row["times"]["fused"]["median_ms"]
    for tag in ("reference_tf32", "fused"):
        row[f"{tag}_argmax_differs_vs_reference_fp32"] = float((preds[tag].argmax(1) != preds["reference_fp32"].argmax(1)).float().mean())
    # distance to float64; DGCNN: every side on the TF32-off run's neighbours
    pinned = []
    if model == "dgcnn":
        orig = ref_mod.knn

        def record(v, k):
            pinned.append(orig(v, k))
            return pinned[-1]

        run("reference_fp32", knn=record)
    m64 = copy.deepcopy(base).double()
    it64 = iter(pinned)
    if model == "dgcnn":
        saved, ref_mod.knn = ref_mod.knn, (lambda v, k: next(it64))
    try:
        with torch.no_grad():
            truth = first(m64([x.double()]))
    finally:
        if model == "dgcnn":
            ref_mod.knn = saved
    del m64
    for tag in models:
        it = iter(pinned)
        if model == "dgcnn":
            with torch.no_grad():
                torch.backends.cudnn.allow_tf32 = tag == "reference_tf32"
                if tag == "fused":
                    got = dgcnn.forward(mnew, [x], knn=lambda v, k: next(it), promote=True)["cls_pred"]
                else:
                    got = run(tag, knn=lambda v, k: next(it))
                torch.backends.cudnn.allow_tf32 = True
        elif tag == "fused":
            torch.backends.cudnn.allow_tf32 = False
            with torch.no_grad():
                got = pointnet.forward(mnew, [x], promote=True)[0]
            torch.backends.cudnn.allow_tf32 = True
        else:
            got = run(tag)
        row[f"{tag}_distance_to_float64"] = elementwise(got, truth)
    row["fused_over_reference_fp32_distance"] = row["fused_distance_to_float64"] / row["reference_fp32_distance_to_float64"]
    # the deepest layer alone, accum 0 / 1
    conv, bn_in = (mnew.conv8[0], mnew.conv7[1]) if model == "dgcnn" else (mnew.conv2, mnew.bn1)
    cout, cin = conv.weight.shape[0], conv.weight.shape[1]
    rows = B * N
    src = torch.randn(cin, rows, device="cuda")
    w = conv.weight.detach().reshape(cout, cin).contiguous()
    packed = torch.empty(L.load().tgn_pw_packed_bytes(cout, cin), dtype=torch.uint8, device="cuda")
    L.call("tgn_pw_pack_weights", cout, cin, L.ptr(w), L.ptr(packed), L.stream_ptr())
    y = torch.empty((cout, rows), device="cuda")
    descs = {}
    for accum in (0, 1):
        d = L.PwLayer()
        d.rows, d.rows_per_batch, d.cin, d.cout, d.mode, d.accum = rows, rows, cin, cout, 0, accum
        d.seg_ptr[0], d.seg_channels[0], d.seg_row_stride[0], d.seg_chan_stride[0] = L.ptr(src), cin, 1, rows
        pn2._PwChain._fill_in_bn(d, bn_in, None)
        d.w_packed, d.y = L.ptr(packed), L.ptr(y)
        descs[f"accum{accum}"] = d
    layer = timed_in_turn({k: (lambda d=d: L.call("tgn_pw_layer_forward", ctypes.byref(d), L.stream_ptr())) for k, d in descs.items()},
                          3, a.windows, 10)
    flop = 2.0 * rows * cin * cout
    row["deepest_layer"] = {"name": "conv8" if model == "dgcnn" else "head conv2", "cin": cin, "cout": cout, "rows": rows, "times": layer,
                            "promoted_over_single_accumulator": layer["accum1"]["median_ms"] / layer["accum0"]["median_ms"],
                            "fp32_equivalent_tflops": {k: flop / (v["median_ms"] * 1e-3) / 1e12 for k, v in layer.items()}}
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=7)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    res = {"card": q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown", "rows": []}
    for model in ("dgcnn", "pointnet"):
        for B in (1, 2):
            res["rows"].append(dict(model=model, **model_rows(model, B, 24000, a)))
            torch.cuda.empty_cache()
    text = json.dumps(res)
    print(text)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
