"""Boundary detection and resampling between tgnet's two networks (InferencePipeLine.get_boundary_sampled_feats,
inference_pipeline_tgn.py:289-330) on synthetic float64 arch meshes of 1e5 and 2e5 vertices with a tooth-bin label field:

* device: the float64 kNN + label vote alone (csrc/knn_f64.cu) and the whole ``boundary.boundary_sample``, CUDA events after a
  warm-up, median of the repetitions;
* drop-in: ``boundary.get_boundary_sampled_feats`` with numpy in and out (uploads and downloads included), host clock;
* reference: the reference's own method (scikit-learn KDTree, count_unique_by_row, FPS on the verbatim pointops kernel) when
  the reference snapshot is staged, host clock, and whether the drop-in's four arrays equal its answer bit for bit.

The card's name and power limit are read in the same run.

    python scripts/boundary_bench.py [--reps 10]
"""
import argparse
import importlib
import json
import os
import subprocess
import sys
import time
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from toothgroupnetwork_b200 import boundary, clouds  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, check=True).stdout.strip().splitlines()
        name, power = (x.strip() for x in out[torch.cuda.current_device()].split(","))
        return {"name": name, "power_limit": power}
    except Exception as e:                   # the numbers stay, the card is named as far as torch knows it
        return {"name": torch.cuda.get_device_name(), "power_limit": f"unknown ({e!r})"[:80]}


def events_ms(fn, reps):
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def host_ms(fn, reps):
    ts, out = [], None
    for _ in range(reps):
        torch.cuda.synchronize()
        t = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t) * 1e3)
    return out, float(np.median(ts))


def reference_method():
    try:
        from oracle import ref_cuda, ref_models
    except Exception:
        return None, None
    if not (ref_models.available() and ref_cuda.available()):
        return None, None
    w = ref_models.World("reference")
    # the world does not preload inference_pipelines: import it inside the world (so it binds the world's gen_utils, models and
    # pointops) and take it back out of sys.modules afterwards
    is_pkg = lambda n: n.split(".")[0] == "inference_pipelines"
    with w:
        saved = {n: sys.modules.pop(n) for n in list(sys.modules) if is_pkg(n)}
        try:
            mod = importlib.import_module("inference_pipelines.inference_pipeline_tgn")
        finally:
            for n in [n for n in sys.modules if is_pkg(n)]:
                del sys.modules[n]
            sys.modules.update(saved)
    return w, mod.InferencePipeLine.get_boundary_sampled_feats


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    a = ap.parse_args()
    c = card()
    print(f"# {c['name']}, power limit {c['power_limit']}")
    world, ref = reference_method()
    me = types.SimpleNamespace(config={"boundary_sampling_info": {"bdl_ratio": 0.7, "num_of_bdl_points": 20000, "num_of_all_points": 24000}})
    rows = []
    for m in (100000, 200000):
        org, sampled, labels = clouds.boundary_inputs(m, 7)
        pts, q = torch.from_numpy(sampled[:, :3]).cuda(), torch.from_numpy(org[:, :3]).cuda()
        lab, feats = torch.from_numpy(labels).cuda(), torch.from_numpy(org).cuda()
        codes = boundary.label_codes(lab)
        vote = lambda: boundary.neighbour_vote(pts, q, codes, 40)
        rng = np.random.default_rng(0)
        whole = lambda: boundary.boundary_sample(pts, lab, feats, bdl_ratio=0.7, num_bdl=20000, num_all=24000, perm=rng.permutation)
        for _ in range(3):
            vote()
            whole()
        torch.cuda.synchronize()
        row = {"vertices": m, "sampled": int(sampled.shape[0]), "k": 40, "gpu": c["name"], "power_limit": c["power_limit"],
               "knn_vote_ms": events_ms(vote, a.reps), "boundary_sample_ms": events_ms(whole, a.reps)}
        np.random.seed(11)
        got, row["dropin_ms"] = host_ms(lambda: boundary.get_boundary_sampled_feats(me, labels, org, sampled, None), a.reps)
        row["boundary_rows_kept"] = int(got[2].shape[0])
        if ref is not None:
            np.random.seed(11)
            with world:
                want, row["reference_ms"] = host_ms(lambda: ref(me, labels, org, sampled, None), 1)
            np.random.seed(11)
            got = boundary.get_boundary_sampled_feats(me, labels, org, sampled, None)
            row["bitwise_equal_to_reference"] = all(g.dtype == r.dtype and np.array_equal(g, r) for g, r in zip(got, want))
        else:
            row["reference_ms"] = "not staged"
        row["host_threads"] = os.cpu_count()
        rows.append(row)
        print(json.dumps(row))


if __name__ == "__main__":
    main()
