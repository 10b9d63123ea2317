"""The label transfers of the inference pipelines (sklearn KDTree(..., leaf_size=2).query(..., k=1, return_distance=False) in
float64) on the GPU KDTree drop-in and on scikit-learn, on synthetic float32 arch meshes of 1e5 and 2e5 vertices:

* tgn_final: inference_pipeline_tgn.py:137-140 -- the tree holds float32 copies of 24 000 first-network samples and of up to
  20 000 kept boundary vertices (random subsets of the mesh's vertices stand in for FPS and the boundary subset), so a vertex in
  both parts is in the tree twice; every mesh vertex is queried;
* tgn_clusters: inference_pipeline_tgn.py:107-114 -- one tree on the 24 000 samples, one query per boundary cluster (16);
* sem_tsegnet: inference_pipeline_tsegnet.py:72-74 / inference_pipeline_sem.py:37-39 -- 24 000 sampled vertices, every mesh
  vertex queried; with a plain mesh and with every vertex duplicated (the pipelines keep duplicated vertices).

Per shape: ``gpu_ms`` the drop-in as a pipeline calls it (construction, copies, kernels, host fallback; host clock, median),
split into ``device_ms`` (grid build + tie-flag query, CUDA events) and ``host_fallback_ms`` (scikit-learn's tree built and
queried on the tied rows alone, host clock); ``sklearn_ms``; ``tied_rows``; ``bitwise_equal`` to scikit-learn.  The card's name
and power limit are read in the same run.  There is no CPU mode: without a CUDA device the script fails.

    python scripts/kdtree_bench.py [--reps 5]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from toothgroupnetwork_b200 import _lib as L  # noqa: E402
from toothgroupnetwork_b200 import clouds, neighbors  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, check=True).stdout.strip().splitlines()
        name, power = (x.strip() for x in out[torch.cuda.current_device()].split(","))
        return {"name": name, "power_limit": power}
    except Exception as e:
        return {"name": torch.cuda.get_device_name(), "power_limit": f"unknown ({e!r})"[:80]}


def host_ms(fn, reps):
    ts, out = [], None
    for _ in range(reps):
        torch.cuda.synchronize()
        t = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t) * 1e3)
    return out, float(np.median(ts)), [round(min(ts), 3), round(max(ts), 3)]


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


def shapes(m, seed):
    """(name, tree points, list of query sets) per pipeline shape"""
    verts = clouds.dental_arch(m, seed)[0].numpy()
    rng = np.random.default_rng(seed)
    first = verts[rng.choice(m, 24000, replace=False)]
    bdl = verts[rng.choice(m, min(20000, m // 8), replace=False)]
    clusters = rng.integers(0, 16, bdl.shape[0])
    dup = clouds.with_duplicates(clouds.dental_arch(m // 2, seed)[0], seed).numpy()
    return [
        ("tgn_final", np.concatenate([first, bdl]).astype(np.float32), [verts.astype(np.float64)]),
        ("tgn_clusters", first, [bdl[clusters == c] for c in range(16)]),
        ("sem_tsegnet", first, [verts.astype(np.float64)]),
        ("sem_tsegnet_duplicated_vertices", dup[rng.choice(m, 24000, replace=False)], [dup.astype(np.float64)]),
    ]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("kdtree_bench.py needs a CUDA device: there is no CPU timing of the GPU path")
    from sklearn.neighbors import KDTree as SkKDTree
    c = card()
    print(f"# {c['name']}, power limit {c['power_limit']}")
    for m in (100000, 200000):
        for name, pts, qsets in shapes(m, 7):
            def ours():
                tree = neighbors.KDTree(pts, leaf_size=2)
                return [tree.query(q, k=1, return_distance=False) for q in qsets], tree.host_rows

            def sk():
                tree = SkKDTree(pts, leaf_size=2)
                return [tree.query(q, k=1, return_distance=False) for q in qsets]

            ours()                                                     # warm-up, including the lazy scikit-learn import
            (got, tied), gpu_ms, gpu_range = host_ms(ours, a.reps)
            want, sk_ms, sk_range = host_ms(sk, a.reps)

            # device part: the grid build and one tie-flag query per set on device-resident inputs
            tree = neighbors.KDTree(pts, leaf_size=2)
            qdev = [torch.from_numpy(np.ascontiguousarray(q, dtype=np.float64)).cuda() for q in qsets]
            outs = [(torch.empty((q.shape[0], 1), dtype=torch.int64, device="cuda"), torch.empty(q.shape[0], dtype=torch.uint8, device="cuda"))
                    for q in qdev]

            def device():
                L.call("tgn_knn_f64_build", pts.shape[0], L.ptr(tree._xyz), L.ptr(tree._ws), L.stream_ptr())
                for q, (i, t) in zip(qdev, outs):
                    tree._launch(q, 1, i, None, t)
            device()
            dev_ms = events_ms(device, a.reps)

            # host part: what the drop-in does for the flagged rows -- scikit-learn's tree, built once, queried on them alone
            flagged = [q[tree.query_device(qd, 1)[2].cpu().numpy().astype(bool)] for q, qd in zip(qsets, qdev)]

            def fallback():
                if not any(f.shape[0] for f in flagged):
                    return
                t = SkKDTree(pts, leaf_size=2)
                for f in flagged:
                    if f.shape[0]:
                        t.query(f, k=1, return_distance=False)
            _, fb_ms, _ = host_ms(fallback, a.reps)

            row = {"shape": name, "vertices": m, "tree_points": int(pts.shape[0]), "queries": int(sum(q.shape[0] for q in qsets)),
                   "query_calls": len(qsets), "gpu": c["name"], "power_limit": c["power_limit"],
                   "gpu_ms": round(gpu_ms, 3), "gpu_ms_range": gpu_range, "device_ms": round(dev_ms, 3),
                   "host_fallback_ms": round(fb_ms, 3), "sklearn_ms": round(sk_ms, 3), "sklearn_ms_range": sk_range,
                   "speedup": round(sk_ms / gpu_ms, 2), "tied_rows": int(tied),
                   "bitwise_equal": all(np.array_equal(g, w) for g, w in zip(got, want)), "host_threads": os.cpu_count()}
            print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
