"""The label transfers' tied rows walked on the GPU (neighbors.DeviceKDTree, csrc/kdtree_query.cu) against the host fallback
they replace and against scikit-learn.

Shapes: the tied transfers of DESIGN §3.10 -- tgn's final transfer (FPS samples plus kept boundary vertices, queried with
every vertex) and tsegnet / sem with every vertex twice -- at 10^5 and 2*10^5 vertices, leaf_size 2, k = 1.  Per shape, in one
process and alternating, ``--reps`` rounds (after one warm-up round) of ``cls(points, leaf_size=2).query(vertices, k=1)`` with
a host clock that ends in a device synchronise, for three classes: ``neighbors.KDTree`` (tied rows answered by scikit-learn's
query code on the device-built tree), ``neighbors.DeviceKDTree`` (tied rows walked on the device) and scikit-learn's
``KDTree``.  Also the walk kernel alone on the tied rows (``sklearn_query`` with ``rows=``, CUDA events, tree prebuilt), the
tied, walked and host rows, and whether both GPU classes return scikit-learn's indices and distance bits.  The card's name and
power limit are read in the same run.  There is no CPU mode.

    python scripts/kdtree_query_bench.py [--reps 5]
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
from kdtree_bench import card, events_ms, shapes  # noqa: E402
from toothgroupnetwork_b200 import neighbors  # noqa: E402

LEAF_SIZE = 2


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("kdtree_query_bench.py needs a CUDA device: there is no CPU timing of the GPU path")
    from sklearn.neighbors import KDTree as SkKDTree
    c = card()
    print(f"# {c['name']}, power limit {c['power_limit']}", flush=True)
    classes = {"host_fallback": neighbors.KDTree, "device_walk": neighbors.DeviceKDTree, "sklearn": SkKDTree}
    for m in (100000, 200000):
        for name, pts, qsets in shapes(m, 7):
            if name not in ("tgn_final", "sem_tsegnet_duplicated_vertices"):
                continue
            q = qsets[0]
            times = {v: [] for v in classes}
            outs, trees = {}, {}
            for rep in range(a.reps + 1):
                for variant, cls in classes.items():
                    torch.cuda.synchronize()
                    t = time.perf_counter()
                    tree = cls(pts, leaf_size=LEAF_SIZE)
                    out = tree.query(q, k=1)
                    torch.cuda.synchronize()
                    if rep:                                           # the first round warms every path
                        times[variant].append((time.perf_counter() - t) * 1e3)
                    outs[variant], trees[variant] = out, tree
            wd, wi = outs["sklearn"]
            equal = {v: bool(np.array_equal(outs[v][1], wi) and outs[v][0].tobytes() == wd.tobytes())
                     for v in ("host_fallback", "device_walk")}
            # the walk kernel alone on the tied rows
            q_dev = torch.from_numpy(q).cuda()
            _, _, tie = neighbors.KDTree(pts, leaf_size=LEAF_SIZE).query_device(q_dev, 1)
            tied = torch.nonzero(tie).flatten()
            walk_tree = neighbors.sklearn_tree(torch.from_numpy(np.asarray(pts, np.float64)).cuda(), LEAF_SIZE, radius=False)
            walk_ms = events_ms(lambda: neighbors._walk(walk_tree, q_dev, 1, tied, torch.empty((q.shape[0], 1), dtype=torch.int64,
                                                                                                  device="cuda"),
                                                        None, torch.empty(q.shape[0], dtype=torch.uint8, device="cuda")),
                                a.reps + 5)
            med = {v: float(np.median(t)) for v, t in times.items()}
            rng_ = {v: [round(min(t), 3), round(max(t), 3)] for v, t in times.items()}
            print(json.dumps({"shape": name, "vertices": m, "tree_points": int(pts.shape[0]), "leaf_size": LEAF_SIZE,
                              "gpu": c["name"], "power_limit": c["power_limit"],
                              "host_fallback_ms": round(med["host_fallback"], 3), "host_fallback_range": rng_["host_fallback"],
                              "device_walk_ms": round(med["device_walk"], 3), "device_walk_range": rng_["device_walk"],
                              "sklearn_ms": round(med["sklearn"], 3), "sklearn_range": rng_["sklearn"],
                              "walk_kernel_ms": round(walk_ms, 4),
                              "speedup_vs_host_fallback": round(med["host_fallback"] / med["device_walk"], 2),
                              "speedup_vs_sklearn": round(med["sklearn"] / med["device_walk"], 2),
                              "tied_rows": int(tied.numel()), "walk_rows": trees["device_walk"].walk_rows,
                              "host_rows": trees["device_walk"].host_rows,
                              "host_fallback_rows": trees["host_fallback"].host_rows,
                              "bitwise_equal": equal}), flush=True)


if __name__ == "__main__":
    main()
