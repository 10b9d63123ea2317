"""scikit-learn's KD tree built on the GPU (neighbors.sklearn_tree, csrc/kdtree_build.cu) against scikit-learn's own build, and
the label transfers' tie fallback before and after it.

* build: dental arches of 24 000, 44 000 and 200 000 points, leaf_size 2, 30 and 40, without and with duplicates (a fifth of
  the points repeated).  ``device_ms``: the device build alone (CUDA events, the radius left on the device unset, as MeanShift
  uses it); ``tree_ms``: ``sklearn_tree`` with the host radius pass, ending in a synchronise (host clock); ``sklearn_ms``:
  ``KDTree(X, leaf_size)`` (host clock); ``bitwise_equal`` of the arrays.
* fallback: the tied shapes of scripts/kdtree_bench.py (tgn's final transfer; every vertex twice), leaf_size 2, k = 1:
  ``neighbors.KDTree(...).query`` with the tie fallback's tree built on the host (``before_ms``, the path an installation
  with another state layout still takes) and restored from the device build (``after_ms``), alternating in one process.

Medians of ``--reps`` runs; the card's name and power limit are read in the same run.  There is no CPU mode.

    python scripts/kdtree_build_bench.py [--reps 7]
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
from kdtree_bench import card, events_ms, host_ms, shapes  # noqa: E402
from toothgroupnetwork_b200 import clouds, neighbors  # noqa: E402


def arch(n, seed, duplicates):
    X = clouds.dental_arch(n, seed)[0].double().numpy()
    if duplicates:
        rng = np.random.default_rng(seed)
        X[rng.choice(n, n // 5, replace=False)] = X[rng.choice(n, n // 5)]
    return X


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("kdtree_build_bench.py needs a CUDA device: there is no CPU timing of the GPU path")
    from sklearn.neighbors import KDTree as SkKDTree
    c = card()
    print(f"# {c['name']}, power limit {c['power_limit']}", flush=True)
    for n in (24000, 44000, 200000):
        for leaf_size in (2, 30, 40):
            for dup in (False, True):
                X = arch(n, 3, dup)
                xyz = torch.from_numpy(X).cuda()
                got = [t.cpu().numpy() for t in neighbors.sklearn_tree(X, leaf_size)[1:]]      # warm-up and check
                dev_ms = events_ms(lambda: neighbors.sklearn_tree(xyz, leaf_size, radius=False), a.reps)
                _, tree_ms, tree_range = host_ms(lambda: neighbors.sklearn_tree(X, leaf_size), a.reps)
                want, sk_ms, sk_range = host_ms(lambda: SkKDTree(X, leaf_size=leaf_size).get_arrays(), a.reps)
                equal = (np.array_equal(got[0], want[1]) and got[1].tobytes() == np.ascontiguousarray(want[2]).tobytes()
                         and got[2].tobytes() == want[3].tobytes())
                print(json.dumps({"part": "build", "points": n, "leaf_size": leaf_size, "duplicates": dup, "gpu": c["name"],
                                  "power_limit": c["power_limit"], "device_ms": round(dev_ms, 3), "tree_ms": round(tree_ms, 3),
                                  "tree_ms_range": tree_range, "sklearn_ms": round(sk_ms, 3), "sklearn_ms_range": sk_range,
                                  "bitwise_equal": bool(equal)}), flush=True)

    for m in (100000, 200000):
        for name, pts, qsets in shapes(m, 7):
            if name not in ("tgn_final", "sem_tsegnet_duplicated_vertices"):
                continue

            def run():
                tree = neighbors.KDTree(pts, leaf_size=2)
                return [tree.query(q, k=1, return_distance=False) for q in qsets], tree.host_rows

            times = {"before": [], "after": []}
            outs = {}
            for rep in range(a.reps + 1):
                for mode in ("before", "after"):
                    neighbors._state_ok = False if mode == "before" else None
                    out, ms, _ = host_ms(run, 1)
                    outs[mode] = out
                    if rep:                                               # the first round warms both paths
                        times[mode].append(ms)
            neighbors._state_ok = None
            want = SkKDTree(pts, leaf_size=2)
            equal = all(np.array_equal(g, want.query(q, k=1, return_distance=False)) for g, q in zip(outs["after"][0], qsets))
            before, after = float(np.median(times["before"])), float(np.median(times["after"]))
            print(json.dumps({"part": "fallback", "shape": name, "vertices": m, "tree_points": int(pts.shape[0]), "gpu": c["name"],
                              "power_limit": c["power_limit"], "before_ms": round(before, 3), "after_ms": round(after, 3),
                              "before_range": [round(min(times["before"]), 3), round(max(times["before"]), 3)],
                              "after_range": [round(min(times["after"]), 3), round(max(times["after"]), 3)],
                              "speedup": round(before / after, 2), "tied_rows": int(outs["after"][1]),
                              "same_tied_rows": outs["after"][1] == outs["before"][1], "bitwise_equal": bool(equal)}), flush=True)


if __name__ == "__main__":
    main()
