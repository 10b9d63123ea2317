"""MeanShift(bandwidth=0.07) of get_clustering_labels' elongated-cluster split on the GPU against scikit-learn (DESIGN §3.14).

    python scripts/meanshift_bench.py [--reps 5]

Rows: two adjacent teeth pulled to centroids 0.03 and 0.06 apart (pull 0.93, jitter 0.003), and the two elongated DBSCAN
clusters of an untrained network's cloud (the unmoved arch, 24 000 points).  Per row: the device ascent
(CUDA events, median), the whole ``clustering.MeanShift.fit`` (host clock, median), scikit-learn's fit (once), the seeds redone
on the host, and whether centres, labels and n_iter_ are equal.  Then ``get_clustering_labels`` on that cloud with
scikit-learn's MeanShift (before) and with the device one (after), and equality of the two.  One JSON line, with the card's
name and power limit.
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
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
from make_sklearn_meanshift_golden import merged_teeth  # noqa: E402
from sklearn.cluster import MeanShift as SkMeanShift  # noqa: E402
from toothgroupnetwork_b200 import clouds, clustering  # noqa: E402


def untrained_cloud():
    """moved_cloud(24000, 2, 0.0, 0.0) of tests/test_gpu_clustering.py: the arch as an untrained network leaves it"""
    xyz, _, label = clouds.dental_arch(24000, 2)
    return xyz.numpy(), np.where(label.numpy() < 0, 0, label.numpy()).astype(np.int64)


def elongated_clusters(pts, label):
    """the members get_clustering_labels hands MeanShift, in its order"""
    fg = pts[label != 0]
    lab, core = clustering.dbscan(fg, 0.03, 30)
    core_mask = np.zeros(len(lab), bool)
    core_mask[core] = True
    uniq = [int(u) for u in np.unique(lab) if u != -1]
    eg = np.array([clustering._explained_variance(fg[core_mask & (lab == u)])[0] for u in uniq])
    order = np.argsort(-eg)
    e = eg[order]
    return [fg[lab == uniq[order[i]]].astype(np.float64) for i in range(3) if e[i] / e[3:].mean() > 8]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    pts, label = untrained_cloud()
    split = elongated_clusters(pts, label)
    rows = [("two teeth 0.03 apart", merged_teeth((7, 8), 0.03)), ("two teeth 0.06 apart", merged_teeth((7, 8), 0.06))]
    rows += [(f"untrained arch, elongated cluster {i + 1}", X) for i, X in enumerate(split)]
    res = {"card": card, "rows": []}
    for name, X in rows:
        clustering.MeanShift(0.07).fit(X)                              # warm-up (library load, allocator)
        tree = [torch.from_numpy(t).cuda() for t in clustering.meanshift_tree(X)]
        ev = []
        for _ in range(a.reps):
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            clustering.meanshift_device(*tree, 0.07)
            e.record()
            torch.cuda.synchronize()
            ev.append(s.elapsed_time(e))
        before = clustering.MeanShift.host_seeds
        fit_ms = []
        for _ in range(a.reps):
            t0 = time.perf_counter()
            got = clustering.MeanShift(0.07).fit(X)
            torch.cuda.synchronize()
            fit_ms.append(1e3 * (time.perf_counter() - t0))
        host_seeds = (clustering.MeanShift.host_seeds - before) // a.reps
        t0 = time.perf_counter()
        ref = SkMeanShift(bandwidth=0.07).fit(X)
        sk_ms = 1e3 * (time.perf_counter() - t0)
        equal = (np.array_equal(got.cluster_centers_.view(np.int64), ref.cluster_centers_.view(np.int64))
                 and np.array_equal(got.labels_, ref.labels_) and got.n_iter_ == ref.n_iter_)
        row = {"input": name, "points": len(X), "ascent_ms": float(np.median(ev)), "fit_ms": float(np.median(fit_ms)), "sklearn_ms": sk_ms,
               "speedup": sk_ms / float(np.median(fit_ms)), "host_seeds": int(host_seeds), "centres": len(ref.cluster_centers_),
               "n_iter": int(ref.n_iter_), "equal": bool(equal)}
        res["rows"].append(row)
        print(json.dumps(row), file=sys.stderr)
    # get_clustering_labels on the untrained cloud, scikit-learn's MeanShift in the split (before) and the device one (after)
    device_class = clustering.MeanShift
    t0 = time.perf_counter()
    clustering.MeanShift = SkMeanShift
    try:
        want = clustering.get_clustering_labels(pts, label)
    finally:
        clustering.MeanShift = device_class
    before_s = time.perf_counter() - t0
    t0 = time.perf_counter()
    got = clustering.get_clustering_labels(pts, label)
    after_s = time.perf_counter() - t0
    res["get_clustering_labels"] = {"splits": len(split), "before_s": before_s, "after_s": after_s, "equal": bool(np.array_equal(got, want))}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
