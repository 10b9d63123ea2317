"""Writes tests/golden/ref_sklearn_meanshift.npz: scikit-learn 1.9's own MeanShift(bandwidth, max_iter).fit on float64 (n, 3)
clusters like the ones ops_utils.get_clustering_labels splits, for tests/test_cpu_meanshift.py and tests/test_gpu_meanshift.py.

    python tests/golden/make_sklearn_meanshift_golden.py

Per case ``<name>_``: points, bandwidth, max_iter, idx_array (of ``KDTree(points, leaf_size=30)``), the per-seed results of
``_mean_shift_single_seed`` (seed_means, seed_counts, seed_iters), and the fit's cluster_centers, labels and n_iter.
"""
import os
import sys

import numpy as np
from sklearn.cluster import MeanShift
from sklearn.cluster._mean_shift import _mean_shift_single_seed
from sklearn.neighbors import KDTree, NearestNeighbors

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from toothgroupnetwork_b200 import clouds  # noqa: E402


def merged_teeth(teeth, sep, seed=2, n=24000, pull=0.93, jitter=0.003):
    """the points of adjacent teeth whose centroids a partly trained network pulled to within ``sep`` of each other: one
    elongated DBSCAN cluster"""
    xyz, _, label = clouds.dental_arch(n, seed)
    xyz, label = xyz.numpy().astype(np.float64), label.numpy().astype(np.int64)
    label = np.where(label < 0, 0, label)
    cent = np.stack([xyz[label == c].mean(0) if (label == c).any() else np.zeros(3) for c in range(int(label.max()) + 1)])
    d = cent[teeth[-1]] - cent[teeth[0]]
    d /= np.linalg.norm(d)
    mid = cent[list(teeth)].mean(0)
    for j, t in enumerate(teeth):
        cent[t] = mid + d * sep * (j - (len(teeth) - 1) / 2)
    rng = np.random.default_rng(seed)
    moved = xyz + pull * (cent[label] - xyz) + rng.normal(0, jitter, xyz.shape)
    return moved.astype(np.float32)[np.isin(label, teeth)].astype(np.float64)


def cases():
    rng = np.random.default_rng(11)
    yield "two_teeth", merged_teeth((7, 8), 0.03), 0.07, 300
    yield "three_teeth", merged_teeth((6, 7, 8), 0.04), 0.07, 300
    xyz, _, label = clouds.dental_arch(24000, 2)
    arch = xyz.numpy()[label.numpy() > 0].astype(np.float64)
    yield "arch", arch[rng.permutation(len(arch))[:3000]], 0.07, 300           # many modes along the arch, long climbs
    x0 = rng.normal(0, 0.03, (1200, 3))
    x0[:300, 0] = 0.0
    x0[300:600, 0] = -0.0
    x0[600:650, 1] = -0.0
    x0[650:700] = -0.0                                                           # (-0, -0, -0) and, after these, (+0, -0, -0)
    x0[700:720] = np.array([0.0, -0.0, -0.0])
    yield "signed_zeros", x0, 0.07, 300
    dup = rng.normal(0, 0.02, (400, 3)) + np.array([0.05, 0.0, 0.0]) * rng.integers(0, 3, (400, 1))
    yield "duplicates", np.concatenate([dup, dup[:250], dup[:60]])[rng.permutation(710)], 0.07, 300
    yield "small", rng.normal(0, 0.03, (30, 3)), 0.07, 300
    yield "max_iter_2", merged_teeth((7, 8), 0.06), 0.07, 2
    plane = np.concatenate([rng.uniform(-0.1, 0.1, (900, 2)) * np.array([1.5, 1.0]), np.full((900, 1), 0.25)], axis=1)
    yield "planar", plane, 0.07, 300


def main():
    out = {}
    for name, X, r, max_iter in cases():
        X = np.ascontiguousarray(X, dtype=np.float64)
        idx = KDTree(X, leaf_size=30).get_arrays()[1]
        nbrs = NearestNeighbors(radius=r, n_jobs=1).fit(X)
        seeds = [_mean_shift_single_seed(x, X, nbrs, max_iter) for x in X]
        ms = MeanShift(bandwidth=r, max_iter=max_iter).fit(X)
        out.update({f"{name}_points": X, f"{name}_bandwidth": r, f"{name}_max_iter": max_iter, f"{name}_idx_array": idx,
                    f"{name}_seed_means": np.array([s[0] for s in seeds]), f"{name}_seed_counts": np.array([s[1] for s in seeds]),
                    f"{name}_seed_iters": np.array([s[2] for s in seeds]), f"{name}_cluster_centers": ms.cluster_centers_,
                    f"{name}_labels": ms.labels_, f"{name}_n_iter": ms.n_iter_})
        print(name, X.shape, "centres", len(ms.cluster_centers_), "n_iter", ms.n_iter_)
    np.savez_compressed(os.path.join(os.path.dirname(os.path.abspath(__file__)), "ref_sklearn_meanshift.npz"), **out)


if __name__ == "__main__":
    main()
