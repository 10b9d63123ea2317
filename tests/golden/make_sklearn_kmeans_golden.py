"""Writes tests/golden/ref_sklearn_kmeans.npz: scikit-learn's own KMeans(k, init="k-means++", random_state=seed).fit on float32
(n, 3) inputs, single-threaded (threadpool_limits(1)), for tests/test_cpu_kmeans.py and tests/test_gpu_kmeans.py.

    python tests/golden/make_sklearn_kmeans_golden.py

Per case ``<name>_``: points, k, seed, labels, init (the kmeans_plusplus indices of the centred points), centers, n_iter,
inertia, and the legacy generator state after the fit (state_keys, state_pos) of ``np.random.seed(seed)`` + ``random_state=None``.
"""
import os
import sys
import warnings

import numpy as np
from threadpoolctl import threadpool_limits
from sklearn.cluster import KMeans, kmeans_plusplus

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from toothgroupnetwork_b200 import clouds  # noqa: E402


def blobs(n, k, sigma, seed, shift=0.0):
    r = np.random.default_rng(seed)
    c = r.uniform(-0.6, 0.6, (k, 3))
    return (c[r.integers(0, k, n)] + r.normal(0, sigma, (n, 3)) + shift).astype(np.float32)


def cases():
    yield "tight", blobs(14400, 16, 0.015, 1), 16, 3
    yield "loose", blobs(9000, 16, 0.05, 2), 17, 4
    yield "arch", clouds.dental_arch(12000, 3)[0].numpy().astype(np.float32), 15, 5
    twice = blobs(3000, 8, 0.02, 4)
    yield "twice", np.concatenate([twice, twice]), 8, 6
    yield "far", blobs(5000, 12, 0.02, 5, shift=np.array([120.0, -80.0, 45.0])), 12, 7
    yield "k1", blobs(700, 3, 0.03, 6), 1, 8
    yield "n_eq_k", blobs(9, 3, 0.1, 7), 9, 9
    few = blobs(4, 4, 0.2, 8)                       # 4 distinct points, k = 6: clusters empty and scikit-learn relocates them
    yield "few_distinct", few[np.random.default_rng(8).integers(0, 4, 300)], 6, 10


def main():
    out = {}
    warnings.simplefilter("ignore")
    with threadpool_limits(1):
        for name, X, k, seed in cases():
            np.random.seed(seed)
            km = KMeans(k, init="k-means++").fit(X)
            state = np.random.get_state()
            _, init = kmeans_plusplus(X - X.mean(axis=0), k, random_state=np.random.RandomState(seed))
            out.update({f"{name}_points": X, f"{name}_k": k, f"{name}_seed": seed, f"{name}_labels": km.labels_,
                        f"{name}_init": init, f"{name}_centers": km.cluster_centers_, f"{name}_n_iter": km.n_iter_,
                        f"{name}_inertia": np.float32(km.inertia_), f"{name}_state_keys": state[1], f"{name}_state_pos": state[2]})
            print(name, X.shape, k, "n_iter", km.n_iter_, "distinct", len(set(km.labels_)))
    np.savez_compressed(os.path.join(os.path.dirname(os.path.abspath(__file__)), "ref_sklearn_kmeans.npz"), **out)


if __name__ == "__main__":
    main()
