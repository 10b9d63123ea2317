"""Writes tests/golden/ref_sklearn_kdtree.npz: scikit-learn 1.9's own ``KDTree(X, leaf_size).get_arrays()`` on a selection of
the clouds of oracle_kdtree.cases() and on one input that drives the introselect to its depth limit, for
tests/test_cpu_kdtree_build.py and tests/test_gpu_kdtree_build.py.

    python tests/golden/make_sklearn_kdtree_golden.py

Per case ``<name>_``: points (n,3) float64, leaf_size, idx_array int64, node_data (n_nodes, 4) int64 (NodeData_t's records,
the radius as its float64 bits) and node_bounds (2, n_nodes, 3) float64.
"""
import os
import sys

import numpy as np
from sklearn.neighbors import KDTree

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle_kdtree import oracle  # noqa: E402


def cases():
    for name, X, leaf_size in oracle.cases():
        n = X.shape[0]
        if n in (1, 13) or (leaf_size == 40 and n > 1200) or (leaf_size == 2 and 250 < n < 300):
            yield name, X, leaf_size
    X = np.zeros((1500, 3))
    X[:, 0] = oracle.killer_adversary(1500)
    X[:, 1] = np.arange(1500) % 7 * 1e-9
    yield "killer_n1500_leaf40", X, 40


def main():
    out = {}
    for name, X, leaf_size in cases():
        _, idx, node_data, bounds = KDTree(X, leaf_size=leaf_size).get_arrays()
        out[f"{name}_points"] = X
        out[f"{name}_leaf_size"] = np.int64(leaf_size)
        out[f"{name}_idx_array"] = idx.astype(np.int64)
        out[f"{name}_node_data"] = np.ascontiguousarray(node_data).view(np.int64).reshape(-1, 4)
        out[f"{name}_node_bounds"] = bounds
    path = os.path.join(ROOT, "tests", "golden", "ref_sklearn_kdtree.npz")
    np.savez_compressed(path, **out)
    print(path, len(out) // 5, "cases")


if __name__ == "__main__":
    main()
