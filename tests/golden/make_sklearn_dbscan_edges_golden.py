"""Generate tests/golden/ref_sklearn_dbscan_edges.npz: ``sklearn.cluster.DBSCAN(eps, min_samples).fit(points)``'s ``labels_``
and ``core_sample_indices_`` on clouds whose eps sits within one ulp of a pair's distance.

scikit-learn's DBSCAN builds ``NearestNeighbors(radius=eps)`` with the default ``n_neighbors=5``, and ``algorithm="auto"`` then
searches by brute force when ``5 >= n // 2``, i.e. for n <= 11.  The brute-force path compares the expanded distance
|x|^2 - 2 x.y + |y|^2 (BLAS norms and a GEMM, in float64, clamped at 0) with eps^2; the KD tree of n >= 12 compares the direct
(dx^2 + dy^2) + dz^2.  At eps = a pair's distance +- 1 ulp the two disagree on some tiny clouds, never on larger ones.  Cases:

* ``repro``: four float32 points on which the two forms disagree at eps = 0.4909613419409203, min_samples = 2;
* ``tiny{k}``: 40 seeded clouds of 2-11 float32 points, eps one ulp either side of the direct distance of a random pair,
  min_samples = 2;
* ``small{k}``: the same recipe at 12-40 points;
* ``lattice8`` / ``lattice27``: the 2x2x2 and 3x3x3 lattices of step 1/8 at eps = 1/8 (the first shell exactly at eps).

The script prints how many tiny and small cases disagree with the direct form, so the fixture is known to hold some.

    python tests/golden/make_sklearn_dbscan_edges_golden.py
"""
import os
import sys

import numpy as np
import sklearn
from sklearn.cluster import DBSCAN

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from oracle import oracle as O  # noqa: E402

REPRO = np.array([[0.1257302165031433, -0.13210485875606537, 0.6404226422309875],
                  [0.10490011423826218, -0.5356693863868713, 0.3615950644016266],
                  [1.3040000200271606, 0.9470809698104858, -0.7037352323532104],
                  [-1.2654215097427368, -0.6232744455337524, 0.04132597893476486]], np.float32)
REPRO_EPS = 0.4909613419409203


def pair_eps(pts: np.ndarray, rng: np.random.Generator) -> float:
    """the direct float64 distance of a random pair, moved one ulp up or down"""
    i, j = rng.choice(len(pts), 2, replace=False)
    d = pts[i].astype(np.float64) - pts[j].astype(np.float64)
    dist = float(np.sqrt((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2]))
    return float(np.nextafter(dist, np.inf if rng.random() < 0.5 else 0.0))


def cases():
    yield "repro", REPRO, REPRO_EPS, 2
    for prefix, lo, hi, seed0 in (("tiny", 2, 12, 100), ("small", 12, 41, 200)):
        for k in range(40):
            rng = np.random.default_rng(seed0 + k)
            pts = rng.normal(size=(int(rng.integers(lo, hi)), 3)).astype(np.float32)
            yield f"{prefix}{k}", pts, pair_eps(pts, rng), 2
    for name, half in (("lattice8", None), ("lattice27", 1)):
        axis = np.arange(2) / 8.0 if half is None else np.arange(-half, half + 1) / 8.0
        pts = np.stack(np.meshgrid(axis, axis, axis, indexing="ij"), -1).reshape(-1, 3).astype(np.float32)
        pts = pts[np.random.default_rng(7).permutation(len(pts))]
        yield name, pts, 0.125, 4


def main():
    """one array per field, the cases concatenated: case k holds rows offsets[k]:offsets[k + 1] of points / labels / core"""
    names, pts_all, eps_all, ms_all, labels_all, core_all = [], [], [], [], [], []
    disagree = {"tiny": 0, "small": 0, "other": 0}
    for name, pts, eps, ms in cases():
        c = DBSCAN(eps=eps, min_samples=ms).fit(pts)
        core = np.zeros(len(pts), bool)
        core[c.core_sample_indices_] = True
        for column, value in zip((names, pts_all, eps_all, ms_all, labels_all, core_all),
                                 (name, pts, eps, ms, c.labels_.astype(np.int64), core)):
            column.append(value)
        direct = O.dbscan(pts, eps, ms)
        if not (np.array_equal(direct[0], c.labels_) and np.array_equal(direct[1], c.core_sample_indices_)):
            disagree[name.rstrip("0123456789") if name.startswith(("tiny", "small")) else "other"] += 1
    fix = {"sklearn_version": np.array(sklearn.__version__), "names": np.array(names),
           "offsets": np.cumsum([0] + [len(p) for p in pts_all]).astype(np.int64), "points": np.concatenate(pts_all),
           "eps": np.array(eps_all, np.float64), "min_samples": np.array(ms_all, np.int64),
           "labels": np.concatenate(labels_all), "core": np.concatenate(core_all)}
    out = os.path.join(HERE, "ref_sklearn_dbscan_edges.npz")
    np.savez_compressed(out, **fix)
    print(f"scikit-learn {sklearn.__version__}: {len(names)} cases; disagreements with the direct form: "
          f"tiny (2-11 points) {disagree['tiny']}/40, small (12-40 points) {disagree['small']}/40, others {disagree['other']}")
    print(out, os.path.getsize(out), "bytes")


if __name__ == "__main__":
    main()
