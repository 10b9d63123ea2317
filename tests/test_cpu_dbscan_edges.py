"""CPU: the host side of DBSCAN at its edges.  Clouds of at most 11 points, which scikit-learn searches by brute force with an
expanded distance that can land on the other side of eps, are fitted by scikit-learn itself (pinned against its own choice of
search and against tests/golden/ref_sklearn_dbscan_edges.npz); non-finite coordinates are refused like scikit-learn refuses
them; and the premise of the lattice cases of test_gpu_dbscan_edges.py holds: on the 1/8 lattice every float64 distance and
eps^2 are exact."""
import itertools
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import oracle as O  # noqa: E402
from toothgroupnetwork_b200 import _lib as L  # noqa: E402
from toothgroupnetwork_b200 import clouds, clustering  # noqa: E402

FIXTURE = os.path.join(ROOT, "tests", "golden", "ref_sklearn_dbscan_edges.npz")


def fixture_cases():
    fix = np.load(FIXTURE)
    off = fix["offsets"]
    for k, name in enumerate(fix["names"].tolist()):
        sl = slice(off[k], off[k + 1])
        yield name, fix["points"][sl], float(fix["eps"][k]), int(fix["min_samples"][k]), fix["labels"][sl], np.flatnonzero(fix["core"][sl])


def test_brute_force_routing_is_scikit_learns_own():
    """DBSCAN's NearestNeighbors(radius=eps) (default n_neighbors=5, algorithm="auto") picks brute force for exactly the sizes
    that clustering.dbscan sends to the host"""
    neighbors = pytest.importorskip("sklearn.neighbors")
    for n in range(1, 41):
        X = np.random.default_rng(n).normal(size=(n, 3)).astype(np.float32)
        nn = neighbors.NearestNeighbors(radius=0.5).fit(X)
        if not hasattr(nn, "_fit_method"):
            pytest.skip("NearestNeighbors no longer exposes _fit_method")
        assert nn._fit_method == ("brute" if n <= clustering._BRUTE_MAX_N else "kd_tree"), n


def test_the_fixture_holds_brute_force_disagreements_and_none_from_12_points():
    """the direct predicate (oracle.dbscan, the kernel's) equals scikit-learn from 12 points on, and differs on some tiny clouds"""
    tiny_differ = 0
    for name, pts, eps, ms, labels, core in fixture_cases():
        o_labels, o_core = O.dbscan(pts, eps, ms)
        same = np.array_equal(o_labels, labels) and np.array_equal(o_core, core)
        if len(pts) >= 12:
            assert same, name
        else:
            tiny_differ += not same
        if name == "repro":
            assert labels.tolist() == [0, 0, -1, -1] and o_labels.tolist() == [-1, -1, -1, -1]
    assert tiny_differ >= 2


def test_tiny_fits_are_scikit_learns_without_a_gpu():
    pytest.importorskip("sklearn.cluster")
    seen = 0
    for name, pts, eps, ms, labels, core in fixture_cases():
        if len(pts) >= 12:
            continue
        before = clustering.DBSCAN.host_fits
        got = clustering.DBSCAN(eps=eps, min_samples=ms).fit(pts)
        assert clustering.DBSCAN.host_fits == before + 1
        assert np.array_equal(got.labels_, labels) and np.array_equal(got.core_sample_indices_, core), name
        assert np.array_equal(got.components_, pts[core])
        assert np.array_equal(clustering.DBSCAN(eps=eps, min_samples=ms).fit_predict(pts), labels)
        f_labels, f_core = clustering.dbscan(pts, eps, ms)
        assert f_labels.dtype == np.int64 and np.array_equal(f_labels, labels) and np.array_equal(f_core, core)
        import torch
        t_labels, t_core = clustering.dbscan(torch.from_numpy(pts), eps, ms)        # a CPU tensor takes the same route
        assert np.array_equal(t_labels, labels) and np.array_equal(t_core, core)
        seen += 1
    assert seen > 40


def test_tiny_fits_without_scikit_learn_raise(monkeypatch):
    monkeypatch.setitem(sys.modules, "sklearn.cluster", None)        # makes `from sklearn.cluster import ...` raise ImportError
    with pytest.raises(L.TgnError, match="scikit-learn"):
        clustering.dbscan(np.zeros((5, 3), np.float32), 0.1, 2)


@pytest.mark.parametrize("n", [5, 40])
@pytest.mark.parametrize("bad", [np.nan, np.inf, -np.inf])
def test_non_finite_coordinates_are_refused(n, bad):
    """scikit-learn's ValueError and the start of its message, before any device work (so also on a machine without a GPU)"""
    pts = np.random.default_rng(0).normal(size=(n, 3)).astype(np.float32)
    pts[n // 2, 1] = bad
    want = "^Input X contains NaN" if np.isnan(bad) else "^Input X contains infinity"
    for call in (lambda: clustering.dbscan(pts, 0.1, 3), lambda: clustering.DBSCAN(eps=0.1, min_samples=3).fit(pts),
                 lambda: clustering.DBSCAN(eps=0.1, min_samples=3).fit(pts.astype(np.float64)),
                 lambda: clustering.get_clustering_labels(pts, np.ones(n, np.int64))):
        with pytest.raises(ValueError, match=want):
            call()
    sk = pytest.importorskip("sklearn.cluster")
    with pytest.raises(ValueError, match=want):
        sk.DBSCAN(eps=0.1, min_samples=3).fit(pts)


def test_lattice_distances_and_eps_are_exact():
    """the lattice cases of test_gpu_dbscan_edges.py: points (i, j, l) / 8 with |i|, |j|, |l| <= 12.  Every coordinate is a float32
    value, every difference k / 8 (|k| <= 24) and its square are exact in float64, so (dx dx + dy dy) + dz dz is the exact
    (a^2 + b^2 + c^2) / 64; eps = 1/8, 1/4, 3/8 square exactly to 1/64, 4/64, 9/64; one ulp below eps squares below eps^2."""
    pts = clouds.lattice(12, seed=1).numpy()
    assert len(pts) == 25 ** 3 and np.array_equal(np.sort(np.unique(pts)), np.arange(-12, 13) / 8.0)
    k = np.array(list(itertools.product(range(-24, 25), repeat=3)))
    d = k / 8.0
    assert np.array_equal(d * 8.0, k.astype(np.float64))
    d2 = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
    assert np.array_equal(d2 * 64.0, (k * k).sum(1).astype(np.float64))
    # the differences of actual coordinates are those k / 8
    a, b = pts[:4000].astype(np.float64), pts[-4000:].astype(np.float64)
    assert np.array_equal((a - b) * 8.0, np.round((a - b) * 8.0))
    for e in (1, 2, 3):
        eps = e / 8.0
        assert eps * eps == e * e / 64.0
        below = float(np.nextafter(eps, 0.0))
        assert below * below < eps * eps
        # every squared lattice distance below eps^2 is below by at least 1/64: the shell at eps is the only one decided
        assert not ((d2 < eps * eps) & (d2 > below * below)).any() and ((d2 == eps * eps) & (d2 > below * below)).any()
