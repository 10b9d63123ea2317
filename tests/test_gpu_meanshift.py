"""csrc/meanshift.cu against the numpy restatement (bitwise, per seed) and clustering.MeanShift / get_clustering_labels against
live scikit-learn and the reference's own function."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle_meanshift import oracle  # noqa: E402
from toothgroupnetwork_b200 import clouds, clustering  # noqa: E402

pytestmark = pytest.mark.gpu
sklearn_cluster = pytest.importorskip("sklearn.cluster")

FIX = np.load(os.path.join(ROOT, "tests", "golden", "ref_sklearn_meanshift.npz"))
NAMES = sorted({k[:-len("_points")] for k in FIX.files if k.endswith("_points")})


def bits(a):
    return np.asarray(a, np.float64).view(np.int64)


def device_seeds(X, r, max_iter=300):
    Xt, idx, nodes, bounds = clustering.meanshift_tree(X)
    dev = [torch.from_numpy(a).cuda() for a in (Xt, idx, nodes, bounds)]
    return clustering.meanshift_unpack(clustering.meanshift_device(*dev, r, max_iter).cpu().numpy())


def assert_equal_fit(got, ref):
    assert np.array_equal(bits(got.cluster_centers_), bits(ref.cluster_centers_))
    assert got.labels_.dtype == ref.labels_.dtype and np.array_equal(got.labels_, ref.labels_)
    assert got.n_iter_ == ref.n_iter_


@pytest.mark.parametrize("name", NAMES)
def test_kernel_equals_oracle_on_fixtures(name):
    X, idx, r, max_iter = FIX[f"{name}_points"], FIX[f"{name}_idx_array"], float(FIX[f"{name}_bandwidth"]), int(FIX[f"{name}_max_iter"])
    means, counts, iters, flags = device_seeds(X, r, max_iter)
    w_means, w_counts, w_iters, w_flags = oracle.ascent(X, idx, r, max_iter)
    assert not flags.any() and np.array_equal(flags, w_flags)
    assert np.array_equal(bits(means), bits(w_means)) and np.array_equal(bits(means), bits(FIX[f"{name}_seed_means"]))
    assert np.array_equal(counts, w_counts) and np.array_equal(iters, w_iters)
    before = clustering.MeanShift.host_seeds
    got = clustering.MeanShift(r, max_iter=max_iter).fit(X)
    assert clustering.MeanShift.host_seeds == before
    assert np.array_equal(bits(got.cluster_centers_), bits(FIX[f"{name}_cluster_centers"]))
    assert np.array_equal(got.labels_, FIX[f"{name}_labels"]) and got.n_iter_ == int(FIX[f"{name}_n_iter"])


@pytest.mark.parametrize("seed", range(4))
def test_class_equals_live_sklearn(seed):
    rng = np.random.default_rng(20 + seed)
    n = int(rng.choice([12, 40, 500, 1500]))
    centres = rng.uniform(-0.2, 0.2, (int(rng.integers(1, 6)), 3))
    X = centres[rng.integers(0, len(centres), n)] + rng.normal(0, 0.02 + 0.01 * seed, (n, 3))
    r = float(rng.choice([0.03, 0.07, 0.1]))
    before = clustering.MeanShift.host_seeds
    assert_equal_fit(clustering.MeanShift(bandwidth=r).fit(X), sklearn_cluster.MeanShift(bandwidth=r).fit(X))
    assert clustering.MeanShift.host_seeds == before


def test_lattice_at_the_bandwidth_goes_to_the_host_and_still_equals_sklearn():
    """spacing 0.5 = r: reduced distances equal r^2 exactly, where scikit-learn's node bounds decide; those seeds are flagged and
    redone on the host"""
    lat = np.stack(np.meshgrid(*[np.arange(5) * 0.5] * 3, indexing="ij"), -1).reshape(-1, 3)
    lat = lat[np.random.default_rng(0).permutation(len(lat))]
    _, idx, _, _ = clustering.meanshift_tree(lat)
    means, counts, iters, flags = device_seeds(lat, 0.5)
    w_means, w_counts, w_iters, w_flags = oracle.ascent(lat, idx, 0.5)
    assert flags.any() and np.array_equal(flags, w_flags)
    ok = ~flags
    assert np.array_equal(bits(means[ok]), bits(w_means[ok])) and np.array_equal(counts[ok], w_counts[ok])
    before = clustering.MeanShift.host_seeds
    got = clustering.MeanShift(bandwidth=0.5).fit(lat)
    assert clustering.MeanShift.host_seeds == before + int(flags.sum())
    assert_equal_fit(got, sklearn_cluster.MeanShift(bandwidth=0.5).fit(lat))


def merged_teeth_cloud(teeth=(6, 7, 8), sep=0.03, seed=2, n=24000, pull=0.93, jitter=0.003, outliers=0.01):
    """an arch whose adjacent ``teeth`` a partly trained network pulled to centroids ``sep`` apart on a line -- one elongated
    DBSCAN cluster -- with a few predictions gone astray (DBSCAN noise)"""
    xyz, _, label = clouds.dental_arch(n, seed)
    xyz, label = xyz.numpy(), label.numpy().astype(np.int64)
    label = np.where(label < 0, 0, label)
    cent = np.stack([xyz[label == c].mean(0) if (label == c).any() else np.zeros(3, np.float32) for c in range(int(label.max()) + 1)])
    d = cent[teeth[-1]] - cent[teeth[0]]
    d /= np.linalg.norm(d)
    mid = cent[list(teeth)].mean(0)
    for j, t in enumerate(teeth):
        cent[t] = mid + d * sep * (j - (len(teeth) - 1) / 2)
    rng = np.random.default_rng(seed)
    moved = (xyz + pull * (cent[label] - xyz) + rng.normal(0, jitter, xyz.shape)).astype(np.float32)
    stray = rng.random(len(moved)) < outliers
    moved[stray] += rng.normal(0, 0.08, (int(stray.sum()), 3)).astype(np.float32)
    return moved, label


def test_get_clustering_labels_splits_on_the_device(monkeypatch):
    """the whole of ops_utils.get_clustering_labels on a cloud whose merged teeth take the MeanShift branch, with scikit-learn's
    MeanShift made unusable for the device version"""
    from oracle import ref_models
    if ref_models.reference_root() is None:
        pytest.skip("reference checkout not staged")
    pts, label = merged_teeth_cloud()
    with ref_models.World("reference") as w:
        want = w.mod("ops_utils").get_clustering_labels(pts, label)
    assert (want >= 100).any()                                       # the split branch fired: its labels start at 100

    class Refused:
        def __init__(self, *a, **k):
            raise AssertionError("sklearn.cluster.MeanShift called")
    monkeypatch.setattr(sklearn_cluster, "MeanShift", Refused)
    fits = []
    real_fit = clustering.MeanShift.fit
    monkeypatch.setattr(clustering.MeanShift, "fit", lambda self, X, y=None: fits.append(len(X)) or real_fit(self, X, y))
    before = clustering.MeanShift.host_fits
    got = clustering.get_clustering_labels(pts, label)
    assert fits and clustering.MeanShift.host_fits == before
    assert got.dtype == want.dtype and np.array_equal(got, want)
