"""MeanShift without a GPU: the numpy restatement (oracle_meanshift) against scikit-learn's fixtures and live scikit-learn, the
three pinned rules of the seed ascent, the class's host steps and refusals, and the kernel's ptxas report."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle_meanshift import oracle  # noqa: E402
from toothgroupnetwork_b200 import _lib, clustering  # noqa: E402

FIX = np.load(os.path.join(ROOT, "tests", "golden", "ref_sklearn_meanshift.npz"))
NAMES = sorted({k[:-len("_points")] for k in FIX.files if k.endswith("_points")})
CHEAP = ["duplicates", "max_iter_2", "small", "signed_zeros"]       # the cases live scikit-learn fits in a few seconds


def case(name):
    f = lambda key: FIX[f"{name}_{key}"]  # noqa: E731
    return f("points"), f("idx_array"), float(f("bandwidth")), int(f("max_iter")), f


def bits(a):
    return np.asarray(a, np.float64).view(np.int64)


def skylakex_blas() -> bool:
    """np.linalg.norm's order was pinned where numpy's OpenBLAS runs its SkylakeX ddot kernel (AVX-512 Intel hosts)"""
    from threadpoolctl import threadpool_info
    import numpy.linalg  # noqa: F401  (loads numpy's OpenBLAS)
    archs = {i.get("architecture") for i in threadpool_info() if i.get("internal_api") == "openblas"}
    return bool(archs) and archs <= {"SkylakeX", "SapphireRapids"}


@pytest.mark.parametrize("name", NAMES)
def test_oracle_equals_sklearn_fixture(name):
    X, idx, r, max_iter, f = case(name)
    means, counts, iters, flags = oracle.ascent(X, idx, r, max_iter)
    assert not flags.any()
    assert np.array_equal(bits(means), bits(f("seed_means")))
    assert np.array_equal(counts, f("seed_counts")) and np.array_equal(iters, f("seed_iters"))
    centers, labels, n_iter = oracle.postprocess(X, means, counts, iters, r)
    assert np.array_equal(bits(centers), bits(f("cluster_centers")))
    assert np.array_equal(labels, f("labels")) and n_iter == int(f("n_iter"))


@pytest.mark.parametrize("name", NAMES)
def test_class_postprocessing_of_the_restatement_equals_the_fit(name):
    """clustering.meanshift_postprocess (scikit-learn's calls) fed the restatement's seeds gives the fixture's fit"""
    pytest.importorskip("sklearn")
    X, idx, r, max_iter, f = case(name)
    means, counts, iters, _ = oracle.ascent(X, idx, r, max_iter)
    centers, labels, n_iter = clustering.meanshift_postprocess(X, means, counts, iters, r)
    assert np.array_equal(bits(centers), bits(f("cluster_centers")))
    assert np.array_equal(labels, f("labels")) and n_iter == int(f("n_iter"))


@pytest.mark.parametrize("name", CHEAP)
def test_oracle_equals_live_sklearn(name):
    sk = pytest.importorskip("sklearn.cluster")
    X, idx, r, max_iter, _ = case(name)
    ref = sk.MeanShift(bandwidth=r, max_iter=max_iter).fit(X)
    means, counts, iters, _ = oracle.ascent(X, clustering.meanshift_tree(X)[1], r, max_iter)
    centers, labels, n_iter = oracle.postprocess(X, means, counts, iters, r)
    assert np.array_equal(bits(centers), bits(ref.cluster_centers_))
    assert np.array_equal(labels, ref.labels_) and n_iter == ref.n_iter_


@pytest.mark.parametrize("name", ["two_teeth", "arch", "signed_zeros"])
def test_tree_arrays_are_the_fit_s_tree(name):
    """KDTree(X, 30), whose arrays the kernel walks, is the tree NearestNeighbors(radius=r).fit(X) builds inside MeanShift.fit"""
    neighbors = pytest.importorskip("sklearn.neighbors")
    X, idx, r, _, _ = case(name)
    nn = neighbors.NearestNeighbors(radius=r, n_jobs=1).fit(X)
    assert nn._fit_method == "kd_tree"
    want = nn._tree.get_arrays()
    got = neighbors.KDTree(X, leaf_size=30).get_arrays()
    for a, b in zip(got, want):
        assert np.array_equal(a, b)
    Xt, gidx, nodes, bounds = clustering.meanshift_tree(X)
    assert np.array_equal(gidx, idx) and np.array_equal(Xt, X[idx]) and np.array_equal(bounds, want[3])
    assert np.array_equal(nodes[:, 0], want[2]["idx_start"]) and np.array_equal(nodes[:, 1], want[2]["idx_end"])
    assert np.array_equal(nodes[:, 2], want[2]["is_leaf"])


@pytest.mark.parametrize("name", ["two_teeth", "arch", "planar", "signed_zeros"])
def test_membership_order_and_mean_chain_against_sklearn(name):
    """rules 1 and 2: radius_neighbors returns {(((0 + dx*dx) + dy*dy) + dz*dz) <= r*r} in ascending tree position, and
    np.mean(axis=0) of those rows is their sequential chain divided by the count"""
    neighbors = pytest.importorskip("sklearn.neighbors")
    X, idx, r, _, _ = case(name)
    nn = neighbors.NearestNeighbors(radius=r, n_jobs=1).fit(X)
    pos = np.empty(len(X), np.int64)
    pos[idx] = np.arange(len(X))
    rng = np.random.default_rng(len(X))
    queries = X[rng.integers(0, len(X), 300)] + rng.normal(0, r / 2, (300, 3))
    for q in queries:
        got = nn.radius_neighbors([q], r, return_distance=False)[0]
        d = q - X
        rd = ((0.0 + d[:, 0] * d[:, 0]) + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
        want = np.flatnonzero(rd <= r * r)
        assert np.array_equal(got, want[np.argsort(pos[want])])
        if len(got):
            assert np.array_equal(bits(np.mean(X[got], axis=0)), bits(np.add.accumulate(X[got], axis=0)[-1] / len(got)))


@pytest.mark.skipif(not skylakex_blas(), reason="the pinned order is that of OpenBLAS's SkylakeX ddot kernel")
def test_norm_order_against_numpy():
    """rule 3: np.linalg.norm of a 3-vector is sqrt(fma(dz,dz, fma(dy,dy, dx*dx)))"""
    rng = np.random.default_rng(0)
    for _ in range(20000):
        new, old = rng.normal(0, 1e-3, 3) * rng.random(), rng.normal(0, 1e-3, 3) * rng.random()
        assert np.sqrt(oracle.step_sq(new, old)) == np.linalg.norm(new - old)


@pytest.mark.parametrize("name", ["two_teeth", "planar"])
def test_host_seed_equals_sklearn_single_seed(name):
    """the re-run of a flagged seed (scikit-learn's public calls) returns _mean_shift_single_seed's values"""
    neighbors = pytest.importorskip("sklearn.neighbors")
    X, _, r, max_iter, f = case(name)
    nn = neighbors.NearestNeighbors(radius=r, n_jobs=1).fit(X)
    for i in np.random.default_rng(1).integers(0, len(X), 40):
        mean, count, it = clustering.meanshift_seed_host(X, X[i], nn, r, max_iter)
        assert np.array_equal(bits(mean), bits(f("seed_means")[i]))
        assert count == f("seed_counts")[i] and it == f("seed_iters")[i]


def test_lattice_at_the_bandwidth_is_flagged():
    """on a lattice with spacing equal to the bandwidth, reduced distances equal r^2 exactly: the restatement flags those seeds"""
    lat = np.stack(np.meshgrid(*[np.arange(4) * 0.5] * 3, indexing="ij"), -1).reshape(-1, 3)
    _, idx, _, _ = clustering.meanshift_tree(lat)
    flags = oracle.ascent(lat, idx, 0.5)[3]
    assert flags.any()


def test_sklearn_defaults_are_accepted():
    ms = clustering.MeanShift(0.07, seeds=None, bin_seeding=False, min_bin_freq=1, cluster_all=True, n_jobs=None, max_iter=300)
    assert ms.bandwidth == 0.07 and ms.max_iter == 300
    assert clustering.MeanShift(bandwidth=1, max_iter=0).max_iter == 0


@pytest.mark.parametrize("kwargs", [dict(bandwidth=None), dict(seeds=np.zeros((2, 3))), dict(bin_seeding=True), dict(min_bin_freq=3),
                                    dict(cluster_all=False), dict(bandwidth=-1.0), dict(bandwidth=float("nan")), dict(max_iter=-1)])
def test_unsupported_arguments_are_refused(kwargs):
    kwargs = {"bandwidth": 0.07, **kwargs}
    with pytest.raises(_lib.TgnError):
        clustering.MeanShift(**kwargs)


def test_unsupported_inputs_are_refused():
    pytest.importorskip("sklearn")
    ms = clustering.MeanShift(0.07)
    with pytest.raises(_lib.TgnError):
        ms.fit(np.zeros((40, 3), np.float32))
    with pytest.raises(_lib.TgnError):
        ms.fit(np.zeros((40, 2), np.float64))
    with pytest.raises(_lib.TgnError):
        ms.fit(np.zeros((40, 3), np.int64))
    for bad in (np.nan, np.inf):
        X = np.zeros((40, 3))
        X[3, 1] = bad
        with pytest.raises(ValueError):
            ms.fit(X)
    with pytest.raises(ValueError):
        ms.fit(np.zeros((0, 3)))


def test_small_inputs_go_to_sklearn_whole():
    sk = pytest.importorskip("sklearn.cluster")
    X = np.random.default_rng(4).normal(0, 0.05, (11, 3))
    before = clustering.MeanShift.host_fits
    got = clustering.MeanShift(0.07).fit(X)
    ref = sk.MeanShift(bandwidth=0.07).fit(X)
    assert clustering.MeanShift.host_fits == before + 1
    assert np.array_equal(bits(got.cluster_centers_), bits(ref.cluster_centers_))
    assert np.array_equal(got.labels_, ref.labels_) and got.n_iter_ == ref.n_iter_


def test_meanshift_kernel_has_no_spills():
    src = os.path.join(ROOT, "toothgroupnetwork_b200", "csrc", "meanshift.cu")
    from toothgroupnetwork_b200 import build
    res = subprocess.run([build._nvcc()] + build.NVCC_FLAGS + ["-Xptxas", "-v", "-c", src, "-o", os.devnull], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    report = res.stderr
    assert "meanshift_kernel" in report
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", report)
    assert spills and all(s == ("0", "0") for s in spills), report
