"""csrc/kmeans.cu against the numpy restatement (bitwise) and clustering.KMeans against live scikit-learn (single-threaded)."""
import os
import sys
import types
import warnings

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle_kmeans import oracle  # noqa: E402
from toothgroupnetwork_b200 import clouds, clustering  # noqa: E402

pytestmark = pytest.mark.gpu
sklearn_cluster = pytest.importorskip("sklearn.cluster")
threadpoolctl = pytest.importorskip("threadpoolctl")

from test_cpu_kmeans import skylakex_blas  # noqa: E402

live_sklearn = pytest.mark.skipif(not skylakex_blas(), reason="equal to scikit-learn where its OpenBLAS runs the SkylakeX kernels")
FIX = np.load(os.path.join(ROOT, "tests", "golden", "ref_sklearn_kmeans.npz"))
NAMES = sorted({k[:-len("_points")] for k in FIX.files if k.endswith("_points")})


def device_fits(prepared, k):
    """one launch for all prepared fits (oracle.prepare outputs) -> per fit dicts"""
    Xs = [p[0] for p in prepared]
    offs = np.concatenate([[0], np.cumsum([len(x) for x in Xs])]).astype(np.int32)
    T = 2 + int(np.log(k))
    u = np.stack([p[4].reshape(k - 1, T) for p in prepared])
    out = clustering.kmeans_device(torch.from_numpy(np.concatenate(Xs)).cuda(), torch.from_numpy(offs).cuda(), k,
                                   torch.tensor([p[3] for p in prepared], dtype=torch.int32).cuda(), torch.from_numpy(u).cuda(),
                                   torch.tensor([p[2] for p in prepared], dtype=torch.float32).cuda())
    labels, init, centres, n_iter, inertia, relocated = [t.cpu().numpy() for t in out]
    return [dict(labels=labels[offs[f]:offs[f + 1]], init=init[f], centers=centres[f], n_iter=int(n_iter[f]), inertia=inertia[f],
                 relocated=bool(relocated[f])) for f in range(len(prepared))]


def assert_same(got, want):
    assert got["relocated"] == want["relocated"]
    if want["relocated"]:
        return
    assert np.array_equal(got["labels"], want["labels"])
    assert np.array_equal(got["init"], want["init"])
    assert got["n_iter"] == want["n_iter"]
    assert np.array_equal(got["centers"].view(np.int32), want["centers"].view(np.int32))
    assert got["inertia"].view(np.int32) == np.float32(want["inertia"]).view(np.int32)


@pytest.mark.parametrize("name", NAMES)
def test_kernel_equals_oracle_on_fixtures(name):
    X, k, seed = FIX[f"{name}_points"], int(FIX[f"{name}_k"]), int(FIX[f"{name}_seed"])
    p = oracle.prepare(X, k, np.random.RandomState(seed))
    assert_same(device_fits([p], k)[0], oracle.fit(p[0], p[3], p[4], p[2]))


@pytest.mark.parametrize("seed", range(12))
def test_kernel_equals_oracle_on_random_shapes(seed):
    rng = np.random.default_rng(100 + seed)
    n = int(rng.choice([1, 2, 7, 33, 257, 4096, 4100, 9001, 15000, 24000]))
    k = int(min(n, rng.integers(1, 33)))
    fam = seed % 3
    if fam == 0:
        X = rng.normal(0, 1, (n, 3))
    elif fam == 1:
        c = rng.uniform(-1, 1, (16, 3))
        X = c[rng.integers(0, 16, n)] + rng.normal(0, 0.03, (n, 3))
    else:
        X = clouds.dental_arch(max(n, 16), seed)[0].numpy()[:n]
    p = oracle.prepare(X.astype(np.float32), k, np.random.RandomState(seed))
    assert_same(device_fits([p], k)[0], oracle.fit(p[0], p[3], p[4], p[2]))


def test_kernel_batch_of_fits():
    rng = np.random.default_rng(7)
    k = 16
    prepared = []
    for f in range(6):
        n = int(rng.integers(k, 20000))
        c = rng.uniform(-1, 1, (18, 3))
        prepared.append(oracle.prepare((c[rng.integers(0, 18, n)] + rng.normal(0, 0.02, (n, 3))).astype(np.float32), k, np.random.RandomState(f)))
    for got, p in zip(device_fits(prepared, k), prepared):
        assert_same(got, oracle.fit(p[0], p[3], p[4], p[2]))


@live_sklearn
@pytest.mark.parametrize("name", [n for n in NAMES if n != "few_distinct"])
def test_class_equals_live_sklearn(name):
    X, k, seed = FIX[f"{name}_points"], int(FIX[f"{name}_k"]), int(FIX[f"{name}_seed"])
    with warnings.catch_warnings(), threadpoolctl.threadpool_limits(1):
        warnings.simplefilter("ignore")         # scikit-learn's ConvergenceWarning on inputs with fewer distinct points than k
        for s in (seed, seed + 1):
            np.random.seed(s)
            ref = sklearn_cluster.KMeans(k, init="k-means++").fit(X)
            want_state = np.random.get_state()
            np.random.seed(s)
            got = clustering.KMeans(k, init="k-means++").fit(X)
            state = np.random.get_state()
            assert np.array_equal(got.labels_, ref.labels_)
            assert np.array_equal(got.cluster_centers_, ref.cluster_centers_) and got.n_iter_ == ref.n_iter_
            assert np.array_equal(state[1], want_state[1]) and state[2] == want_state[2]
            got = clustering.KMeans(k, random_state=s).fit(X)
            assert np.array_equal(got.labels_, sklearn_cluster.KMeans(k, random_state=s).fit(X).labels_)


@live_sklearn
def test_relocation_goes_to_scikit_learn():
    X, k, seed = FIX["few_distinct_points"], int(FIX["few_distinct_k"]), int(FIX["few_distinct_seed"])
    before = clustering.KMeans.host_fits
    with warnings.catch_warnings(), threadpoolctl.threadpool_limits(1):
        warnings.simplefilter("ignore")         # scikit-learn warns that it found fewer distinct clusters than k
        np.random.seed(seed)
        got = clustering.KMeans(k).fit(X)
        state = np.random.get_state()
    assert clustering.KMeans.host_fits == before + 1
    assert np.array_equal(got.labels_, FIX["few_distinct_labels"]) and got.n_iter_ == int(FIX["few_distinct_n_iter"])
    assert np.array_equal(state[1], FIX["few_distinct_state_keys"]) and state[2] == int(FIX["few_distinct_state_pos"])


@live_sklearn
def test_clustering_points_through_accelerate_kmeans():
    """ops_utils.clustering_points(method="kmeans") (ops_utils.py:30-34) with its KMeans name swapped gives the reference's labels"""
    def clustering_points(points, method="kmeans", num_of_clusters=16):
        if method == "kmeans":
            return mod.KMeans(num_of_clusters, init="k-means++").fit(points).labels_
    mod = types.SimpleNamespace(KMeans=sklearn_cluster.KMeans)
    X = FIX["tight_points"]
    with threadpoolctl.threadpool_limits(1):
        np.random.seed(0)
        want = clustering_points(X)
        clustering.accelerate_kmeans(mod)
        np.random.seed(0)
        got = clustering_points(X)
    assert mod.KMeans is clustering.KMeans and np.array_equal(got, want)
