"""KMeans without a GPU: the numpy restatement (oracle_kmeans) against scikit-learn's fixtures, the class's draws and
refusals, and the kernel's ptxas report."""
import os
import re
import subprocess
import sys
import types

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle_kmeans import oracle  # noqa: E402
from toothgroupnetwork_b200 import _lib, clustering, dropin  # noqa: E402

FIX = np.load(os.path.join(ROOT, "tests", "golden", "ref_sklearn_kmeans.npz"))
NAMES = sorted({k[:-len("_points")] for k in FIX.files if k.endswith("_points")})
RELOCATING = {"few_distinct"}


def skylakex_blas() -> bool:
    """the restated sdot / sgemv orders are those of OpenBLAS's SkylakeX kernels, which numpy's OpenBLAS picks on AVX-512 Intel
    hosts (SkylakeX, and SapphireRapids, which reuses them)"""
    from threadpoolctl import threadpool_info
    archs = {i.get("architecture") for i in threadpool_info() if i.get("internal_api") == "openblas"}
    return bool(archs) and archs <= {"SkylakeX", "SapphireRapids"}


@pytest.mark.parametrize("name", NAMES)
def test_oracle_equals_sklearn_fixture(name):
    f = lambda key: FIX[f"{name}_{key}"]  # noqa: E731
    got = oracle.kmeans(f("points"), int(f("k")), np.random.RandomState(int(f("seed"))))
    if name in RELOCATING:
        assert got["relocated"]
        return
    assert not got["relocated"]
    assert np.array_equal(got["labels"], f("labels"))
    assert np.array_equal(got["init"], f("init"))
    assert got["n_iter"] == int(f("n_iter"))
    assert np.array_equal(got["centers"].view(np.int32), f("centers").view(np.int32))
    assert got["inertia"] == f("inertia")


@pytest.mark.parametrize("name", NAMES)
def test_draws_leave_the_generator_where_sklearn_does(name):
    np.random.seed(int(FIX[f"{name}_seed"]))
    oracle.prepare(FIX[f"{name}_points"], int(FIX[f"{name}_k"]), None)
    state = np.random.get_state()
    assert np.array_equal(state[1], FIX[f"{name}_state_keys"]) and state[2] == int(FIX[f"{name}_state_pos"])


@pytest.mark.skipif(not skylakex_blas(), reason="the pinned orders are those of OpenBLAS's SkylakeX kernels")
def test_blas_orders_against_numpy():
    """the restated sdot / sgemv orders are numpy's own matmul results (single-threaded), over the block edges"""
    from threadpoolctl import threadpool_limits
    rng = np.random.default_rng(0)
    with threadpool_limits(1):
        for n in (1, 3, 31, 32, 33, 63, 64, 65, 100, 4095, 4096, 4097, 4100, 8196, 9001, 24000):
            x = (rng.random((6, n)) ** 3).astype(np.float32)
            assert oracle.sdot_sum(x[0]) == (x[:1] @ np.ones(n, np.float32))[0]
            for T in range(2, 7):
                assert np.array_equal(oracle.sgemv_sum(x[:T]), (x[:T] @ np.ones((n, 1), np.float32))[:, 0])


@pytest.mark.parametrize("name", NAMES)
def test_class_preparation_leaves_the_generator_where_sklearn_does(name):
    """clustering.kmeans_prepare is the class's host step: its values equal the restatement's and, on numpy's global generator
    (random_state=None, as the pipeline calls it), it leaves the state scikit-learn's fit left"""
    X, k, seed = FIX[f"{name}_points"], int(FIX[f"{name}_k"]), int(FIX[f"{name}_seed"])
    np.random.seed(seed)
    got = clustering.kmeans_prepare(X, k, 1e-4, clustering._random_state(None))
    state = np.random.get_state()
    assert np.array_equal(state[1], FIX[f"{name}_state_keys"]) and state[2] == int(FIX[f"{name}_state_pos"])
    want = oracle.prepare(X, k, np.random.RandomState(seed))
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1]) and got[2] == want[2] and got[3] == want[3]
    assert np.array_equal(got[4], want[4])
    assert clustering._random_state(seed).get_state()[1][0] == np.random.RandomState(seed).get_state()[1][0]


def test_sklearn_defaults_are_accepted():
    km = clustering.KMeans(4, init="k-means++", n_init="auto", max_iter=300, tol=1e-4, verbose=0, random_state=None, copy_x=True,
                           algorithm="lloyd")
    assert km.n_clusters == 4


@pytest.mark.parametrize("kwargs", [dict(init="random"), dict(algorithm="elkan"), dict(n_init=3), dict(copy_x=False), dict(verbose=1)])
def test_unsupported_arguments_are_refused(kwargs):
    with pytest.raises(_lib.TgnError):
        clustering.KMeans(4, **kwargs)


def test_unsupported_inputs_are_refused():
    km = clustering.KMeans(2)
    with pytest.raises(_lib.TgnError):
        km.fit(np.zeros((10, 3), np.float64))
    with pytest.raises(_lib.TgnError):
        km.fit(np.zeros((10, 2), np.float32))
    with pytest.raises(_lib.TgnError):
        km.fit(np.zeros((10, 3), np.float32), sample_weight=np.ones(10))
    with pytest.raises(ValueError, match="should be >= n_clusters"):
        clustering.KMeans(5).fit(np.zeros((4, 3), np.float32))


def test_accelerate_kmeans_swaps_only_the_name():
    mod = types.SimpleNamespace(KMeans=object, DBSCAN=object)
    dropin.accelerate_kmeans(mod)
    assert mod.KMeans is clustering.KMeans and mod.DBSCAN is object


def test_kmeans_kernel_has_no_spills():
    src = os.path.join(ROOT, "toothgroupnetwork_b200", "csrc", "kmeans.cu")
    from toothgroupnetwork_b200 import build
    res = subprocess.run([build._nvcc()] + build.NVCC_FLAGS + ["-Xptxas", "-v", "-c", src, "-o", os.devnull], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    report = res.stderr
    assert "kmeans_kernel" in report
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", report)
    assert spills and all(s == ("0", "0") for s in spills), report
