"""CPU: the restatement of scikit-learn's KDTree build (oracle_kdtree) against live scikit-learn and the committed fixture,
the counting partition the device uses against the sequential Hoare partition, the host pieces of the device build (node
count, radius, the restore from arrays, the state-layout check) and the code generation of csrc/kdtree_build.cu."""
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle_kdtree import oracle  # noqa: E402
from toothgroupnetwork_b200 import _lib as L  # noqa: E402
from toothgroupnetwork_b200 import build, neighbors  # noqa: E402

SkKDTree = pytest.importorskip("sklearn.neighbors").KDTree
FIX = np.load(os.path.join(ROOT, "tests", "golden", "ref_sklearn_kdtree.npz"))
FIX_NAMES = sorted({k[:-len("_points")] for k in FIX.files if k.endswith("_points")})


def assert_same_tree(got, want):
    """(idx_array, node_data, node_bounds) bit for bit"""
    idx, nodes, bounds = got
    w_idx, w_nodes, w_bounds = want
    assert np.array_equal(np.asarray(idx, np.int64), np.asarray(w_idx, np.int64))
    assert np.ascontiguousarray(nodes).tobytes() == np.ascontiguousarray(w_nodes).tobytes()
    assert bounds.shape == w_bounds.shape and bounds.tobytes() == w_bounds.tobytes()


@pytest.mark.parametrize("leaf_size", oracle.LEAF_SIZES)
def test_oracle_equals_live_sklearn(leaf_size):
    cases = [c for c in oracle.cases() if c[2] == leaf_size]
    assert {X.shape[0] for _, X, _ in cases} >= {1, 2, 3, 11, 12, 13, leaf_size + 1, 4 * leaf_size - 1}
    for name, X, ls in cases:
        try:
            assert_same_tree(oracle.build(X, ls), SkKDTree(X, leaf_size=ls).get_arrays()[1:])
        except AssertionError as e:
            raise AssertionError(name) from e


def test_depth_limit_input_takes_heap_select_and_equals_sklearn():
    for n, leaf_size in ((200, 2), (1000, 40), (2001, 30)):
        X = np.zeros((n, 3))
        X[:, 0] = oracle.killer_adversary(n)
        X[:, 2] = np.arange(n) % 5 * 1e-9                   # x keeps the widest spread, so the root splits on it
        stats = oracle.Stats()
        got = oracle.build(X, leaf_size, stats)
        assert stats.heap_selects >= 1
        assert_same_tree(got, SkKDTree(X, leaf_size=leaf_size).get_arrays()[1:])
    stats = oracle.Stats()
    oracle.build(oracle.cloud("normal", 2001, 0), 30, stats)
    assert stats.heap_selects == 0 and stats.partitions > 0


@pytest.mark.parametrize("name", FIX_NAMES)
def test_fixture_equals_oracle(name):
    X, leaf_size = FIX[f"{name}_points"], int(FIX[f"{name}_leaf_size"])
    want = (FIX[f"{name}_idx_array"], FIX[f"{name}_node_data"], FIX[f"{name}_node_bounds"])
    idx, nodes, bounds = oracle.build(X, leaf_size)
    assert_same_tree((idx, np.ascontiguousarray(nodes).view(np.int64).reshape(-1, 4), bounds), want)


def test_fixture_holds_the_depth_limit_case():
    assert any(name.startswith("killer") for name in FIX_NAMES)


def test_counting_partition_equals_hoare_partition():
    """the device's count / prefix / scatter against the sequential __unguarded_partition, after the same median of three"""
    rng = np.random.default_rng(5)
    for trial in range(300):
        n = int(rng.integers(4, 300))
        keys = rng.integers(0, int(rng.integers(1, 50)), n).astype(np.float64)
        ids = rng.permutation(n)
        comp = lambda a, b: a[1] < b[1] if a[0] == b[0] else a[0] < b[0]
        v = list(zip(keys.tolist(), ids.tolist()))
        oracle._move_median_to_first(v, 0, 1, n // 2, n - 1, comp)
        k2, i2 = np.array([a for a, _ in v]), np.array([b for _, b in v])
        cut = oracle._unguarded_partition(v, 1, n, 0, comp)
        got_cut = oracle.partition_by_counting(k2, i2, 0, n)
        assert got_cut == cut
        assert np.array_equal(k2, [a for a, _ in v]) and np.array_equal(i2, [b for _, b in v])


def test_node_count_is_sklearns_float_expression():
    lib = L.load()
    for leaf_size in (1, 2, 3, 7, 30, 40, 1000):
        for n in list(range(1, 300)) + [leaf_size * 2 ** j + d for j in range(18) for d in (-1, 0, 1)] + [2 ** 30]:
            if 1 <= n <= 2 ** 30:
                want = oracle.tree_shape(n, leaf_size)[1]
                assert neighbors.tree_nodes(n, leaf_size) == want
                assert lib.tgn_kdtree_nodes(n, leaf_size) == want, (n, leaf_size)
    assert lib.tgn_kdtree_nodes(0, 2) == -1 and lib.tgn_kdtree_nodes(5, 0) == -1


def test_host_radius_equals_sklearn():
    """the C library's pow over the bounds, as init_node computes it, on nodes whose squares and square roots are not exact"""
    rng = np.random.default_rng(6)
    naive_differs = 0
    for X, leaf_size in ((rng.standard_normal((20000, 3)), 2), (rng.random((3000, 3)) * 1e3, 1), (oracle.cloud("far", 999, 1), 30)):
        _, _, node_data, bounds = SkKDTree(X, leaf_size=leaf_size).get_arrays()
        mine = np.ascontiguousarray(node_data).copy()
        mine["radius"] = np.nan
        neighbors._fill_radius(mine.view(np.int64).reshape(-1, 4), np.ascontiguousarray(bounds))
        assert mine.tobytes() == np.ascontiguousarray(node_data).tobytes()
        half = 0.5 * np.abs(bounds[1] - bounds[0])
        naive_differs += int((np.sqrt((half[:, 0] * half[:, 0] + half[:, 1] * half[:, 1]) + half[:, 2] * half[:, 2])
                              != node_data["radius"]).sum())
    assert naive_differs > 0          # a correctly rounded sqrt of correctly rounded squares is not scikit-learn's radius


def test_restored_tree_answers_like_the_built_one():
    """a KDTree restored by __setstate__ from get_arrays() (the fallback's path, here with the oracle's arrays) queries
    bitwise like scikit-learn's built tree, ties included"""
    cls = neighbors.host_kdtree_class()
    assert neighbors._state_layout_ok(cls)
    rng = np.random.default_rng(7)
    X = oracle.cloud("duplicates", 3000, 8)
    X[:400] = np.round(X[:400] * 4) / 4
    Q = np.concatenate([X[rng.choice(3000, 1000)], np.round(rng.standard_normal((1000, 3)) * 4) / 4 + 0.125])
    for leaf_size in (2, 40):
        idx, nodes, bounds = oracle.build(X, leaf_size)
        tree = neighbors.restore(cls, X, idx.astype(np.intp), nodes, bounds, leaf_size)
        ref = SkKDTree(X, leaf_size=leaf_size)
        for k in (1, 5):
            d, i = tree.query(Q, k=k)
            wd, wi = ref.query(Q, k=k)
            assert np.array_equal(i, wi) and d.tobytes() == wd.tobytes()
        assert_same_tree(tree.get_arrays()[1:], ref.get_arrays()[1:])


def test_unexpected_state_layout_is_detected(monkeypatch):
    class Other:
        def __getstate__(self):
            return (np.zeros((1, 1)), np.zeros(1, np.intp))
    monkeypatch.setattr(neighbors, "_state_ok", None)
    assert not neighbors._state_layout_ok(Other)
    monkeypatch.setattr(neighbors, "_state_ok", None)
    assert neighbors._state_layout_ok(SkKDTree)


def test_build_is_declared():
    with open(os.path.join(ROOT, "include", "tgn_b200.h")) as f:
        header = " ".join(f.read().split())
    assert ("int tgn_kdtree_build(int n, int leaf_size, const double *xyz, long long *idx_array, long long *node_data, "
            "double *node_bounds, void *workspace, void *stream);") in header
    assert "size_t tgn_kdtree_bytes(int n, int leaf_size);" in header
    assert "kdtree_build.cu" in build.SOURCES
    assert {"tgn_kdtree_build", "tgn_kdtree_bytes", "tgn_kdtree_radius", "tgn_kdtree_nodes"} <= set(L.EXPORTS)


def test_build_kernel_does_not_spill():
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    out = os.path.join(os.environ.get("TMPDIR", "/tmp"), f"kdtree_build_{os.getpid()}.o")
    cmd = [nvcc] + build.NVCC_FLAGS + ["-Xptxas", "-v", "-c", os.path.join(build.CSRC, "kdtree_build.cu"), "-o", out]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if os.path.exists(out):
        os.remove(out)
    assert res.returncode == 0, res.stdout + res.stderr
    current, seen = None, {}
    for line in (res.stdout + res.stderr).splitlines():
        m = re.search(r"Compiling entry function '(\w+)'", line)
        if m:
            current = m.group(1) if "kdtree_level_kernel" in m.group(1) else None
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and current:
            seen[current] = m.groups()
    assert len(seen) == 1, seen
    assert all(v[1:] == ("0", "0") for v in seen.values()), seen
