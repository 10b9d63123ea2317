"""CPU: the restatement of scikit-learn's KDTree.query (oracle_kdtree.oracle.query: depth-first walk, heap_push, the 2-way
introsort) against live scikit-learn; its exact-square arithmetic and flag rule, which csrc/kdtree_query.cu computes; the
declarations, the name swap of the label transfers and the code generation of the walk kernel."""
import math
import os
import re
import shutil
import subprocess
import sys
import types

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle_kdtree import oracle  # noqa: E402
from toothgroupnetwork_b200 import _lib as L  # noqa: E402
from toothgroupnetwork_b200 import build, dropin, neighbors  # noqa: E402

SkKDTree = pytest.importorskip("sklearn.neighbors").KDTree
sorting = pytest.importorskip("sklearn.utils._sorting")

KS = (1, 2, 3, 8, 15, 16, 17, 40, 63)             # 15 / 16 / 17 straddle the insertion-sort cut
INPUTS = list(oracle.tied_query_inputs(full=False))


def cases(k):
    """the tied inputs (queries thinned for the Python walk), n = k, and a single point"""
    for name, pts, q in INPUTS:
        yield name, pts, q[::3] if q.shape[0] > 400 else q
    pts = INPUTS[1][1]
    yield "n_equals_k", pts[:k], INPUTS[0][2][:60]
    if k == 1:
        yield "single_point", pts[:1], INPUTS[0][2][:20]


@pytest.mark.parametrize("leaf_size", oracle.LEAF_SIZES)
@pytest.mark.parametrize("k", KS)
def test_oracle_equals_sklearn_and_exact_squares_where_unflagged(k, leaf_size):
    for name, pts, q in cases(k):
        tree = SkKDTree(pts, leaf_size=leaf_size)
        _, idx, nodes, bounds = tree.get_arrays()
        wd, wi = tree.query(q, k=k)
        d, i, _ = oracle.query(pts, idx, nodes, bounds, q, k)
        assert np.array_equal(i, wi) and d.tobytes() == wd.tobytes(), name
        d, i, flag = oracle.query(pts, idx, nodes, bounds, q, k, square=oracle.exact_square)
        ok = flag == 0
        assert np.array_equal(i[ok], wi[ok]) and d[ok].tobytes() == wd[ok].tobytes(), name


def test_tied_inputs_tie():
    """the inputs exercise what they are for: rows whose two nearest distances are equal"""
    for name, pts, q in INPUTS:
        d, _ = SkKDTree(pts, leaf_size=2).query(q, k=2)
        assert int((d[:, 0] == d[:, 1]).sum()) > 20, name


def test_introsort_equals_sklearn_at_every_length():
    rng = np.random.default_rng(3)
    for n in range(1, 64):
        for trial in range(20):
            v = rng.integers(0, int(rng.integers(1, 8)), n).astype(np.float64)
            if trial % 2:
                v = v * 0.1 + rng.integers(0, 2, n) * 1e-3
            ind = rng.permutation(n).astype(np.intp)
            a, b = v.tolist(), ind.tolist()
            oracle.simultaneous_sort(a, b)
            sorting._py_simultaneous_sort(v, ind, n, use_three_way_partition=False)
            assert a == v.tolist() and b == ind.tolist(), (n, trial)


@pytest.mark.parametrize("n", [48, 63])
def test_introsort_depth_limit_takes_heapsort_and_equals_sklearn(n):
    v = oracle.sort_killer(n)
    v = np.floor(v / 2)                                   # pairs of equal values: the heapsort's order among them counts
    stats = oracle.SortStats()
    a, b = v.tolist(), list(range(n))
    oracle.simultaneous_sort(a, b, stats=stats)
    ind = np.arange(n, dtype=np.intp)
    sorting._py_simultaneous_sort(v, ind, n, use_three_way_partition=False)
    assert stats.heapsorts >= 1
    assert a == v.tolist() and b == ind.tolist()


def test_random_input_does_not_reach_the_depth_limit():
    stats = oracle.SortStats()
    oracle.simultaneous_sort(np.random.default_rng(1).random(63).tolist(), list(range(63)), stats=stats)
    assert stats.heapsorts == 0 and stats.partitions > 0


def test_heap_push_equals_sklearns_neighbors_heap():
    from sklearn.neighbors._kd_tree import NeighborsHeap64
    rng = np.random.default_rng(4)
    for size in (1, 2, 3, 8, 63):
        heap = NeighborsHeap64(1, size)
        values, indices = [math.inf] * size, [0] * size
        for i, val in enumerate(rng.integers(0, 12, 400).astype(np.float64).tolist()):
            heap.push(0, val, i)
            oracle.heap_push(values, indices, val, i)
        d, ind = heap.get_arrays(sort=False)
        assert d[0].tolist() == values and ind[0].tolist() == indices


def test_flag_rule_catches_where_pow_decides_otherwise():
    """on a seeded input found by search, the walk with the C library's pow and the walk with h*h take different trim
    decisions, and the rule flags every such row"""
    X, Q, leaf_size, k, rows = oracle.pow_decides_otherwise()
    _, idx, nodes, bounds = SkKDTree(X, leaf_size=leaf_size).get_arrays()
    q = Q[list(rows)]
    with_pow, with_square = [], []
    oracle.query(X, idx, nodes, bounds, q, k, trace=with_pow)
    _, _, flag = oracle.query(X, idx, nodes, bounds, q, k, square=oracle.exact_square, trace=with_square)
    assert all(a != b for a, b in zip(with_pow, with_square))
    assert flag.tolist() == [1] * len(rows)


def test_exact_square_test():
    assert oracle._is_exact(0.5, 0.25) and oracle._is_exact(3.0, 9.0) and oracle._is_exact(0.0, 0.0)
    assert not oracle._is_exact(0.1, 0.1 * 0.1)
    h = float(np.float32(0.3)) - float(np.float32(0.1))   # a difference of float32 values: 25 significant bits
    assert oracle._is_exact(h, h * h)


def test_query_is_declared():
    with open(os.path.join(ROOT, "include", "tgn_b200.h")) as f:
        header = " ".join(f.read().split())
    assert ("int tgn_kdtree_query(int n, int n_nodes, int k, const double *xyz, const long long *idx_array, "
            "const long long *node_data, const double *node_bounds, int m, const double *queries, const long long *rows, "
            "int n_rows, long long *idx, double *dist, unsigned char *flag, void *stream);") in header
    assert "kdtree_query.cu" in build.SOURCES
    assert "tgn_kdtree_query" in L.EXPORTS


def test_label_transfer_swap_chooses_the_tie_path():
    mod = types.SimpleNamespace(KDTree=SkKDTree)
    dropin.accelerate_label_transfer(mod, ties="device")
    assert mod.KDTree is neighbors.DeviceKDTree and issubclass(neighbors.DeviceKDTree, neighbors.KDTree)
    dropin.accelerate_label_transfer(mod)
    assert mod.KDTree is neighbors.KDTree
    with pytest.raises(ValueError):
        dropin.accelerate_label_transfer(mod, ties="gpu")
    assert mod.KDTree is neighbors.KDTree


def test_query_kernel_does_not_spill():
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    out = os.path.join(os.environ.get("TMPDIR", "/tmp"), f"kdtree_query_{os.getpid()}.o")
    cmd = [nvcc] + build.NVCC_FLAGS + ["-Xptxas", "-v", "-c", os.path.join(build.CSRC, "kdtree_query.cu"), "-o", out]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if os.path.exists(out):
        os.remove(out)
    assert res.returncode == 0, res.stdout + res.stderr
    current, seen = None, {}
    for line in (res.stdout + res.stderr).splitlines():
        m = re.search(r"Compiling entry function '(\w+)'", line)
        if m:
            current = m.group(1) if "kdtree_query_kernel" in m.group(1) else None
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and current:
            seen[current] = m.groups()
    assert len(seen) == 1, seen
    assert all(v[1:] == ("0", "0") for v in seen.values()), seen
