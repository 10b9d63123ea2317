"""oracle_kdtree/oracle.py -- Python restatement of scikit-learn 1.9's ``KDTree(X, leaf_size)`` build (TEST INFRASTRUCTURE ONLY).

``build(X, leaf_size)`` returns what ``KDTree(X, leaf_size).get_arrays()[1:]`` returns -- idx_array, node_data and
node_bounds -- computed step by step from scikit-learn's ``_binary_tree.pxi.tp`` and libstdc++'s ``std::nth_element``:

- ``n_levels`` / ``n_nodes``: scikit-learn's float expression, ``int(log2(fmax(1, (n - 1) / leaf_size)) + 1)``;
- ``_recursive_build``: ``init_node`` (bounds by ``fmin`` / ``fmax`` in idx_array order, radius by ``pow``), then for an
  inner node ``find_node_split_dim`` (the first dimension with the largest spread, strict ``>`` from 0) and
  ``partition_node_indices`` to the midpoint ``n_points / 2``;
- ``partition_node_indices`` is ``std::nth_element`` with the comparator ``(x[split], index)``: ``__introselect`` with the
  depth limit ``2 * floor(log2 n)``, ``__move_median_to_first``, ``__unguarded_partition``, ``__insertion_sort`` of the last
  <= 3 elements, and on the depth limit ``__heap_select`` + ``iter_swap``.

The compiled ``init_node`` keeps the running bound when a point equals it: ``fmin(lo, v) = v if v < lo else lo``.  So among
equal values (+0.0 and -0.0) the earlier element wins, and a bound's sign of zero is that of the first element equal to it
in the node's idx_array order (pinned against live scikit-learn by tests/test_cpu_kdtree_build.py).  ``stats`` records which branches a build took (for the depth-limit test).

Nothing under ``toothgroupnetwork_b200/`` may import it.
"""
from __future__ import annotations

import math

import numpy as np


def tree_shape(n: int, leaf_size: int):
    """(n_levels, n_nodes) with scikit-learn's float expression"""
    n_levels = int(np.log2(max(1.0, (n - 1) / leaf_size)) + 1)
    return n_levels, 2 ** n_levels - 1


def node_ranges(n: int, n_nodes: int):
    """idx_start, idx_end of every node: the root is [0, n), a node [s, e) splits at s + (e - s) // 2"""
    start = np.zeros(n_nodes, np.int64)
    end = np.zeros(n_nodes, np.int64)
    end[0] = n
    for i in range(n_nodes):
        if 2 * i + 1 < n_nodes:
            s, e = int(start[i]), int(end[i])
            m = s + (e - s) // 2
            start[2 * i + 1], end[2 * i + 1] = s, m
            start[2 * i + 2], end[2 * i + 2] = m, e
    return start, end


class Stats:
    def __init__(self):
        self.heap_selects = 0
        self.partitions = 0


def _move_median_to_first(v, result, a, b, c, comp):
    if comp(v[a], v[b]):
        if comp(v[b], v[c]):
            s = b
        elif comp(v[a], v[c]):
            s = c
        else:
            s = a
    elif comp(v[a], v[c]):
        s = a
    elif comp(v[b], v[c]):
        s = c
    else:
        s = b
    v[result], v[s] = v[s], v[result]


def _unguarded_partition(v, first, last, pivot, comp):
    while True:
        while comp(v[first], v[pivot]):
            first += 1
        last -= 1
        while comp(v[pivot], v[last]):
            last -= 1
        if not first < last:
            return first
        v[first], v[last] = v[last], v[first]
        first += 1


def _adjust_heap(v, first, hole, length, value, comp):
    top = hole
    second = hole
    while second < (length - 1) // 2:
        second = 2 * (second + 1)
        if comp(v[first + second], v[first + second - 1]):
            second -= 1
        v[first + hole] = v[first + second]
        hole = second
    if (length & 1) == 0 and second == (length - 2) // 2:
        second = 2 * (second + 1)
        v[first + hole] = v[first + second - 1]
        hole = second - 1
    parent = (hole - 1) // 2
    while hole > top and comp(v[first + parent], value):
        v[first + hole] = v[first + parent]
        hole = parent
        parent = (hole - 1) // 2
    v[first + hole] = value


def _heap_select(v, first, middle, last, comp):
    length = middle - first
    if length >= 2:                                   # __make_heap
        parent = (length - 2) // 2
        while True:
            _adjust_heap(v, first, parent, length, v[first + parent], comp)
            if parent == 0:
                break
            parent -= 1
    for i in range(middle, last):
        if comp(v[i], v[first]):                      # __pop_heap(first, middle, i)
            value = v[i]
            v[i] = v[first]
            _adjust_heap(v, first, 0, length, value, comp)


def _insertion_sort(v, first, last, comp):
    for i in range(first + 1, last):
        val = v[i]
        if comp(val, v[first]):
            v[first + 1:i + 1] = v[first:i]
            v[first] = val
        else:
            j = i
            while comp(val, v[j - 1]):
                v[j] = v[j - 1]
                j -= 1
            v[j] = val


def nth_element(v: list, first: int, nth: int, last: int, comp, stats: Stats | None = None) -> None:
    """libstdc++'s std::nth_element(v + first, v + nth, v + last, comp) on a Python list"""
    if first == last or nth == last:
        return
    depth = 2 * ((last - first).bit_length() - 1)
    while last - first > 3:
        if depth == 0:
            _heap_select(v, first, nth + 1, last, comp)
            v[first], v[nth] = v[nth], v[first]
            if stats is not None:
                stats.heap_selects += 1
            return
        depth -= 1
        mid = first + (last - first) // 2
        _move_median_to_first(v, first, first + 1, mid, last - 1, comp)
        cut = _unguarded_partition(v, first + 1, last, first, comp)
        if stats is not None:
            stats.partitions += 1
        if cut <= nth:
            first = cut
        else:
            last = cut
    _insertion_sort(v, first, last, comp)


def _fmin(a, b):
    return b if b < a else a


def _fmax(a, b):
    return b if b > a else a


def build(X, leaf_size: int, stats: Stats | None = None):
    """(idx_array int64 (n), node_data NodeData (n_nodes), node_bounds float64 (2, n_nodes, d)) of scikit-learn's KDTree"""
    X = np.ascontiguousarray(X, dtype=np.float64)
    n, d = X.shape
    n_levels, n_nodes = tree_shape(n, leaf_size)
    idx = list(range(n))
    node_data = np.zeros(n_nodes, dtype=[("idx_start", "<i8"), ("idx_end", "<i8"), ("is_leaf", "<i8"), ("radius", "<f8")])
    bounds = np.zeros((2, n_nodes, d), np.float64)
    cols = [X[:, j].tolist() for j in range(d)]
    p = 2.0

    def init_node(i, s, e):
        rad = 0.0
        for j in range(d):
            lo, hi = math.inf, -math.inf
            col = cols[j]
            for t in range(s, e):
                lo, hi = _fmin(lo, col[idx[t]]), _fmax(hi, col[idx[t]])
            bounds[0, i, j], bounds[1, i, j] = lo, hi
            rad += math.pow(0.5 * abs(hi - lo), p)
        node_data[i] = (s, e, 0, math.pow(rad, 1.0 / p))

    stack = [(0, 0, n)]
    while stack:
        i, s, e = stack.pop()
        init_node(i, s, e)
        if 2 * i + 1 >= n_nodes:
            node_data["is_leaf"][i] = 1
            continue
        if e - s < 2:
            raise AssertionError("scikit-learn allocates no node with fewer than 2 points")
        spread = [bounds[1, i, j] - bounds[0, i, j] for j in range(d)]
        j_max, best = 0, 0.0
        for j in range(d):
            if spread[j] > best:
                best, j_max = spread[j], j
        col = cols[j_max]
        comp = lambda a, b, col=col: a < b if col[a] == col[b] else col[a] < col[b]
        m = s + (e - s) // 2
        nth_element(idx, s, m, e, comp, stats)
        stack.append((2 * i + 2, m, e))
        stack.append((2 * i + 1, s, m))
    return np.asarray(idx, np.int64), node_data, bounds


def partition_by_counting(keys: np.ndarray, ids: np.ndarray, first: int, last: int):
    """``__unguarded_partition(first + 1, last, pivot = first)`` as the device computes it, with a count, a prefix sum and a
    scatter (DESIGN §3.16): with distinct (key, index) keys and the pivot outside [first + 1, last), the i-th element greater
    than the pivot counted from first + 1 swaps with the i-th element less than it counted from last - 1, and the cut is
    first + 1 + #(< pivot).  Returns the cut; keys and ids are permuted in place."""
    kp, ip = keys[first], ids[first]
    k, i = keys[first + 1:last], ids[first + 1:last]
    less = (k < kp) | ((k == kp) & (i < ip))
    cut = int(less.sum())
    left_g = np.flatnonzero(~less[:cut])                  # greater elements left of the cut, from the left
    right_l = np.flatnonzero(less[cut:])[::-1] + cut      # less elements right of it, from the right
    a, b = left_g, right_l
    k[a], k[b] = k[b].copy(), k[a].copy()
    i[a], i[b] = i[b].copy(), i[a].copy()
    return first + 1 + cut


def cloud(kind: str, n: int, seed: int) -> np.ndarray:
    """(n, 3) float64 test clouds: ``normal``, ``duplicates`` (a third of the points repeated), ``identical`` (every point the
    same), ``lattice`` (a shuffled grid in steps of 1/8), ``flat`` (zero spread on z, equal spread on x and y), ``float32``
    (float32 values), ``far`` (1e6 from the origin), ``zeros`` (+0.0 and -0.0 coordinates)"""
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((n, 3))
    if kind == "duplicates" and n > 1:
        X[rng.choice(n, n // 3)] = X[rng.choice(n, n // 3)]
    elif kind == "identical":
        X[:] = X[0]
    elif kind == "lattice":
        X = rng.integers(0, 6, (n, 3)) / 8.0
    elif kind == "flat":
        X[:, 2] = 0.25
        X[:, :2] = rng.integers(0, 2, (n, 2)) * 2.0 - 1.0
        X[: max(1, n // 2), 0] = -1.0
        X[: max(1, n // 2), 1] = 1.0
    elif kind == "float32":
        X = X.astype(np.float32).astype(np.float64)
    elif kind == "far":
        X = X * 1e-3 + np.array([1e6, -2e6, 5e5])
    elif kind == "zeros":
        X[rng.random(n) < 0.3] = 0.0
        X[rng.random((n, 3)) < 0.3] = -0.0
    return X


KINDS = ("normal", "duplicates", "identical", "lattice", "flat", "float32", "far", "zeros")
LEAF_SIZES = (1, 2, 30, 40)


def cases():
    """(name, X, leaf_size): n in {1, 2, 3, 11, 12, 13} and leaf_size * 2^j +- 1, every leaf size and cloud kind"""
    out = []
    for leaf_size in LEAF_SIZES:
        sizes = {1, 2, 3, 11, 12, 13}
        for j in range(0, 7):
            if leaf_size * 2 ** j <= 2500:
                sizes |= {leaf_size * 2 ** j - 1, leaf_size * 2 ** j + 1}
        for n in sorted(s for s in sizes if s >= 1):
            for k, kind in enumerate(KINDS):
                out.append((f"{kind}_n{n}_leaf{leaf_size}", cloud(kind, n, 1000 * leaf_size + 10 * n + k), leaf_size))
    return out


def killer_adversary(n: int) -> np.ndarray:
    """McIlroy's "killer adversary" against ``nth_element(arange(n), n // 2)``: values in 0 .. n-1 under which the
    introselect's pivots are as bad as its comparisons allow, so that it reaches the depth limit"""
    gas = n
    val = [gas] * n
    state = {"solid": 0, "candidate": 0}

    def freeze(x):
        val[x] = state["solid"]
        state["solid"] += 1

    def comp(x, y):
        if val[x] == gas and val[y] == gas:
            freeze(x if x == state["candidate"] else y)
        if val[x] == gas:
            state["candidate"] = x
        elif val[y] == gas:
            state["candidate"] = y
        return val[x] < val[y]

    nth_element(list(range(n)), 0, n // 2, n, comp)
    for x in range(n):
        if val[x] == gas:
            freeze(x)
    return np.asarray(val, np.float64)
