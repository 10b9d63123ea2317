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

``query(data, idx_array, node_data, node_bounds, Q, k, square)`` restates ``KDTree.query``: the depth-first walk, ``heap_push``
and the 2-way introsort of ``simultaneous_sort``.  With ``square=libm_square`` (the C library's ``pow``) it is scikit-learn's;
with ``square=exact_square`` it is the device's arithmetic with its flag rule (DESIGN §3.17).

Nothing under ``toothgroupnetwork_b200/`` may import it.
"""
from __future__ import annotations

import ctypes
import ctypes.util
import math
import operator

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


# ------------------------------------------------------------------ KDTree.query(X, k): depth first, heap_push, simultaneous_sort
_libm = ctypes.CDLL(ctypes.util.find_library("m") or "libm.so.6")
_libm.pow.argtypes = [ctypes.c_double, ctypes.c_double]
_libm.pow.restype = ctypes.c_double


def libm_square(h: float) -> float:
    """``pow(h, 2.0)`` of the C library, the square scikit-learn's ``min_rdist`` takes (p = 2 held at run time)"""
    return _libm.pow(h, 2.0)


def exact_square(h: float) -> float:
    """the device's square: the correctly rounded h * h"""
    return h * h


def _is_exact(h: float, s: float) -> bool:
    """whether s is h^2 exactly (the device tests fma(h, h, -h*h) == 0)"""
    p, q = h.as_integer_ratio()
    ps, qs = s.as_integer_ratio()
    return p * p * qs == ps * q * q


BAND = 2.0 ** -40


def _close(a: float, b: float) -> bool:
    """a decision between a and b that a few ulps in one operand could turn: the flag rule's margin"""
    return b != math.inf and abs(a - b) <= BAND * max(a, b)


class SortStats:
    def __init__(self):
        self.heapsorts = 0
        self.partitions = 0


def heap_push(values: list, indices: list, val: float, i_val: int) -> None:
    """utils/_heap.pyx heap_push: a fixed-size max-heap; rejected when val >= values[0]"""
    size = len(values)
    if val >= values[0]:
        return
    cur = 0
    while True:
        left, right = 2 * cur + 1, 2 * cur + 2
        if left >= size:
            break
        if right >= size:
            if values[left] > val:
                swap = left
            else:
                break
        elif values[left] >= values[right]:
            if val < values[left]:
                swap = left
            else:
                break
        elif val < values[right]:
            swap = right
        else:
            break
        values[cur], indices[cur] = values[swap], indices[swap]
        cur = swap
    values[cur], indices[cur] = val, i_val


def _sort_swap(v, ix, a, b):
    v[a], v[b] = v[b], v[a]
    ix[a], ix[b] = ix[b], ix[a]


def _sort_sift_down(v, ix, off, start, end, less):
    root = start
    while True:
        child = 2 * root + 1
        maxind = root
        if child < end and less(v[off + maxind], v[off + child]):
            maxind = child
        if child + 1 < end and less(v[off + maxind], v[off + child + 1]):
            maxind = child + 1
        if maxind == root:
            return
        _sort_swap(v, ix, off + root, off + maxind)
        root = maxind


def _sort_heapsort(v, ix, off, n, less):
    start = (n - 2) // 2
    while True:
        _sort_sift_down(v, ix, off, start, n, less)
        if start == 0:
            break
        start -= 1
    end = n - 1
    while end > 0:
        _sort_swap(v, ix, off, off + end)
        _sort_sift_down(v, ix, off, 0, end, less)
        end -= 1


def _sort_insertion(v, ix, off, n, less):
    for i in range(1, n):
        tv, ti = v[off + i], ix[off + i]
        j = i
        while j > 0 and less(tv, v[off + j - 1]):
            v[off + j], ix[off + j] = v[off + j - 1], ix[off + j - 1]
            j -= 1
        v[off + j], ix[off + j] = tv, ti


def _introsort_2way(v, ix, off, n, maxd, less, stats):
    while n > 15:
        if maxd <= 0:
            _sort_heapsort(v, ix, off, n, less)
            if stats is not None:
                stats.heapsorts += 1
            return
        maxd -= 1
        p = n // 2                                    # inplace_median3
        if less(v[off + n - 1], v[off]):
            _sort_swap(v, ix, off, off + n - 1)
        if less(v[off + p], v[off + n - 1]):
            _sort_swap(v, ix, off + n - 1, off + p)
            if less(v[off + n - 1], v[off]):
                _sort_swap(v, ix, off, off + n - 1)
        pivot = v[off + n - 1]
        i, j = 1, n - 2
        while True:
            while i <= j and less(v[off + i], pivot):
                i += 1
            while i <= j and less(pivot, v[off + j]):
                j -= 1
            if i >= j:
                break
            _sort_swap(v, ix, off + i, off + j)
            i += 1
            j -= 1
        _sort_swap(v, ix, off + i, off + n - 1)
        if stats is not None:
            stats.partitions += 1
        _introsort_2way(v, ix, off, i, maxd, less, stats)
        off += i + 1
        n -= i + 1
    _sort_insertion(v, ix, off, n, less)


def simultaneous_sort(values: list, indices: list, less=operator.lt, stats: SortStats | None = None) -> None:
    """utils/_sorting.pyx simultaneous_sort with the default 2-way introsort, in place; ``less`` stands for the ``<`` of
    doubles (``a > b`` is ``less(b, a)``)"""
    n = len(values)
    if n:
        _introsort_2way(values, indices, 0, n, 2 * int(math.log2(n)), less, stats)


def query(data, idx_array, node_data, node_bounds, Q, k: int, square=libm_square, trace: list | None = None):
    """``KDTree.query(Q, k)`` of the tree (data, idx_array, node_data, node_bounds) -> (dist (m,k), ind (m,k), flag (m)).

    With ``square=libm_square`` every value is scikit-learn's.  With ``square=exact_square`` it is the device's arithmetic,
    and flag[i] = 1 when row i took a trim (LB > largest) or child-order (LB1 <= LB2) decision that involved a bound with an
    inexact square and operands within a relative 2^-40: the rows where that arithmetic may leave scikit-learn's walk.
    ``trace``, a list, receives per row the walk's decisions: the nodes entered, each with whether it was trimmed."""
    data = np.ascontiguousarray(data, np.float64)
    Q = np.ascontiguousarray(Q, np.float64)
    nodes = np.ascontiguousarray(node_data)
    if nodes.dtype.names is None:
        nodes = nodes.view([("idx_start", "<i8"), ("idx_end", "<i8"), ("is_leaf", "<i8"), ("radius", "<f8")]).reshape(-1)
    starts, ends, leaves = nodes["idx_start"].tolist(), nodes["idx_end"].tolist(), nodes["is_leaf"].tolist()
    lo, hi = node_bounds[0].tolist(), node_bounds[1].tolist()
    idx = np.asarray(idx_array).tolist()
    pts = data.tolist()
    m = Q.shape[0]
    dist = np.empty((m, k), np.float64)
    ind = np.empty((m, k), np.intp)
    flag = np.zeros(m, np.uint8)

    def min_rdist(node, q):
        r, exact = 0.0, True
        for j in range(3):
            d_lo = lo[node][j] - q[j]
            d_hi = q[j] - hi[node][j]
            h = 0.5 * ((d_lo + abs(d_lo)) + (d_hi + abs(d_hi)))
            s = square(h)
            exact = exact and _is_exact(h, s)
            r += s
        return r, exact

    for row, q in enumerate(Q.tolist()):
        values, indices = [math.inf] * k, [0] * k
        flagged = False
        lb, ex = min_rdist(0, q)
        stack = [(0, lb, ex)]
        walk = []
        while stack:
            node, lb, ex = stack.pop()
            flagged |= not ex and _close(lb, values[0])
            walk.append((node, lb > values[0]))
            if lb > values[0]:
                continue
            if leaves[node]:
                for i in range(starts[node], ends[node]):
                    x = pts[idx[i]]
                    dx, dy, dz = q[0] - x[0], q[1] - x[1], q[2] - x[2]
                    heap_push(values, indices, ((0.0 + dx * dx) + dy * dy) + dz * dz, idx[i])
            else:
                i1, i2 = 2 * node + 1, 2 * node + 2
                lb1, ex1 = min_rdist(i1, q)
                lb2, ex2 = min_rdist(i2, q)
                flagged |= not (ex1 and ex2) and _close(lb1, lb2)
                if lb1 <= lb2:
                    stack += [(i2, lb2, ex2), (i1, lb1, ex1)]
                else:
                    stack += [(i1, lb1, ex1), (i2, lb2, ex2)]
        if trace is not None:
            trace.append(walk)
        simultaneous_sort(values, indices)
        dist[row] = np.sqrt(np.asarray(values))
        ind[row] = indices
        flag[row] = flagged
    return dist, ind, flag


def sort_killer(n: int) -> np.ndarray:
    """values 0 .. n-1 on which ``simultaneous_sort`` partitions as badly as its comparisons allow (McIlroy's adversary, as
    ``killer_adversary``), so that a long enough input reaches the depth limit and its heapsort"""
    gas = n
    val = [gas] * n
    state = {"solid": 0, "candidate": 0}

    def freeze(x):
        val[x] = state["solid"]
        state["solid"] += 1

    def less(x, y):
        if val[x] == gas and val[y] == gas:
            freeze(x if x == state["candidate"] else y)
        if val[x] == gas:
            state["candidate"] = x
        elif val[y] == gas:
            state["candidate"] = y
        return val[x] < val[y]

    simultaneous_sort(list(range(n)), list(range(n)), less)
    for x in range(n):
        if val[x] == gas:
            freeze(x)
    return np.asarray(val, np.float64)


def tied_query_inputs(full: bool):
    """(name, points, queries) float64 inputs whose nearest distances tie, as in the label transfers: tgn's final tree (FPS
    samples and kept boundary vertices of one arch, float32, queried with every vertex), a float32 arch with every vertex twice
    queried with its own points, and the 1/8 lattice queried with offset and random 1/128 points.  ``full`` gives the
    pipelines' sizes (10^5 vertices), otherwise a few hundred rows for the Python walk."""
    from toothgroupnetwork_b200 import clouds
    m, first, bdl, arch_n, side, nq = (100000, 24000, 20000, 12000, 12, 800) if full else (1500, 360, 300, 300, 6, 60)
    verts = clouds.dental_arch(m, 11)[0].numpy()
    rng = np.random.default_rng(11)
    tree = np.concatenate([verts[rng.choice(m, first, replace=False)], verts[rng.choice(m, bdl, replace=False)]])
    yield "tgn_final", tree.astype(np.float64), verts.astype(np.float64)
    pts = clouds.with_duplicates(clouds.dental_arch(arch_n, 12)[0], 12).double().numpy()
    yield "arch_duplicates", pts, pts
    pts = np.stack(np.meshgrid(*[np.arange(side) / 8.0] * 3, indexing="ij"), -1).reshape(-1, 3)
    pts = pts[np.random.default_rng(13).permutation(pts.shape[0])]
    q = np.concatenate([pts[:nq] + np.array([1.0, 0.5, 0.0]) / 16.0,
                        np.random.default_rng(14).integers(-8, 16 * side, (nq, 3)) / 128.0])
    yield "lattice", pts, q


def pow_decides_otherwise():
    """(points, queries, leaf_size, k, rows): a seeded input, found by search, on which the walk with the C library's pow and
    the walk with h*h take different trim decisions at ``rows`` (every point twice, nearly every leaf a single point, so
    that a leaf's bound equals the distance of its tied twin)"""
    rng = np.random.default_rng(0)
    P = rng.random((33, 3)) * 0.3
    X = np.concatenate([P, P])[rng.permutation(66)]
    Q = rng.random((4000, 3)) * 0.3
    return X, Q, 1, 1, (51, 498, 3863)
