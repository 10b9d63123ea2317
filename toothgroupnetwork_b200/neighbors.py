"""Exact nearest-neighbour label transfers of the inference pipelines on the GPU: a ``KDTree`` drop-in (DESIGN §3.10).

Every inference pipeline ends by giving each mesh vertex the label of its nearest sampled point through
``sklearn.neighbors.KDTree(points, leaf_size=2).query(vertices, k=1)`` in float64 on the host (inference_pipeline_tgn.py:107-114
and :137-140, inference_pipeline_tsegnet.py:72-74, inference_pipeline_sem.py:37-39).  ``KDTree`` here builds the float64 grid
of csrc/knn_f64.cu once per point set and answers every ``query`` with one upload, one launch and one download.

The kernel's neighbours are ordered by (d2, index), while the KDTree keeps whichever exactly tied point its depth-first walk
meets first -- an order set by its in-leaf layout.  So each query also returns a tie flag: a row whose min(k+1, n) best squared
distances are all distinct has one answer under any tie-break rule and is taken from the GPU; the flagged rows are re-answered
by scikit-learn's own query code.  Duplicated vertices make such rows common (a point that is both an FPS sample and a kept
boundary vertex is in tgn's final tree twice).  ``host_rows`` counts them.

The tree those rows need is scikit-learn's, bit for bit, and ``sklearn_tree`` builds it on the device (csrc/kdtree_build.cu,
DESIGN §3.16): on the first flagged row its arrays are copied to the host once and a scikit-learn ``KDTree`` is restored from
them with ``__setstate__``, without a host build.  An installation whose pickled state has another layout builds it on the host.

``DeviceKDTree`` answers the flagged rows on the device instead: ``sklearn_query`` walks that tree the way scikit-learn's
``query`` does (csrc/kdtree_query.cu, DESIGN §3.17), and only the rows whose walk it flags reach scikit-learn's query code.

``accelerate(module, ties)`` points a module's ``KDTree`` name at one of the classes.  scikit-learn is imported only when a row
is flagged.
"""
from __future__ import annotations

import operator
from typing import Tuple

import numpy as np
import torch

from . import _lib as L

MAX_K = 63                                    # the tie flag keeps k + 1 entries in the kernel's 64-entry list


def _as_points(X) -> np.ndarray:
    """float64 (n, d) C-contiguous, refused with scikit-learn's exception type (check_array: ValueError) when not 2-D, empty or
    not finite."""
    X = np.asarray(X, dtype=np.float64)
    if X.ndim != 2:
        raise ValueError(f"Expected 2D array, got {X.ndim}D array instead")
    if X.shape[0] == 0:
        raise ValueError(f"Found array with 0 sample(s) (shape={X.shape}) while a minimum of 1 is required.")
    if not np.isfinite(X).all():
        raise ValueError("Input contains NaN or infinity.")
    return np.ascontiguousarray(X)


class KDTree:
    """The slice of ``sklearn.neighbors.KDTree`` the reference uses -- ``KDTree(X, leaf_size=...)`` then
    ``.query(X, k, return_distance)`` -- with the same indices and bitwise-equal distances.  Euclidean (the default
    ``metric="minkowski"``, p = 2) on (n, 3) points, k <= 63, sorted results; anything else is refused with ``TgnError``.
    ``leaf_size`` only shapes the host tree that resolves exactly tied rows.  The grid is built on the current CUDA stream."""

    def __init__(self, X, leaf_size: int = 40, metric: str = "minkowski", **kwargs):
        if metric != "minkowski" or kwargs:
            raise L.TgnError(f"KDTree: only the default Euclidean metric is implemented (got metric={metric!r}, {kwargs})")
        X = _as_points(X)
        if leaf_size < 1:
            raise ValueError("leaf_size must be greater than or equal to 1")
        if X.shape[1] != 3:
            raise L.TgnError(f"KDTree: only (n, 3) points are implemented, got {X.shape}")
        if not torch.cuda.is_available():
            raise L.TgnError("KDTree needs a CUDA device (there is no CPU path)")
        self.leaf_size = leaf_size
        self.host_rows = 0                    # rows answered by scikit-learn's tree because of an exact tie
        self._X = X
        self._host_tree = None
        self._n = int(X.shape[0])
        dev = torch.device("cuda", torch.cuda.current_device())
        self._xyz = torch.from_numpy(X).to(dev)
        self._ws = torch.empty(int(L.load().tgn_knn_f64_bytes(self._n)), dtype=torch.uint8, device=dev)
        L.call("tgn_knn_f64_build", self._n, L.ptr(self._xyz), L.ptr(self._ws), L.stream_ptr())

    @property
    def device(self) -> torch.device:
        return self._xyz.device

    def _launch(self, queries: torch.Tensor, k: int, idx, dist, tie) -> None:
        L.call("tgn_knn_f64_query", self._n, int(queries.shape[0]), int(k), L.ptr(self._xyz), L.ptr(queries), L.ptr(self._ws),
               None, L.ptr(idx), L.ptr(dist), None, None, L.ptr(tie), L.stream_ptr())

    def query_device(self, queries: torch.Tensor, k: int = 1) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        """queries (m,3) float64 on the tree's device -> (idx int64 (m,k), dist float64 (m,k), tie uint8 (m)), all on the device:
        neighbours ascending by (squared distance, index), tie = 1 where two adjacent of the min(k+1, n) best squared distances
        are equal (only those rows can differ from scikit-learn's KDTree).  No host tree is involved."""
        k = operator.index(k)
        if not torch.is_tensor(queries) or queries.dim() != 2 or queries.shape[1] != 3 or queries.dtype != torch.float64:
            raise L.TgnError(f"KDTree.query_device: queries must be an (m, 3) float64 tensor, got "
                             f"{tuple(queries.shape) if torch.is_tensor(queries) else type(queries)}")
        if not 1 <= k <= min(self._n, MAX_K):
            raise L.TgnError(f"KDTree.query_device: need 1 <= k <= min(n, {MAX_K}), got k={k} with n={self._n}")
        L.require_cuda(queries)
        if queries.device != self.device:
            raise L.TgnError(f"KDTree.query_device: queries on {queries.device}, tree on {self.device}")
        if not bool(torch.isfinite(queries).all()):
            raise L.TgnError("KDTree.query_device: non-finite coordinates")
        queries = queries.contiguous()
        m = queries.shape[0]
        idx = torch.empty((m, k), dtype=torch.int64, device=self.device)
        dist = torch.empty((m, k), dtype=torch.float64, device=self.device)
        tie = torch.empty(m, dtype=torch.uint8, device=self.device)
        if m:
            self._launch(queries, k, idx, dist, tie)
        return idx, dist, tie

    def query(self, X, k: int = 1, return_distance: bool = True, dualtree: bool = False, breadth_first: bool = False,
              sort_results: bool = True):
        """``sklearn.neighbors.KDTree.query``: (dist float64 (m,k), ind intp (m,k)), or ind alone without return_distance."""
        if dualtree or breadth_first or not sort_results:
            raise L.TgnError("KDTree.query: only the default single-tree, depth-first, sorted query is implemented")
        k = operator.index(k)
        X = _as_points(X)
        if X.shape[1] != 3:
            raise ValueError("query data dimension must match training data dimension")
        if self._n < k:
            raise ValueError("k must be less than or equal to the number of training points")
        if not 1 <= k <= MAX_K:
            raise L.TgnError(f"KDTree.query: need 1 <= k <= {MAX_K}, got k={k}")
        m = X.shape[0]
        # one device buffer for every output, so that one copy brings them back: idx, [dist,] tie
        n_idx, n_dist = 8 * m * k, (8 * m * k if return_distance else 0)
        out = torch.empty(n_idx + n_dist + m, dtype=torch.uint8, device=self.device)
        idx = out[:n_idx].view(torch.int64).view(m, k)
        dist = out[n_idx:n_idx + n_dist].view(torch.float64).view(m, k) if return_distance else None
        queries = torch.from_numpy(X).to(self.device)
        self._launch(queries, k, idx, dist, out[n_idx + n_dist:])
        host = out.cpu().numpy()
        tied = np.flatnonzero(host[n_idx + n_dist:])
        if tied.size:
            host = self._walk_ties(queries, k, idx, dist, out[n_idx + n_dist:], tied, out, host)
        ind = host[:n_idx].view(np.intp).reshape(m, k)
        d = host[n_idx:n_idx + n_dist].view(np.float64).reshape(m, k) if return_distance else None
        rows = np.flatnonzero(host[n_idx + n_dist:])
        if rows.size:
            if self._host_tree is None:
                self._host_tree = host_tree(self._X, self._xyz, self.leaf_size)
            self.host_rows += int(rows.size)
            if return_distance:
                d[rows], ind[rows] = self._host_tree.query(X[rows], k=k)
            else:
                ind[rows] = self._host_tree.query(X[rows], k=k, return_distance=False)
        return (d, ind) if return_distance else ind

    def _walk_ties(self, queries, k, idx, dist, flag, tied, out, host):
        """The rows the grid flags (``tied``, ascending) before the host fallback: here all of them stay flagged.  Returns the
        host copy of ``out``, whose flag bytes name the rows left to the host."""
        return host


class DeviceKDTree(KDTree):
    """``KDTree`` whose tied rows are answered on the device: scikit-learn's own depth-first walk over its own tree
    (``sklearn_query`` on ``sklearn_tree(X, leaf_size, radius=False)``, built once on the first tie, nothing copied to the
    host).  Only the rows the walk flags go to scikit-learn's query code (``host_rows``); ``walk_rows`` counts the rows the walk
    answered.  A tree outside the device build's range, a leaf_size that is not an integer or a scikit-learn whose pickled
    KDTree has another layout than the 1.9 the walk restates keep every tied row on the host, as ``KDTree`` does."""

    def __init__(self, X, leaf_size: int = 40, metric: str = "minkowski", **kwargs):
        super().__init__(X, leaf_size, metric, **kwargs)
        self.walk_rows = 0
        self._walk_tree = None
        self._walk_ok = None

    def _walk_ties(self, queries, k, idx, dist, flag, tied, out, host):
        if self._walk_ok is None:
            ls = self.leaf_size
            self._walk_ok = (not isinstance(ls, bool) and isinstance(ls, (int, np.integer))
                             and int(L.load().tgn_kdtree_nodes(self._n, int(ls))) == tree_nodes(self._n, int(ls))
                             and _sklearn_layout_ok())
        if not self._walk_ok:
            return host
        if self._walk_tree is None:
            self._walk_tree = sklearn_tree(self._xyz, int(self.leaf_size), radius=False)
        _walk(self._walk_tree, queries, k, torch.from_numpy(tied).to(self.device), idx, dist, flag)
        host = out.cpu().numpy()
        self.walk_rows += int(tied.size) - int(np.count_nonzero(host[host.size - flag.numel():]))
        return host


NODE_DATA = np.dtype([("idx_start", "<i8"), ("idx_end", "<i8"), ("is_leaf", "<i8"), ("radius", "<f8")])   # NodeData_t


def tree_nodes(n: int, leaf_size: int) -> int:
    """scikit-learn's node count: 2^n_levels - 1 with n_levels = int(log2(max(1, (n - 1) / leaf_size)) + 1)"""
    n_levels = int(np.log2(max(1.0, (n - 1) / leaf_size)) + 1)
    return 2 ** n_levels - 1


def _device_points(X) -> torch.Tensor:
    """(n, 3) float64 finite points -> a contiguous CUDA tensor, refused (ValueError, as scikit-learn) before any launch"""
    if torch.is_tensor(X):
        L.require_cuda(X)
        if X.dim() != 2 or X.shape[1] != 3 or X.dtype != torch.float64:
            raise L.TgnError(f"sklearn_tree: expected (n, 3) float64 points, got {tuple(X.shape)} {X.dtype}")
        if X.shape[0] == 0:
            raise ValueError("X is an empty array")
        if not bool(torch.isfinite(X).all()):
            raise ValueError("Input contains NaN or infinity.")
        return X.contiguous()
    X = _as_points(X)
    if X.shape[1] != 3:
        raise L.TgnError(f"sklearn_tree: only (n, 3) points are implemented, got {X.shape}")
    if not torch.cuda.is_available():
        raise L.TgnError("sklearn_tree needs a CUDA device (there is no CPU path)")
    return torch.from_numpy(X).cuda()


def _build(xyz: torch.Tensor, leaf_size: int):
    """csrc/kdtree_build.cu on the current stream -> (idx_array int64 (n), node_data int64 (n_nodes, 4) with the radius
    column NaN, node_bounds float64 (2, n_nodes, 3)), all on xyz's device"""
    if isinstance(leaf_size, bool) or not isinstance(leaf_size, (int, np.integer)) or leaf_size < 1:
        raise ValueError("leaf_size must be greater than or equal to 1")
    n = int(xyz.shape[0])
    n_nodes = tree_nodes(n, int(leaf_size))
    if int(L.load().tgn_kdtree_nodes(n, int(leaf_size))) != n_nodes:
        raise L.TgnError(f"sklearn_tree: n={n} leaf_size={leaf_size} is outside the device build's range")
    dev = xyz.device
    idx = torch.empty(n, dtype=torch.int64, device=dev)
    node_data = torch.empty((n_nodes, 4), dtype=torch.int64, device=dev)
    bounds = torch.empty((2, n_nodes, 3), dtype=torch.float64, device=dev)
    ws = torch.empty(int(L.load().tgn_kdtree_bytes(n, int(leaf_size))), dtype=torch.uint8, device=dev)
    L.call("tgn_kdtree_build", n, int(leaf_size), L.ptr(xyz), L.ptr(idx), L.ptr(node_data), L.ptr(bounds), L.ptr(ws),
           L.stream_ptr())
    return idx, node_data, bounds


def _fill_radius(node_data: np.ndarray, bounds: np.ndarray) -> None:
    """init_node's radius into host node_data (n_nodes, 4) 8-byte records from host node_bounds, with the C library's pow as
    scikit-learn computes it (the device's correctly rounded sqrt and squares differ from it in about 1 node in 1000)"""
    L.load().tgn_kdtree_radius(int(node_data.shape[0]), bounds.ctypes.data, node_data.ctypes.data)


def sklearn_tree(X, leaf_size: int = 40, radius: bool = True):
    """``sklearn.neighbors.KDTree(X, leaf_size).get_arrays()`` built on the GPU, bit for bit: (data (n,3) float64,
    idx_array int64 (n), node_data int64 (n_nodes, 4) = NodeData_t's idx_start, idx_end, is_leaf and the float64 bits of
    radius, node_bounds float64 (2, n_nodes, 3)), all on the device.  X is host (n, 3) points or a float64 CUDA tensor; empty,
    non-finite input and leaf_size < 1 are refused with scikit-learn's ValueError before any launch.  The radius is computed
    on the host from the bounds (one copy each way); with ``radius=False`` it stays NaN and nothing leaves the device.
    ``node_data.cpu().numpy().view(NODE_DATA)`` is scikit-learn's record array."""
    if isinstance(leaf_size, bool) or not isinstance(leaf_size, (int, np.integer)) or leaf_size < 1:
        raise ValueError("leaf_size must be greater than or equal to 1")
    xyz = _device_points(X)
    idx, node_data, bounds = _build(xyz, leaf_size)
    if not radius:
        return xyz, idx, node_data, bounds
    host_bounds = bounds.cpu().numpy()
    host_nodes = node_data.cpu().numpy()
    _fill_radius(host_nodes, host_bounds)
    node_data[:, 3].copy_(torch.from_numpy(np.ascontiguousarray(host_nodes[:, 3])))
    return xyz, idx, node_data, bounds


def _walk(tree, queries: torch.Tensor, k: int, rows, idx, dist, flag) -> None:
    """csrc/kdtree_query.cu on the current stream: rows (int64 on the device) or every row when None"""
    xyz, idx_array, node_data, bounds = tree
    L.call("tgn_kdtree_query", int(xyz.shape[0]), int(node_data.shape[0]), int(k), L.ptr(xyz), L.ptr(idx_array),
           L.ptr(node_data), L.ptr(bounds), int(queries.shape[0]), L.ptr(queries), L.ptr(rows),
           0 if rows is None else int(rows.numel()), L.ptr(idx), L.ptr(dist), L.ptr(flag), L.stream_ptr())


def sklearn_query(tree, queries: torch.Tensor, k: int = 1, rows=None):
    """``sklearn.neighbors.KDTree(X, leaf_size).query(queries, k)`` walked on the GPU over ``tree``, the tuple
    ``sklearn_tree(X, leaf_size, radius=False)`` returns: scikit-learn's depth-first visit order, its heap and its final sort
    (csrc/kdtree_query.cu, DESIGN §3.17).  queries (m, 3) float64 CUDA -> (dist float64 (m, k), idx int64 (m, k),
    flag uint8 (m)) on the device.  Every row with flag 0 is scikit-learn's answer, indices and distance bits; a flagged row
    compared a node bound within 2^-40 of the other operand where scikit-learn's ``pow`` could round differently.
    ``rows`` (row numbers, host or device) restricts the walk to those rows; the other rows of the outputs are left
    uninitialised.  Refusals raise before any launch: scikit-learn's ValueError where it refuses (empty or non-finite
    queries, another width, k > n), TgnError for what is not implemented (k outside 1..63, non-CUDA or non-float64 queries, a
    malformed tree)."""
    if not isinstance(tree, tuple) or len(tree) != 4 or not all(torch.is_tensor(t) for t in tree):
        raise L.TgnError("sklearn_query: tree must be the tuple sklearn_tree(X, leaf_size, radius=False) returns")
    xyz, idx_array, node_data, bounds = tree
    L.require_cuda(*tree)
    n, n_nodes = int(xyz.shape[0]), int(node_data.shape[0])
    if (xyz.dtype != torch.float64 or idx_array.dtype != torch.int64 or node_data.dtype != torch.int64
            or bounds.dtype != torch.float64 or tuple(xyz.shape) != (n, 3) or tuple(idx_array.shape) != (n,)
            or tuple(node_data.shape) != (n_nodes, 4) or tuple(bounds.shape) != (2, n_nodes, 3)
            or not all(t.is_contiguous() and t.device == xyz.device for t in tree)
            or not 1 <= n <= 2 ** 30 or n_nodes & (n_nodes + 1) or (n_nodes + 1) // 2 > n):
        raise L.TgnError("sklearn_query: tree must be the tuple sklearn_tree(X, leaf_size, radius=False) returns")
    if not torch.is_tensor(queries) or queries.dtype != torch.float64:
        raise L.TgnError(f"sklearn_query: queries must be a float64 CUDA tensor, got "
                         f"{queries.dtype if torch.is_tensor(queries) else type(queries)}")
    L.require_cuda(queries)
    if queries.device != xyz.device:
        raise L.TgnError(f"sklearn_query: queries on {queries.device}, tree on {xyz.device}")
    if queries.dim() != 2:
        raise ValueError(f"Expected 2D array, got {queries.dim()}D array instead")
    if queries.shape[0] == 0:
        raise ValueError(f"Found array with 0 sample(s) (shape={tuple(queries.shape)}) while a minimum of 1 is required.")
    if queries.shape[1] != 3:
        raise ValueError("query data dimension must match training data dimension")
    if not bool(torch.isfinite(queries).all()):
        raise ValueError("Input contains NaN or infinity.")
    k = operator.index(k)
    if n < k:
        raise ValueError("k must be less than or equal to the number of training points")
    if not 1 <= k <= MAX_K:
        raise L.TgnError(f"sklearn_query: need 1 <= k <= {MAX_K}, got k={k}")
    m = int(queries.shape[0])
    if rows is not None:
        host_rows = np.asarray(rows.cpu() if torch.is_tensor(rows) else rows)
        if host_rows.ndim != 1 or (host_rows.size and host_rows.dtype.kind not in "iu"):
            raise L.TgnError("sklearn_query: rows must be a 1-D array of row numbers")
        if host_rows.size and (host_rows.min() < 0 or host_rows.max() >= m):
            raise L.TgnError(f"sklearn_query: rows must lie in [0, {m})")
        rows = torch.from_numpy(host_rows.astype(np.int64)).to(xyz.device)
    queries = queries.contiguous()
    idx = torch.empty((m, k), dtype=torch.int64, device=xyz.device)
    dist = torch.empty((m, k), dtype=torch.float64, device=xyz.device)
    flag = torch.empty(m, dtype=torch.uint8, device=xyz.device)
    if rows is None or rows.numel():
        _walk(tree, queries, k, rows, idx, dist, flag)
    return dist, idx, flag


def host_kdtree_class():
    """The host class the tie fallback restores (or, on an unexpected state layout, builds): scikit-learn's KDTree."""
    from sklearn.neighbors import KDTree as HostKDTree
    return HostKDTree


_state_ok = None


def _state_layout_ok(cls) -> bool:
    """Whether this scikit-learn pickles a KDTree the way 1.9 does: 13 fields, float64 data, intp idx_array, NodeData_t
    records, float64 bounds, a Euclidean metric object -- checked once on an empty instance, without a build."""
    global _state_ok
    if _state_ok is None:
        try:
            st = cls.__new__(cls).__getstate__()
            from sklearn.metrics import DistanceMetric
            metric = DistanceMetric.get_metric("minkowski", p=2)
            _state_ok = (len(st) == 13 and st[0].dtype == np.float64 and st[1].dtype == np.intp and st[2].dtype == NODE_DATA
                         and st[3].dtype == np.float64 and st[3].ndim == 3 and type(metric).__name__ == "EuclideanDistance64")
        except Exception:
            _state_ok = False
    return _state_ok


def _sklearn_layout_ok() -> bool:
    """Whether the installed scikit-learn is the 1.9 whose query the device walk restates, judged by its KDTree's state
    layout (the check the tie fallback's restore makes, shared with it)."""
    from sklearn.neighbors import KDTree as SkKDTree
    return _state_layout_ok(SkKDTree)


def host_tree(X: np.ndarray, xyz: torch.Tensor, leaf_size: int):
    """scikit-learn's ``KDTree(X, leaf_size)`` for host queries: built on the device from xyz (X on the device), copied once
    and restored with ``__setstate__``; built on the host when this scikit-learn's state layout is not the expected one."""
    cls = host_kdtree_class()
    if not _state_layout_ok(cls) or isinstance(leaf_size, bool) or not isinstance(leaf_size, (int, np.integer)):
        return cls(X, leaf_size=leaf_size)
    idx, node_data, bounds = _build(xyz, leaf_size)
    n, n_nodes = idx.numel(), node_data.shape[0]
    flat = torch.cat([idx, node_data.reshape(-1), bounds.reshape(-1).view(torch.int64)]).cpu().numpy()   # one copy
    idx_h = flat[:n].astype(np.intp, copy=False)
    nodes_h = np.ascontiguousarray(flat[n:n + 4 * n_nodes]).reshape(n_nodes, 4)
    bounds_h = np.ascontiguousarray(flat[n + 4 * n_nodes:]).view(np.float64).reshape(2, n_nodes, 3)
    _fill_radius(nodes_h, bounds_h)
    return restore(cls, X, idx_h, nodes_h.view(NODE_DATA).reshape(n_nodes), bounds_h, leaf_size)


def restore(cls, X: np.ndarray, idx_array: np.ndarray, node_data: np.ndarray, node_bounds: np.ndarray, leaf_size: int):
    """A scikit-learn KDTree of class ``cls`` from the arrays ``get_arrays()`` returns, by ``__setstate__`` (no build): the
    state of a freshly built tree -- no query counters, the Euclidean metric, no sample weights."""
    from sklearn.metrics import DistanceMetric
    n_nodes = int(node_data.shape[0])
    tree = cls.__new__(cls)
    tree.__setstate__((X, idx_array, node_data, node_bounds, int(leaf_size), int(np.log2(n_nodes + 1)), n_nodes, 0, 0, 0, 0,
                       DistanceMetric.get_metric("minkowski", p=2), None))
    return tree


def accelerate(module, ties: str = "host") -> None:
    """Point a module's ``KDTree`` name (``from sklearn.neighbors import KDTree`` in inference_pipeline_tgn.py:6,
    inference_pipeline_tsegnet.py:5, inference_pipeline_sem.py:4) at the device implementation: ``KDTree`` with
    ties="host", ``DeviceKDTree`` (tied rows walked on the device) with ties="device"."""
    classes = {"host": KDTree, "device": DeviceKDTree}
    if ties not in classes:
        raise ValueError(f"ties must be 'host' or 'device', got {ties!r}")
    if hasattr(module, "KDTree"):
        module.KDTree = classes[ties]
