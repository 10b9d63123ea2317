"""Exact nearest-neighbour label transfers of the inference pipelines on the GPU: a ``KDTree`` drop-in (DESIGN §3.10).

Every inference pipeline ends by giving each mesh vertex the label of its nearest sampled point through
``sklearn.neighbors.KDTree(points, leaf_size=2).query(vertices, k=1)`` in float64 on the host (inference_pipeline_tgn.py:107-114
and :137-140, inference_pipeline_tsegnet.py:72-74, inference_pipeline_sem.py:37-39).  ``KDTree`` here builds the float64 grid
of csrc/knn_f64.cu once per point set and answers every ``query`` with one upload, one launch and one download.

The kernel's neighbours are ordered by (d2, index), while the KDTree keeps whichever exactly tied point its depth-first walk
meets first -- an order set by its in-leaf layout, which the GPU cannot reproduce.  So each query also returns a tie flag: a row
whose min(k+1, n) best squared distances are all distinct has one answer under any tie-break rule and is taken from the GPU; the
flagged rows are re-answered by scikit-learn's own tree, built on the first flag and kept.  Duplicated vertices make such rows
common (a point that is both an FPS sample and a kept boundary vertex is in tgn's final tree twice).  ``host_rows`` counts them.

``accelerate(module)`` points a module's ``KDTree`` name at the class.  scikit-learn is imported only when a row is flagged.
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
        self._launch(torch.from_numpy(X).to(self.device), k, idx, dist, out[n_idx + n_dist:])
        host = out.cpu().numpy()
        ind = host[:n_idx].view(np.intp).reshape(m, k)
        d = host[n_idx:n_idx + n_dist].view(np.float64).reshape(m, k) if return_distance else None
        rows = np.flatnonzero(host[n_idx + n_dist:])
        if rows.size:
            if self._host_tree is None:
                from sklearn.neighbors import KDTree as HostKDTree
                self._host_tree = HostKDTree(self._X, leaf_size=self.leaf_size)
            self.host_rows += int(rows.size)
            if return_distance:
                d[rows], ind[rows] = self._host_tree.query(X[rows], k=k)
            else:
                ind[rows] = self._host_tree.query(X[rows], k=k, return_distance=False)
        return (d, ind) if return_distance else ind


def accelerate(module) -> None:
    """Point a module's ``KDTree`` name (``from sklearn.neighbors import KDTree`` in inference_pipeline_tgn.py:6,
    inference_pipeline_tsegnet.py:5, inference_pipeline_sem.py:4) at the device implementation."""
    if hasattr(module, "KDTree"):
        module.KDTree = KDTree
