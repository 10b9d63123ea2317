"""The clustering step between the two stages of the reference's two-stage models, on the GPU (SURVEY.md 8(f)-4).

``ops_utils.get_clustering_labels`` (ops_utils.py:86-144, called at grouping_network_module.py:65) runs
``sklearn.cluster.DBSCAN(eps=0.03, min_samples=30)`` on the offset-moved foreground points, splits suspiciously elongated
clusters with MeanShift and gives every noise point the majority label of its 10 nearest labelled points (a KDTree).  On a
trained network the DBSCAN alone costs 0.9 s per cloud on the host -- an order of magnitude more than the two networks.

Here ``dbscan`` is csrc/dbscan.cu (labels and core samples equal to scikit-learn's: the float64 predicate of its KD-tree
search, (dx^2 + dy^2) + dz^2 <= eps^2, the same cluster numbering, the same border rule).  scikit-learn searches clouds of at
most 11 points by brute force instead, whose expanded distance can fall on the other side of eps; ``dbscan`` and ``DBSCAN``
hand those to scikit-learn on the host.  Non-finite coordinates raise scikit-learn's ValueError.  The noise vote uses the
float64 selection kernel of csrc/crop_knn.cu, and
``get_clustering_labels`` keeps the reference's steps and return value.  The elongation test is the reference's (PCA
eigenvalues of the core points); the MeanShift split of at most three elongated clusters is ``MeanShift`` below, whose seed
ascent is csrc/meanshift.cu (scikit-learn's seeds, centres and labels bit for bit).  ``accelerate(ops_utils_module)`` swaps the
function in an imported reference ``ops_utils``.

``KMeans`` (csrc/kmeans.cu) is ``ops_utils.clustering_points(method="kmeans")``'s k-means++ / Lloyd fit.
"""
from __future__ import annotations

from typing import Tuple

import numpy as np
import torch

from . import _lib as L
from . import crops
from . import neighbors

_ws = {}


def _workspace(n: int, device) -> torch.Tensor:
    need = int(L.load().tgn_dbscan_bytes(int(n)))
    key = (device.index, torch.cuda.current_stream(device).cuda_stream)
    buf = _ws.get(key)
    if buf is None or buf.numel() < need:
        buf = torch.empty(need, dtype=torch.uint8, device=device)
        _ws[key] = buf
    return buf


def dbscan_device(points: torch.Tensor, eps: float = 0.03, min_samples: int = 30) -> Tuple[torch.Tensor, torch.Tensor]:
    """points (n,3) float32 CUDA -> (labels (n) int32, core (n) uint8), both on the device; equal to
    ``sklearn.cluster.DBSCAN(eps, min_samples).fit(points)``'s ``labels_`` / ``core_sample_indices_`` wherever scikit-learn
    takes its KD-tree path (n >= 12).  At every n the kernel applies that path's predicate; a point with a non-finite
    coordinate is no one's neighbour, not even its own, so it is noise."""
    L.require_cuda(points)
    if points.dim() != 2 or points.shape[1] != 3 or points.dtype != torch.float32:
        raise L.TgnError(f"dbscan expects (n,3) float32 points, got {tuple(points.shape)} {points.dtype}")
    points = points.contiguous()
    n = points.shape[0]
    labels = torch.empty(n, dtype=torch.int32, device=points.device)
    core = torch.empty(n, dtype=torch.uint8, device=points.device)
    if n:
        ws = _workspace(n, points.device)
        L.call("tgn_dbscan", n, L.ptr(points), float(eps), int(min_samples), L.ptr(ws), L.ptr(labels), L.ptr(core), None, L.stream_ptr())
    return labels, core


def _as_float32(points: np.ndarray) -> np.ndarray:
    """The kernel takes float32 coordinates (what ops_utils.get_clustering_labels is handed: float32 points + float32 offsets) and
    evaluates distances in float64 like scikit-learn.  Wider input is accepted when it holds float32 values; anything else would be
    clustered on rounded coordinates and could differ from scikit-learn, so it is refused."""
    points = np.asarray(points)
    if points.dtype == np.float32:
        return np.ascontiguousarray(points)
    down = np.ascontiguousarray(points, dtype=np.float32)
    if not np.array_equal(down.astype(points.dtype), points):
        raise L.TgnError(f"dbscan: {points.dtype} coordinates that are not float32 values are not supported")
    return down


def _check_finite(x) -> None:
    """scikit-learn's refusal of non-finite coordinates (``sklearn.utils.check_array``), with the start of its messages"""
    if isinstance(x, torch.Tensor):
        if bool(torch.isfinite(x).all()):
            return
        nan, dtype = bool(torch.isnan(x).any()), np.dtype(str(x.dtype).replace("torch.", ""))
    else:
        if np.isfinite(x).all():
            return
        nan, dtype = bool(np.isnan(x).any()), x.dtype
    if nan:
        raise ValueError("Input X contains NaN.")
    raise ValueError(f"Input X contains infinity or a value too large for {dtype!r}.")


# DBSCAN's NearestNeighbors(radius=eps) keeps the default n_neighbors=5, and algorithm="auto" searches by brute force when
# 5 >= n // 2.  That path compares |x|^2 - 2 x.y + |y|^2 (BLAS norms and a GEMM) with eps^2, not the KD tree's
# (dx^2 + dy^2) + dz^2, and the two disagree on pairs within rounding of eps: such clouds go to scikit-learn itself.
_BRUTE_MAX_N = 11


def _host_dbscan(X: np.ndarray, eps: float, min_samples: int) -> Tuple[np.ndarray, np.ndarray]:
    try:
        from sklearn.cluster import DBSCAN as SkDBSCAN
    except ImportError as e:
        raise L.TgnError(f"dbscan: clouds of at most {_BRUTE_MAX_N} points take scikit-learn's brute-force path on the host, "
                         f"and scikit-learn cannot be imported ({e})") from e
    DBSCAN.host_fits += 1
    ref = SkDBSCAN(eps=eps, min_samples=min_samples).fit(X)
    return ref.labels_.astype(np.int64), ref.core_sample_indices_.astype(np.int64)


def dbscan(points, eps: float = 0.03, min_samples: int = 30) -> Tuple[np.ndarray, np.ndarray]:
    """numpy or tensor (n,3) -> (labels_ int64 (n), core_sample_indices_ int64) like the attributes of a fitted sklearn DBSCAN.
    Non-finite coordinates raise scikit-learn's ValueError; clouds of 1 to 11 points are fitted by scikit-learn on the host."""
    host = None if isinstance(points, torch.Tensor) else np.asarray(points)
    pts = points.float() if host is None else host
    if pts.ndim != 2 or pts.shape[1] != 3:
        raise L.TgnError(f"dbscan expects (n,3) points, got {tuple(pts.shape)}")
    _check_finite(pts)
    if host is not None:
        pts = torch.as_tensor(_as_float32(host))
    if 1 <= pts.shape[0] <= _BRUTE_MAX_N:
        # the caller's array as it is: the brute-force path rounds differently on float32 and float64 input
        return _host_dbscan(pts.cpu().numpy() if host is None else host, eps, min_samples)
    if not pts.is_cuda and not torch.cuda.is_available():
        raise L.TgnError("dbscan needs a CUDA device (there is no CPU path)")
    pts = pts if pts.is_cuda else pts.cuda()
    labels, core = dbscan_device(pts, eps, min_samples)
    both = torch.stack([labels, core.int()]).cpu().numpy()             # one device -> host copy
    return both[0].astype(np.int64), np.flatnonzero(both[1]).astype(np.int64)


class DBSCAN:
    """The slice of ``sklearn.cluster.DBSCAN`` the reference uses -- ``DBSCAN(eps=..., min_samples=...).fit(X, y)`` then
    ``.labels_`` / ``.core_sample_indices_`` / ``.components_`` -- on csrc/dbscan.cu: ops_utils.py:28,98, tsegnet.py:59,
    inference_pipeline_tsegnet.py:39.  Euclidean metric only, which is all the reference asks for.  Fits of 1 to 11 points, which
    scikit-learn searches by brute force, are scikit-learn's own and counted in ``host_fits``."""

    host_fits = 0

    def __init__(self, eps: float = 0.5, *, min_samples: int = 5, metric: str = "euclidean", **unsupported):
        if metric != "euclidean" or any(v is not None for v in unsupported.values()):
            raise L.TgnError(f"DBSCAN: only the Euclidean metric with default options is implemented (got metric={metric!r}, {unsupported})")
        self.eps, self.min_samples = eps, min_samples

    def fit(self, X, y=None, sample_weight=None):
        if sample_weight is not None:
            raise L.TgnError("DBSCAN: sample_weight is not implemented")
        X = np.asarray(X)
        if X.ndim != 2 or X.shape[1] != 3:
            raise L.TgnError(f"DBSCAN: expected (n, 3) points, got {X.shape}")
        self.labels_, self.core_sample_indices_ = dbscan(X, self.eps, self.min_samples)
        self.components_ = X[self.core_sample_indices_].copy()
        self.n_features_in_ = 3
        return self

    def fit_predict(self, X, y=None, sample_weight=None):
        return self.fit(X, y, sample_weight).labels_


def _explained_variance(points: np.ndarray) -> np.ndarray:
    """sklearn PCA(n_components=3).fit(points).explained_variance_ (ops_utils.get_eg_values :51-56): eigenvalues of the
    sample covariance, descending."""
    if points.shape[0] < 3:
        return np.array([0, 0, 0])
    x = np.asarray(points, dtype=np.float64)
    x = x - x.mean(0)
    ev = np.linalg.eigvalsh(x.T @ x / (x.shape[0] - 1))[::-1]
    return np.maximum(ev, 0.0)


def _majority(rows: np.ndarray) -> np.ndarray:
    """per row: the most frequent value, the smallest one among equals (np.unique + argmax, ops_utils.py:139-141)."""
    values, inv = np.unique(rows, return_inverse=True)
    inv = inv.reshape(rows.shape)
    counts = np.zeros((rows.shape[0], values.shape[0]), dtype=np.int32)
    np.add.at(counts, (np.arange(rows.shape[0])[:, None], inv), 1)
    return values[np.argmax(counts, axis=1)]


def get_clustering_labels(moved_points, labels):
    """Drop-in for ops_utils.get_clustering_labels (:86-144): moved_points (N,3), labels (N,) or (N,1) semantic classes ->
    cluster label of every foreground point (labels != 0), int64.  Non-finite foreground coordinates raise scikit-learn's
    ValueError, as the reference's DBSCAN.fit does."""
    moved_points = np.asarray(moved_points)
    cond = np.asarray(labels) != 0
    fg = moved_points[cond, :]
    _check_finite(fg)
    if not torch.cuda.is_available():
        raise L.TgnError("get_clustering_labels needs a CUDA device (there is no CPU path)")
    fg_dev = torch.as_tensor(_as_float32(fg)).cuda()
    lab_dev, core_dev = dbscan_device(fg_dev, 0.03, 30)
    both = torch.stack([lab_dev, core_dev.int()]).cpu().numpy()
    clustering_labels = both[0].astype(np.int64)
    core_mask = both[1].astype(bool)
    dbscan_labels = clustering_labels.copy()

    uniq = [int(u) for u in np.unique(dbscan_labels) if u != -1]
    eg_values = np.array([_explained_variance(fg[core_mask & (dbscan_labels == u), :3]) for u in uniq])
    eg_first = eg_values[:, 0]
    order = np.argsort(-eg_first)
    eg_first = eg_first[order]
    suspicious = []
    for i in range(3):
        with np.errstate(invalid="ignore", divide="ignore"):
            if eg_first[i] / eg_first[3:].mean() > 8:
                suspicious.append(order[i])
    for idx, which in enumerate(suspicious):
        # the reference indexes its list of clusters by position and then rewrites the label equal to that position (:128-132)
        members = fg[dbscan_labels == uniq[which], :3].astype(np.float64)
        split = MeanShift(bandwidth=0.07).fit(members)
        clustering_labels[clustering_labels == which] = split.labels_ + 100 * (idx + 1)

    noise = clustering_labels == -1
    if noise.any():          # (with no noise at all the reference raises ValueError from KDTree.query on an empty array, :135)
        keep = ~noise
        if int(keep.sum()) < 10:
            raise ValueError("k must be less than or equal to the number of training points")
        near = crops.nearest_neighbor_crops(fg_dev[torch.as_tensor(keep).cuda()].unsqueeze(0), fg_dev[torch.as_tensor(noise).cuda()].unsqueeze(0), 10)[0]
        clustering_labels[noise] = _majority(clustering_labels[keep][near.cpu().numpy()])
    return clustering_labels


def accelerate(ops_utils_module) -> None:
    """Swap ops_utils.get_clustering_labels of an imported reference module for the device version, and the ``DBSCAN`` name the module
    imported from scikit-learn (``clustering_points(method="dbscan")``, ops_utils.py:28) for the class above."""
    ops_utils_module.get_clustering_labels = get_clustering_labels
    accelerate_dbscan(ops_utils_module)


def accelerate_dbscan(module) -> None:
    """Point a module's ``DBSCAN`` name (``from sklearn.cluster import DBSCAN`` in ops_utils.py, models/modules/tsegnet.py,
    inference_pipelines/inference_pipeline_tsegnet.py) at the device implementation."""
    if hasattr(module, "DBSCAN"):
        module.DBSCAN = DBSCAN


_KMEANS_MAX_K = 64


def kmeans_device(X: torch.Tensor, offsets: torch.Tensor, k: int, first: torch.Tensor, uniforms: torch.Tensor, tol: torch.Tensor,
                  max_iter: int = 300):
    """A batch of k-means++ / Lloyd fits on csrc/kmeans.cu, one CTA each.  X (N,3) float32 CUDA, the fits' points already
    centred, fit f at rows offsets[f]:offsets[f+1] (int32, B+1); first (B) int32, uniforms (B, k-1, 2+int(log k)) float64 and tol
    (B) float32 as ``KMeans.fit`` draws and computes them.  Returns (labels (N) int32, init (B,k) int64, centres (B,k,3) float32
    centred, n_iter (B) int32, inertia (B) float32, relocated (B) int32), all on the device."""
    L.require_cuda(X, offsets, first, uniforms, tol)
    B = offsets.numel() - 1
    N = X.shape[0]
    if X.dim() != 2 or X.shape[1] != 3 or X.dtype != torch.float32:
        raise L.TgnError(f"kmeans expects (n,3) float32 points, got {tuple(X.shape)} {X.dtype}")
    if not 1 <= k <= _KMEANS_MAX_K:
        raise L.TgnError(f"kmeans: 1 <= n_clusters <= {_KMEANS_MAX_K} is implemented, got {k}")
    dev = X.device
    X, offsets, first, tol = X.contiguous(), offsets.int().contiguous(), first.int().contiguous(), tol.float().contiguous()
    uniforms = uniforms.double().contiguous()
    labels = torch.empty(N, dtype=torch.int32, device=dev)
    init = torch.empty(B, k, dtype=torch.int64, device=dev)
    centres = torch.empty(B, k, 3, dtype=torch.float32, device=dev)
    n_iter = torch.empty(B, dtype=torch.int32, device=dev)
    inertia = torch.empty(B, dtype=torch.float32, device=dev)
    relocated = torch.empty(B, dtype=torch.int32, device=dev)
    if B:
        ws = torch.empty(int(L.load().tgn_kmeans_bytes(N, B)), dtype=torch.uint8, device=dev)
        L.call("tgn_kmeans", B, N, int(k), int(max_iter), L.ptr(offsets), L.ptr(X), L.ptr(first), L.ptr(uniforms) if k > 1 else None,
               L.ptr(tol), L.ptr(ws), L.ptr(labels), L.ptr(init), L.ptr(centres), L.ptr(n_iter), L.ptr(inertia), L.ptr(relocated),
               L.stream_ptr())
    return labels, init, centres, n_iter, inertia, relocated


def _random_state(seed) -> np.random.RandomState:
    """sklearn.utils.check_random_state: numpy's global generator for None, a new one for an int, the instance itself"""
    if seed is None or seed is np.random:
        return np.random.mtrand._rand
    if isinstance(seed, (int, np.integer)):
        return np.random.RandomState(seed)
    if isinstance(seed, np.random.RandomState):
        return seed
    raise ValueError(f"{seed!r} cannot be used to seed a numpy.random.RandomState instance")


def kmeans_prepare(X: np.ndarray, k: int, tol: float, rs: np.random.RandomState):
    """What ``KMeans.fit`` computes on the host before its k-means++ seeding, with the same numpy calls on the same arrays, and
    the draws of ``_kmeans_plusplus`` on ``rs``: (X - X.mean(0) float32, X.mean(0), float32 tolerance, first index,
    (k-1, 2 + int(log k)) float64 uniforms).  The draws do not depend on the data, so ``rs`` ends where scikit-learn leaves it."""
    X = np.array(X, dtype=np.float32, order="C", copy=True)
    n = X.shape[0]
    sw = np.ones(n, dtype=np.float32)
    tol = np.float32(np.mean(np.var(X, axis=0)) * tol if tol != 0 else 0)
    x_mean = X.mean(axis=0)
    X -= x_mean
    trials = 2 + int(np.log(k))
    first = int(rs.choice(n, p=sw / sw.sum()))
    u = np.stack([rs.uniform(size=trials) for _ in range(k - 1)]) if k > 1 else np.zeros((0, trials))
    return X, x_mean, tol, first, u


class KMeans:
    """The slice of ``sklearn.cluster.KMeans`` the reference uses -- ``KMeans(k, init="k-means++").fit(points)`` then
    ``.labels_`` / ``.cluster_centers_`` / ``.inertia_`` / ``.n_iter_`` (ops_utils.py:32 in ``clustering_points`` and
    ``find_k_kmeans``) -- on csrc/kmeans.cu, on float32 (n, 3) points.

    The host makes exactly scikit-learn's numpy calls (tolerance, mean, the generator draws of k-means++ on the generator
    ``check_random_state(random_state)`` returns, so the global one for ``random_state=None``) and the device does the rest with
    single-threaded scikit-learn's float32 rounding: labels, centres and ``n_iter_`` equal its own.  A fit in which a cluster
    empties is redone by scikit-learn itself from the generator state saved before the draws; ``host_fits`` counts those."""

    host_fits = 0

    def __init__(self, n_clusters: int = 8, *, init="k-means++", n_init="auto", max_iter: int = 300, tol: float = 1e-4,
                 verbose: int = 0, random_state=None, copy_x: bool = True, algorithm: str = "lloyd"):
        if (not isinstance(init, str) or init != "k-means++" or n_init not in ("auto", 1) or algorithm != "lloyd" or verbose
                or copy_x is not True):
            raise L.TgnError(f"KMeans: only init='k-means++', n_init='auto' or 1, algorithm='lloyd', verbose=0, copy_x=True is "
                             f"implemented (got init={init!r}, n_init={n_init!r}, algorithm={algorithm!r}, verbose={verbose!r}, "
                             f"copy_x={copy_x!r})")
        self.n_clusters, self.init, self.n_init, self.max_iter, self.tol = int(n_clusters), init, n_init, int(max_iter), tol
        self.verbose, self.random_state, self.copy_x, self.algorithm = verbose, random_state, copy_x, algorithm

    def fit(self, X, y=None, sample_weight=None):
        if sample_weight is not None:
            raise L.TgnError("KMeans: sample_weight is not implemented")
        X = X.detach().cpu().numpy() if isinstance(X, torch.Tensor) else np.asarray(X)
        if X.dtype != np.float32 or X.ndim != 2 or X.shape[1] != 3:
            raise L.TgnError(f"KMeans: expected (n, 3) float32 points, got {X.shape} {X.dtype}")
        if not np.isfinite(X).all():
            raise ValueError("Input X contains NaN or infinity.")
        n, k = X.shape[0], self.n_clusters
        if n < k:
            raise ValueError(f"n_samples={n} should be >= n_clusters={k}.")
        if not 1 <= k <= _KMEANS_MAX_K:
            raise L.TgnError(f"KMeans: 1 <= n_clusters <= {_KMEANS_MAX_K} is implemented, got {k}")
        if not torch.cuda.is_available():
            raise L.TgnError("KMeans needs a CUDA device (there is no CPU path)")
        rs = _random_state(self.random_state)
        saved = rs.get_state()
        X0 = X
        X, x_mean, tol, first, u = kmeans_prepare(X, k, self.tol, rs)
        trials = u.shape[1]
        host = [np.array([0, n], np.int32), np.array([first], np.int32), np.array([tol], np.float32)]
        dev = [torch.from_numpy(a).cuda() for a in host]
        labels, init, centres, n_iter, inertia, relocated = kmeans_device(
            torch.from_numpy(X).cuda(), dev[0], k, dev[1], torch.from_numpy(u.reshape(1, k - 1, trials)).cuda(), dev[2], self.max_iter)
        small = torch.cat([n_iter.double(), inertia.double(), relocated.double()]).cpu().numpy()
        if small[2]:
            from sklearn.cluster import KMeans as SkKMeans
            type(self).host_fits += 1
            rs.set_state(saved)
            ref = SkKMeans(k, init="k-means++", n_init=1, max_iter=self.max_iter, tol=self.tol, random_state=rs).fit(X0)
            self.labels_, self.cluster_centers_ = ref.labels_, ref.cluster_centers_
            self.inertia_, self.n_iter_ = ref.inertia_, ref.n_iter_
        else:
            self.labels_ = labels.cpu().numpy()
            self.cluster_centers_ = centres[0].cpu().numpy() + x_mean
            self.inertia_, self.n_iter_ = float(np.float32(small[1])), int(small[0])
            self.init_indices_ = init[0].cpu().numpy()
        self.n_features_in_ = 3
        return self

    def fit_predict(self, X, y=None, sample_weight=None):
        return self.fit(X, y, sample_weight).labels_


def accelerate_kmeans(module) -> None:
    """Point a module's ``KMeans`` name (``from sklearn.cluster import KMeans`` in ops_utils.py) at the device implementation."""
    if hasattr(module, "KMeans"):
        module.KMeans = KMeans


_MS_LEAF_SIZE = 30          # NearestNeighbors' default leaf_size, the tree MeanShift.fit queries


def meanshift_device(Xt: torch.Tensor, idx: torch.Tensor, nodes: torch.Tensor, bounds: torch.Tensor, bandwidth: float,
                     max_iter: int = 300) -> torch.Tensor:
    """Every seed's ascent of ``MeanShift(bandwidth, max_iter).fit`` on csrc/meanshift.cu, one warp per seed.  The tree is
    scikit-learn's ``KDTree(X, leaf_size=30).get_arrays()`` on the device: Xt (n,3) float64 = X[idx_array], idx (n) int64 =
    idx_array, nodes (n_nodes,3) int32 = idx_start, idx_end, is_leaf, bounds (2,n_nodes,3) float64 = node_bounds.  Returns one
    uint8 buffer of n * 36 bytes: (n,3) float64 final means, then (n,3) int32 member counts, iterations and flags, by index in X
    (``meanshift_unpack``)."""
    L.require_cuda(Xt, idx, nodes, bounds)
    if Xt.dim() != 2 or Xt.shape[1] != 3 or Xt.dtype != torch.float64:
        raise L.TgnError(f"meanshift expects (n,3) float64 points, got {tuple(Xt.shape)} {Xt.dtype}")
    n = Xt.shape[0]
    Xt, idx, nodes, bounds = Xt.contiguous(), idx.long().contiguous(), nodes.int().contiguous(), bounds.double().contiguous()
    if idx.numel() != n or nodes.dim() != 2 or nodes.shape[1] != 3 or tuple(bounds.shape) != (2, nodes.shape[0], 3):
        raise L.TgnError(f"meanshift: inconsistent tree arrays idx {tuple(idx.shape)} nodes {tuple(nodes.shape)} bounds {tuple(bounds.shape)}")
    out = torch.empty(36 * n, dtype=torch.uint8, device=Xt.device)
    if n:
        means, info = out[:24 * n].view(torch.float64), out[24 * n:].view(torch.int32)
        L.call("tgn_meanshift", n, int(nodes.shape[0]), L.ptr(Xt), L.ptr(idx), L.ptr(nodes), L.ptr(bounds), float(bandwidth),
               1e-3 * bandwidth, int(max_iter), L.ptr(means), L.ptr(info), L.stream_ptr())
    return out


def meanshift_unpack(buf: np.ndarray):
    """the host copy of ``meanshift_device``'s buffer -> (means (n,3) float64, counts (n), iterations (n), flags (n) bool)"""
    n = buf.size // 36
    means = buf[:24 * n].view(np.float64).reshape(n, 3)
    info = buf[24 * n:].view(np.int32).reshape(n, 3)
    return means, info[:, 0].astype(np.int64), info[:, 1].astype(np.int64), info[:, 2].astype(bool)


def meanshift_tree(X: np.ndarray):
    """scikit-learn's ``KDTree(X, leaf_size=30)`` (the tree ``NearestNeighbors(radius=...).fit(X)`` builds for n >= 12) as the
    kernel's arrays: (Xt, idx_array, nodes (n_nodes,3) int32, node_bounds), built by scikit-learn on the host -- the reference
    the device build of ``MeanShift.fit`` is tested against."""
    from sklearn.neighbors import KDTree
    _, idx, node_data, bounds = KDTree(X, leaf_size=_MS_LEAF_SIZE).get_arrays()
    nodes = np.stack([node_data["idx_start"], node_data["idx_end"], node_data["is_leaf"]], axis=1).astype(np.int32)
    return np.ascontiguousarray(X[idx]), np.asarray(idx, np.int64), nodes, np.ascontiguousarray(bounds)


def meanshift_postprocess(X: np.ndarray, means: np.ndarray, counts: np.ndarray, iters: np.ndarray, bandwidth: float, n_jobs=None):
    """``MeanShift.fit`` after the seed ascent, made with scikit-learn's own calls: the intensity dict keyed by the mean tuples,
    the (intensity, tuple) ranking, the near-duplicate pass and the nearest-centre labels -> (cluster_centers_, labels_, n_iter_)."""
    from sklearn.neighbors import NearestNeighbors
    center_intensity = {}
    for mean, c in zip(map(tuple, means), counts.tolist()):
        if c:
            center_intensity[mean] = c
    n_iter = int(max(iters.tolist()))
    if not center_intensity:
        raise ValueError(f"No point was within bandwidth={bandwidth:f} of any seed. Try a different seeding strategy "
                         f"                             or increase the bandwidth.")
    ranked = sorted(center_intensity.items(), key=lambda tup: (tup[1], tup[0]), reverse=True)
    sorted_centers = np.array([tup[0] for tup in ranked])
    unique = np.ones(len(sorted_centers), dtype=bool)
    nbrs = NearestNeighbors(radius=bandwidth, n_jobs=n_jobs).fit(sorted_centers)
    for i, center in enumerate(sorted_centers):
        if unique[i]:
            unique[nbrs.radius_neighbors([center], return_distance=False)[0]] = 0
            unique[i] = 1
    cluster_centers = sorted_centers[unique]
    _, idxs = NearestNeighbors(n_neighbors=1, n_jobs=n_jobs).fit(cluster_centers).kneighbors(X)
    return cluster_centers, idxs.flatten(), n_iter


def meanshift_seed_host(X: np.ndarray, seed: np.ndarray, nbrs, bandwidth: float, max_iter: int):
    """one seed's ascent with scikit-learn's public calls (``radius_neighbors``, ``np.mean``, ``np.linalg.norm``), for the seeds
    the kernel flags -> (mean, count, iterations)"""
    stop_thresh = 1e-3 * bandwidth
    it = 0
    mean = seed
    while True:
        members = nbrs.radius_neighbors([mean], bandwidth, return_distance=False)[0]
        within = X[members]
        if len(within) == 0:
            break
        old = mean
        mean = np.mean(within, axis=0)
        if np.linalg.norm(mean - old) <= stop_thresh or it == max_iter:
            break
        it += 1
    return mean, len(within), it


class MeanShift:
    """The slice of ``sklearn.cluster.MeanShift`` the reference uses -- ``MeanShift(bandwidth=0.07).fit(points)`` then
    ``.labels_`` (ops_utils.py:130 in ``get_clustering_labels``), plus ``.cluster_centers_`` / ``.n_iter_`` -- with the seed
    ascent on csrc/meanshift.cu, on float64 (n, 3) points.

    scikit-learn's own ``KDTree(X, leaf_size=30)`` is built on the device (``neighbors.sklearn_tree``, bit for bit) and stays
    there; every seed climbs on the device with scikit-learn's float64 rounding.  Seeds the kernel flags (a distance or a step within 2^-40 relative of the radius or
    the stop threshold, where scikit-learn's node bounds or another BLAS order could decide otherwise) are redone with
    scikit-learn's public calls and counted in ``host_seeds``.  The post-processing is scikit-learn's, so cluster_centers_,
    labels_ and n_iter_ are its own.  Inputs of at most 11 points, which scikit-learn searches by brute force, go to scikit-learn
    whole (``host_fits``)."""

    host_seeds = 0
    host_fits = 0

    def __init__(self, bandwidth=None, *, seeds=None, bin_seeding=False, min_bin_freq=1, cluster_all=True, n_jobs=None,
                 max_iter=300):
        if bandwidth is None or seeds is not None or bin_seeding or min_bin_freq != 1 or cluster_all is not True:
            raise L.TgnError(f"MeanShift: only an explicit bandwidth with seeds=None, bin_seeding=False, min_bin_freq=1, "
                             f"cluster_all=True is implemented (got bandwidth={bandwidth!r}, seeds={'given' if seeds is not None else None}, "
                             f"bin_seeding={bin_seeding!r}, min_bin_freq={min_bin_freq!r}, cluster_all={cluster_all!r})")
        if not (isinstance(bandwidth, (int, float, np.integer, np.floating)) and np.isfinite(bandwidth) and bandwidth > 0):
            raise L.TgnError(f"MeanShift: bandwidth must be a positive finite number, got {bandwidth!r}")
        if not (isinstance(max_iter, (int, np.integer)) and 0 <= max_iter < 2 ** 31):
            raise L.TgnError(f"MeanShift: max_iter must be a non-negative int, got {max_iter!r}")
        self.bandwidth, self.seeds, self.bin_seeding, self.min_bin_freq = bandwidth, seeds, bin_seeding, min_bin_freq
        self.cluster_all, self.n_jobs, self.max_iter = cluster_all, n_jobs, int(max_iter)

    def fit(self, X, y=None):
        X = X.detach().cpu().numpy() if isinstance(X, torch.Tensor) else np.asarray(X)
        if X.dtype != np.float64 or X.ndim != 2 or X.shape[1] != 3:
            raise L.TgnError(f"MeanShift: expected (n, 3) float64 points, got {X.shape} {X.dtype}")
        from sklearn.utils import check_array
        X = check_array(X, dtype=np.float64, order="C")              # scikit-learn's ValueError for NaN, inf and n = 0
        n, r = X.shape[0], float(self.bandwidth)
        if n < 12:                                                    # NearestNeighbors picks brute force below 12 points
            from sklearn.cluster import MeanShift as SkMeanShift
            type(self).host_fits += 1
            ref = SkMeanShift(bandwidth=self.bandwidth, n_jobs=self.n_jobs, max_iter=self.max_iter).fit(X)
            self.cluster_centers_, self.labels_, self.n_iter_ = ref.cluster_centers_, ref.labels_, ref.n_iter_
            self.n_features_in_ = 3
            return self
        if not torch.cuda.is_available():
            raise L.TgnError("MeanShift needs a CUDA device (there is no CPU path)")
        xyz, idx, node_data, bounds = neighbors.sklearn_tree(X, _MS_LEAF_SIZE, radius=False)
        tree = (xyz[idx], idx, node_data[:, :3].int(), bounds)
        means, counts, iters, flags = meanshift_unpack(meanshift_device(*tree, r, self.max_iter).cpu().numpy())
        flagged = np.flatnonzero(flags)
        if flagged.size:
            from sklearn.neighbors import NearestNeighbors
            type(self).host_seeds += int(flagged.size)
            nbrs = NearestNeighbors(radius=r, n_jobs=1).fit(X)
            means = means.copy()
            for i in flagged.tolist():
                means[i], counts[i], iters[i] = meanshift_seed_host(X, X[i], nbrs, r, self.max_iter)
        self.cluster_centers_, self.labels_, self.n_iter_ = meanshift_postprocess(X, means, counts, iters, r, self.n_jobs)
        self.n_features_in_ = 3
        return self

    def fit_predict(self, X, y=None):
        return self.fit(X).labels_
