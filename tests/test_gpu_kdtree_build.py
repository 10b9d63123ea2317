"""GPU: csrc/kdtree_build.cu through neighbors.sklearn_tree against scikit-learn's own KDTree build, bit for bit (idx_array,
node_data, node_bounds), on every case of the CPU tests, the fixture and dental arches; repeatability, guard bytes, refusals,
the tie fallback of neighbors.KDTree restoring the device tree without a host build, and MeanShift on the device tree."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle_kdtree import oracle  # noqa: E402
from toothgroupnetwork_b200 import _lib as L  # noqa: E402
from toothgroupnetwork_b200 import clouds, clustering, neighbors  # noqa: E402

pytestmark = pytest.mark.gpu
SkKDTree = pytest.importorskip("sklearn.neighbors").KDTree
sklearn_cluster = pytest.importorskip("sklearn.cluster")

FIX = np.load(os.path.join(ROOT, "tests", "golden", "ref_sklearn_kdtree.npz"))
FIX_NAMES = sorted({k[:-len("_points")] for k in FIX.files if k.endswith("_points")})
MS_FIX = np.load(os.path.join(ROOT, "tests", "golden", "ref_sklearn_meanshift.npz"))
MS_NAMES = sorted({k[:-len("_points")] for k in MS_FIX.files if k.endswith("_points")})


def device_arrays(X, leaf_size):
    xyz, idx, node_data, bounds = neighbors.sklearn_tree(X, leaf_size)
    assert xyz.dtype == torch.float64 and idx.dtype == torch.int64 and node_data.dtype == torch.int64
    return idx.cpu().numpy(), node_data.cpu().numpy(), bounds.cpu().numpy()


def assert_equal_sklearn(X, leaf_size, want=None):
    _, w_idx, w_nodes, w_bounds = SkKDTree(X, leaf_size=leaf_size).get_arrays() if want is None else (None,) + want
    idx, nodes, bounds = device_arrays(X, leaf_size)
    assert np.array_equal(idx, w_idx)
    assert nodes.tobytes() == np.ascontiguousarray(w_nodes).tobytes()
    assert bounds.shape == w_bounds.shape and bounds.tobytes() == w_bounds.tobytes()


@pytest.mark.parametrize("leaf_size", oracle.LEAF_SIZES)
def test_every_cpu_case_equals_sklearn(leaf_size):
    for name, X, ls in oracle.cases():
        if ls == leaf_size:
            try:
                assert_equal_sklearn(X, ls)
            except AssertionError as e:
                raise AssertionError(name) from e


@pytest.mark.parametrize("name", FIX_NAMES)
def test_fixture(name):
    want = (FIX[f"{name}_idx_array"], FIX[f"{name}_node_data"], FIX[f"{name}_node_bounds"])
    assert_equal_sklearn(FIX[f"{name}_points"], int(FIX[f"{name}_leaf_size"]), want)


def test_depth_limit_input():
    X = np.zeros((5000, 3))
    X[:, 0] = oracle.killer_adversary(5000)
    X[:, 1] = np.arange(5000) % 3 * 1e-9
    for leaf_size in (2, 40):
        assert_equal_sklearn(X, leaf_size)


def arch(n, seed, duplicates=False):
    X = clouds.dental_arch(n, seed)[0].double().numpy()
    if duplicates:
        rng = np.random.default_rng(seed)
        X[rng.choice(n, n // 5, replace=False)] = X[rng.choice(n, n // 5)]
    return X


@pytest.mark.parametrize("n", [24000, 44000, 200000])
@pytest.mark.parametrize("leaf_size", [2, 30, 40])
def test_arches(n, leaf_size):
    assert_equal_sklearn(arch(n, n % 97), leaf_size)
    assert_equal_sklearn(arch(n, n % 89, duplicates=True), leaf_size)


def test_two_builds_are_identical_and_radius_false_leaves_it_on_the_device():
    X = arch(44000, 3, duplicates=True)
    a = [t.cpu().numpy().tobytes() for t in neighbors.sklearn_tree(X, 2)]
    b = [t.cpu().numpy().tobytes() for t in neighbors.sklearn_tree(torch.from_numpy(X).cuda(), 2)]
    assert a == b
    xyz, idx, node_data, bounds = neighbors.sklearn_tree(X, 2, radius=False)
    nodes = node_data.cpu().numpy()
    assert np.isnan(nodes[:, 3].view(np.float64)).all()
    full = np.frombuffer(a[2], np.int64).reshape(-1, 4)
    assert np.array_equal(nodes[:, :3], full[:, :3]) and bounds.cpu().numpy().tobytes() == a[3]


def test_outputs_stay_inside_their_buffers():
    X = arch(30000, 4)
    n, leaf_size = X.shape[0], 2
    n_nodes = neighbors.tree_nodes(n, leaf_size)
    G = 4096
    xyz = torch.from_numpy(X).cuda()
    bufs = {name: torch.full((G + size + G,), 0x5A, dtype=torch.uint8, device="cuda")
            for name, size in (("idx", 8 * n), ("nodes", 32 * n_nodes), ("bounds", 48 * n_nodes),
                               ("ws", int(L.load().tgn_kdtree_bytes(n, leaf_size))))}
    inner = {k: v[G:-G] for k, v in bufs.items()}
    L.call("tgn_kdtree_build", n, leaf_size, L.ptr(xyz), L.ptr(inner["idx"]), L.ptr(inner["nodes"]), L.ptr(inner["bounds"]),
           L.ptr(inner["ws"]), L.stream_ptr())
    for name, buf in bufs.items():
        assert bool((buf[:G] == 0x5A).all()) and bool((buf[-G:] == 0x5A).all()), name
    _, w_idx, w_nodes, w_bounds = SkKDTree(X, leaf_size=leaf_size).get_arrays()
    assert np.array_equal(inner["idx"].cpu().numpy().view(np.int64), w_idx)
    assert inner["bounds"].cpu().numpy().tobytes() == w_bounds.tobytes()


def test_refusals_before_any_launch():
    before = L.launch_count()
    good = arch(100, 5)
    for X in (np.zeros((0, 3)), torch.zeros((0, 3), dtype=torch.float64, device="cuda")):
        with pytest.raises(ValueError):
            neighbors.sklearn_tree(X, 2)
    for bad_value in (np.nan, np.inf, -np.inf):
        bad = good.copy()
        bad[7, 1] = bad_value
        with pytest.raises(ValueError):
            neighbors.sklearn_tree(bad, 2)
        with pytest.raises(ValueError):
            neighbors.sklearn_tree(torch.from_numpy(bad).cuda(), 2)
    for leaf_size in (0, -1, 2.5, True):
        with pytest.raises(ValueError):
            neighbors.sklearn_tree(good, leaf_size)
    with pytest.raises(L.TgnError):
        neighbors.sklearn_tree(good[:, :2], 2)
    with pytest.raises(L.TgnError):
        neighbors.sklearn_tree(torch.from_numpy(good).cuda().float(), 2)
    assert L.launch_count() == before
    with pytest.raises(L.TgnError, match="n=0"):
        L.call("tgn_kdtree_build", 0, 2, None, None, None, None, None, L.stream_ptr())


# ------------------------------------------------------------------ the tie fallback of neighbors.KDTree.query
def tgn_final_transfer(m, seed):
    verts = clouds.dental_arch(m, seed)[0].numpy()
    rng = np.random.default_rng(seed)
    first = verts[rng.choice(m, 24000, replace=False)]
    bdl = verts[rng.choice(m, min(20000, m // 5), replace=False)]
    return np.concatenate([first, bdl]).astype(np.float32), verts.astype(np.float64)


def lattice(seed):
    pts = np.stack(np.meshgrid(*[np.arange(12) / 8.0] * 3, indexing="ij"), -1).reshape(-1, 3)
    return pts[np.random.default_rng(seed).permutation(pts.shape[0])]


def tied_cases():
    final, verts = tgn_final_transfer(100000, 11)
    yield final, verts, 1, 2
    yield final, verts, 1, 40
    pts = clouds.with_duplicates(clouds.dental_arch(12000, 12)[0], 12).double().numpy()
    for k in (1, 8, 40):
        yield pts, pts, k, 2
        yield pts, pts, k, 40
    pts = lattice(13)
    q = np.concatenate([pts[:800] + np.array([1.0, 0.5, 0.0]) / 16.0, np.random.default_rng(14).integers(-8, 200, (800, 3)) / 128.0])
    for k in (1, 8):
        yield pts, q, k, 2
        yield pts, q, k, 40


def test_tie_fallback_restores_the_device_tree_without_a_host_build(monkeypatch):
    real = neighbors.host_kdtree_class()

    class NoBuild(real):
        def __init__(self, *args, **kwargs):
            raise AssertionError("a scikit-learn KDTree was built on the host")

    monkeypatch.setattr(neighbors, "host_kdtree_class", lambda: NoBuild)
    for pts, q, k, leaf_size in tied_cases():
        ours = neighbors.KDTree(pts, leaf_size=leaf_size)
        d, i = ours.query(q, k=k)
        ind = ours.query(q, k=k, return_distance=False)
        ref = real(pts, leaf_size=leaf_size)
        wd, wi = ref.query(q, k=k)
        assert np.array_equal(i, wi) and np.array_equal(ind, wi) and d.tobytes() == wd.tobytes()
        assert isinstance(ours._host_tree, NoBuild)
        # host_rows counts the flagged rows of both queries, as the host-built tree did
        _, _, tie = ours.query_device(torch.from_numpy(np.asarray(q, np.float64)).cuda(), k)
        assert ours.host_rows == 2 * int(tie.sum()) > 0
        assert_same = [a.tobytes() for a in ours._host_tree.get_arrays()[1:]] == [np.ascontiguousarray(a).tobytes()
                                                                                   for a in ref.get_arrays()[1:]]
        assert assert_same


def test_unexpected_state_layout_builds_on_the_host(monkeypatch):
    monkeypatch.setattr(neighbors, "_state_ok", False)
    built = []
    real = neighbors.host_kdtree_class()

    class Counted(real):
        def __init__(self, *args, **kwargs):
            built.append(1)
            super().__init__(*args, **kwargs)

    monkeypatch.setattr(neighbors, "host_kdtree_class", lambda: Counted)
    pts = lattice(15)
    ours = neighbors.KDTree(pts, leaf_size=2)
    q = pts[:300] + 1.0 / 16.0
    assert np.array_equal(ours.query(q, k=1, return_distance=False), real(pts, leaf_size=2).query(q, k=1, return_distance=False))
    assert built == [1]


# ------------------------------------------------------------------ MeanShift on the device tree
def _no_host_tree(monkeypatch):
    def refused(X):
        raise AssertionError("clustering.meanshift_tree called")
    monkeypatch.setattr(clustering, "meanshift_tree", refused)


@pytest.mark.parametrize("name", MS_NAMES)
def test_meanshift_fixture_on_the_device_tree(name, monkeypatch):
    _no_host_tree(monkeypatch)
    X, r, max_iter = MS_FIX[f"{name}_points"], float(MS_FIX[f"{name}_bandwidth"]), int(MS_FIX[f"{name}_max_iter"])
    got = clustering.MeanShift(r, max_iter=max_iter).fit(X)
    assert np.asarray(got.cluster_centers_).tobytes() == np.asarray(MS_FIX[f"{name}_cluster_centers"], np.float64).tobytes()
    assert np.array_equal(got.labels_, MS_FIX[f"{name}_labels"]) and got.n_iter_ == int(MS_FIX[f"{name}_n_iter"])


@pytest.mark.parametrize("seed", range(4))
def test_meanshift_live_on_the_device_tree(seed, monkeypatch):
    _no_host_tree(monkeypatch)
    rng = np.random.default_rng(20 + seed)
    n = int(rng.choice([12, 40, 500, 1500]))
    centres = rng.uniform(-0.2, 0.2, (int(rng.integers(1, 6)), 3))
    X = centres[rng.integers(0, len(centres), n)] + rng.normal(0, 0.02 + 0.01 * seed, (n, 3))
    r = float(rng.choice([0.03, 0.07, 0.1]))
    got, ref = clustering.MeanShift(bandwidth=r).fit(X), sklearn_cluster.MeanShift(bandwidth=r).fit(X)
    assert np.asarray(got.cluster_centers_).tobytes() == np.asarray(ref.cluster_centers_).tobytes()
    assert got.labels_.dtype == ref.labels_.dtype and np.array_equal(got.labels_, ref.labels_) and got.n_iter_ == ref.n_iter_


def test_meanshift_lattice_at_the_bandwidth_on_the_device_tree(monkeypatch):
    _no_host_tree(monkeypatch)
    lat = np.stack(np.meshgrid(*[np.arange(5) * 0.5] * 3, indexing="ij"), -1).reshape(-1, 3)
    lat = lat[np.random.default_rng(0).permutation(len(lat))]
    got, ref = clustering.MeanShift(bandwidth=0.5).fit(lat), sklearn_cluster.MeanShift(bandwidth=0.5).fit(lat)
    assert np.asarray(got.cluster_centers_).tobytes() == np.asarray(ref.cluster_centers_).tobytes()
    assert np.array_equal(got.labels_, ref.labels_) and got.n_iter_ == ref.n_iter_
