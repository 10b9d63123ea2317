"""GPU: csrc/kdtree_query.cu through neighbors.sklearn_query against scikit-learn's KDTree.query (indices and distance bytes)
and its flags against the oracle's; row lists and guard bytes; DeviceKDTree on the tied label transfers with the host class
unreachable; the tgn per-cluster loop through accelerate_label_transfer(ties="device"); refusals before any launch."""
import os
import sys
import types

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle_kdtree import oracle  # noqa: E402
from toothgroupnetwork_b200 import _lib as L  # noqa: E402
from toothgroupnetwork_b200 import clouds, dropin, neighbors  # noqa: E402

pytestmark = pytest.mark.gpu
SkKDTree = pytest.importorskip("sklearn.neighbors").KDTree

KS = (1, 2, 3, 8, 15, 16, 17, 40, 63)
INPUTS = list(oracle.tied_query_inputs(full=True))
ORACLE_ROWS = 100                     # rows per case whose flags are recomputed by the Python walk


def cases(k):
    """the tied inputs (tgn's final transfer at 10^5 vertices for k = 1, its first 2*10^4 vertices as queries otherwise),
    n = k, and a single point"""
    for name, pts, q in INPUTS:
        yield name, pts, q if k == 1 or name != "tgn_final" else q[:20000]
    yield "n_equals_k", INPUTS[1][1][:k], INPUTS[0][2][:2000]
    if k == 1:
        yield "single_point", INPUTS[1][1][:1], INPUTS[0][2][:500]


@pytest.mark.parametrize("leaf_size", oracle.LEAF_SIZES)
@pytest.mark.parametrize("k", KS)
def test_every_row_equals_sklearn_and_flags_equal_the_oracle(k, leaf_size):
    for name, pts, q in cases(k):
        tree = neighbors.sklearn_tree(pts, leaf_size, radius=False)
        dist, idx, flag = neighbors.sklearn_query(tree, torch.from_numpy(q).cuda(), k)
        dist, idx, flag = dist.cpu().numpy(), idx.cpu().numpy(), flag.cpu().numpy()
        ref = SkKDTree(pts, leaf_size=leaf_size)
        wd, wi = ref.query(q, k=k)
        ok = flag == 0
        assert np.array_equal(idx[ok], wi[ok]) and dist[ok].tobytes() == wd[ok].tobytes(), name
        # the flags of the flagged rows and of the first rows, recomputed by the oracle with the device's arithmetic
        rows = np.unique(np.concatenate([np.flatnonzero(flag)[:ORACLE_ROWS], np.arange(min(ORACLE_ROWS, q.shape[0]))]))
        _, s_idx, s_nodes, s_bounds = ref.get_arrays()
        od, oi, of = oracle.query(pts, s_idx, s_nodes, s_bounds, q[rows], k, square=oracle.exact_square)
        assert np.array_equal(of, flag[rows]), name
        assert np.array_equal(oi, idx[rows]) and od.tobytes() == dist[rows].tobytes(), name


def test_flagged_rows_where_pow_decides_otherwise():
    X, Q, leaf_size, k, rows = oracle.pow_decides_otherwise()
    tree = neighbors.sklearn_tree(X, leaf_size, radius=False)
    _, _, flag = neighbors.sklearn_query(tree, torch.from_numpy(Q).cuda(), k)
    flag = flag.cpu().numpy()
    assert flag[list(rows)].tolist() == [1] * len(rows)
    _, s_idx, s_nodes, s_bounds = SkKDTree(X, leaf_size=leaf_size).get_arrays()
    assert np.array_equal(oracle.query(X, s_idx, s_nodes, s_bounds, Q[:300], k, square=oracle.exact_square)[2], flag[:300])


def test_rows_write_only_those_rows_inside_their_buffers():
    _, pts, q = INPUTS[1]
    n, m, k, leaf_size = pts.shape[0], 5000, 8, 2
    q = q[:m]
    xyz, idx_array, node_data, bounds = neighbors.sklearn_tree(pts, leaf_size, radius=False)
    rows = np.sort(np.random.default_rng(1).choice(m, 700, replace=False))
    G = 4096
    bufs = {name: torch.full((G + size + G,), 0x5A, dtype=torch.uint8, device="cuda")
            for name, size in (("idx", 8 * m * k), ("dist", 8 * m * k), ("flag", m))}
    inner = {name: b[G:-G] for name, b in bufs.items()}
    queries = torch.from_numpy(q).cuda()
    rows_dev = torch.from_numpy(rows).cuda()
    L.call("tgn_kdtree_query", n, int(node_data.shape[0]), k, L.ptr(xyz), L.ptr(idx_array), L.ptr(node_data), L.ptr(bounds), m,
           L.ptr(queries), L.ptr(rows_dev), int(rows.size), L.ptr(inner["idx"]), L.ptr(inner["dist"]), L.ptr(inner["flag"]),
           L.stream_ptr())
    for name, b in bufs.items():
        assert bool((b[:G] == 0x5A).all()) and bool((b[-G:] == 0x5A).all()), name
    idx = inner["idx"].cpu().numpy().view(np.int64).reshape(m, k)
    dist = inner["dist"].cpu().numpy().view(np.float64).reshape(m, k)
    flag = inner["flag"].cpu().numpy()
    other = np.setdiff1d(np.arange(m), rows)
    untouched = np.full(8 * k, 0x5A, np.uint8)
    assert (idx[other].view(np.uint8) == untouched).all() and (dist[other].view(np.uint8) == untouched).all()
    assert (flag[other] == 0x5A).all() and (flag[rows] <= 1).all()
    wd, wi = SkKDTree(pts, leaf_size=leaf_size).query(q[rows], k=k)
    ok = flag[rows] == 0
    assert np.array_equal(idx[rows][ok], wi[ok]) and dist[rows][ok].tobytes() == wd[ok].tobytes()
    # the Python entry point with the same rows
    d2, i2, f2 = neighbors.sklearn_query((xyz, idx_array, node_data, bounds), queries, k, rows=rows)
    assert np.array_equal(i2.cpu().numpy()[rows], idx[rows]) and np.array_equal(f2.cpu().numpy()[rows], flag[rows])


# ------------------------------------------------------------------ DeviceKDTree: the tied rows walked on the device
def tied_cases():
    final, verts = INPUTS[0][1], INPUTS[0][2]
    yield final, verts, 1, 2
    yield final, verts, 1, 40
    pts = INPUTS[1][1]
    for k in (1, 8, 40):
        yield pts, pts, k, 2
        yield pts, pts, k, 40
    pts, q = INPUTS[2][1], INPUTS[2][2]
    for k in (1, 8):
        yield pts, q, k, 2
        yield pts, q, k, 40


def _unreachable_host_class(monkeypatch):
    def refused():
        raise AssertionError("the host KDTree class was reached")
    monkeypatch.setattr(neighbors, "host_kdtree_class", refused)


def test_device_tree_answers_tied_rows_without_the_host(monkeypatch):
    real = neighbors.host_kdtree_class()
    built = []
    real_sklearn_tree = neighbors.sklearn_tree
    monkeypatch.setattr(neighbors, "sklearn_tree", lambda *a, **kw: built.append(kw) or real_sklearn_tree(*a, **kw))
    for pts, q, k, leaf_size in tied_cases():
        q_dev = torch.from_numpy(np.asarray(q, np.float64)).cuda()
        ours = neighbors.DeviceKDTree(pts, leaf_size=leaf_size)
        _, _, tie = ours.query_device(q_dev, k)
        tied = np.flatnonzero(tie.cpu().numpy())
        assert tied.size > 0
        walk_flags = neighbors.sklearn_query(real_sklearn_tree(pts, leaf_size, radius=False), q_dev, k, rows=tied)[2]
        n_flagged = int(walk_flags.cpu().numpy()[tied].sum())
        print(f"tied case k={k} leaf_size={leaf_size}: {tied.size} tied rows, {n_flagged} flagged by the walk")
        if n_flagged == 0:
            _unreachable_host_class(monkeypatch)
        built.clear()
        d, i = ours.query(q, k=k)
        ind = ours.query(q, k=k, return_distance=False)
        wd, wi = real(pts, leaf_size=leaf_size).query(q, k=k)
        assert np.array_equal(i, wi) and np.array_equal(ind, wi) and d.tobytes() == wd.tobytes()
        assert ours.host_rows == 2 * n_flagged and ours.walk_rows == 2 * (tied.size - n_flagged)
        assert built == [{"radius": False}]                  # one device build, on the first tie
        monkeypatch.setattr(neighbors, "host_kdtree_class", lambda: real)


def test_device_tree_without_ties_builds_and_launches_nothing_more(monkeypatch):
    _unreachable_host_class(monkeypatch)
    monkeypatch.setattr(neighbors, "sklearn_tree", lambda *a, **kw: pytest.fail("tree built without a tie"))
    pts = clouds.dental_arch(24000, 1)[0].double().numpy()
    q = clouds.dental_arch(20000, 2)[0].double().numpy()
    ours = neighbors.DeviceKDTree(pts, leaf_size=2)
    before = L.launch_count()
    d, i = ours.query(q, k=1)
    assert L.launch_count() - before == 1 and ours.walk_rows == 0 and ours.host_rows == 0
    wd, wi = SkKDTree(pts, leaf_size=2).query(q, k=1)
    assert np.array_equal(i, wi) and d.tobytes() == wd.tobytes()


def test_unexpected_state_layout_keeps_ties_on_the_host(monkeypatch):
    monkeypatch.setattr(neighbors, "_state_ok", False)
    monkeypatch.setattr(neighbors, "sklearn_tree", lambda *a, **kw: pytest.fail("walk tree built"))
    pts, q = INPUTS[2][1], INPUTS[2][2]
    ours = neighbors.DeviceKDTree(pts, leaf_size=2)
    assert np.array_equal(ours.query(q, k=1, return_distance=False), SkKDTree(pts, leaf_size=2).query(q, k=1, return_distance=False))
    assert ours.host_rows > 0 and ours.walk_rows == 0


def test_tgn_cluster_loop_through_the_label_transfer_swap():
    """inference_pipeline_tgn.py:107-114: one tree on the first network's points, one k = 1 query per boundary cluster"""
    verts = clouds.dental_arch(100000, 15)[0].numpy()
    rng = np.random.default_rng(15)
    first = verts[rng.choice(100000, 24000)].astype(np.float64)      # drawn with replacement: duplicated points tie
    bdl = np.concatenate([first[rng.choice(24000, 8000, replace=False)],
                          verts[rng.choice(100000, 12000, replace=False)].astype(np.float64)])
    clusters = rng.integers(0, 17, bdl.shape[0])
    module = types.SimpleNamespace(KDTree=SkKDTree)
    dropin.accelerate_label_transfer(module, ties="device")
    ours, sk = module.KDTree(first, leaf_size=2), SkKDTree(first, leaf_size=2)
    assert isinstance(ours, neighbors.DeviceKDTree)
    for c in np.unique(clusters):
        sel = bdl[clusters == c]
        assert np.array_equal(ours.query(sel, k=1, return_distance=False), sk.query(sel, k=1, return_distance=False))
    # rows are independent: the tied and walk-flagged rows of the whole set are those of the per-cluster queries
    q_dev = torch.from_numpy(bdl).cuda()
    tied = np.flatnonzero(ours.query_device(q_dev, 1)[2].cpu().numpy())
    flagged = int(neighbors.sklearn_query(ours._walk_tree, q_dev, 1, rows=tied)[2].cpu().numpy()[tied].sum())
    print(f"tgn cluster loop: {tied.size} tied rows, {flagged} flagged by the walk")
    assert ours.walk_rows == tied.size - flagged > 0 and ours.host_rows == flagged


def test_refusals_before_any_launch():
    pts = clouds.dental_arch(500, 3)[0].double().numpy()
    tree = neighbors.sklearn_tree(pts, 2, radius=False)
    small = neighbors.sklearn_tree(pts[:5], 2, radius=False)
    q = torch.from_numpy(pts[:50]).cuda()
    before = L.launch_count()
    for bad, exc in (((torch.zeros((0, 3), dtype=torch.float64, device="cuda"),), ValueError),
                     ((q[:, :2].contiguous(),), ValueError),
                     ((q[0],), ValueError),
                     ((torch.where(torch.arange(50, device="cuda")[:, None] == 7, float("nan"), q),), ValueError),
                     ((q, 501), ValueError),
                     ((q, 0), L.TgnError),
                     ((q, 64), L.TgnError),
                     ((q.float(),), L.TgnError),
                     ((q.cpu(),), L.TgnError),
                     ((pts[:50],), L.TgnError)):
        with pytest.raises(exc):
            neighbors.sklearn_query(tree, *bad)
    with pytest.raises(ValueError):
        neighbors.sklearn_query(small, q, 8)
    with pytest.raises(L.TgnError):
        neighbors.sklearn_query(tree[:3], q)
    with pytest.raises(L.TgnError):
        neighbors.sklearn_query((tree[0], tree[1], tree[2][:2], tree[3]), q)
    with pytest.raises(L.TgnError):
        neighbors.sklearn_query(tree, q, 1, rows=[0, 50])
    with pytest.raises(L.TgnError):
        neighbors.sklearn_query(tree, q, 1, rows=[-1])
    neighbors.sklearn_query(tree, q, 1, rows=[])
    xyz, idx_array, node_data, bounds = tree
    with pytest.raises(L.TgnError, match="n_nodes"):
        L.call("tgn_kdtree_query", 500, 6, 1, L.ptr(xyz), L.ptr(idx_array), L.ptr(node_data), L.ptr(bounds), 50, L.ptr(q), None,
               0, None, None, None, L.stream_ptr())
    with pytest.raises(L.TgnError, match="k="):
        L.call("tgn_kdtree_query", 500, int(node_data.shape[0]), 64, L.ptr(xyz), L.ptr(idx_array), L.ptr(node_data),
               L.ptr(bounds), 50, L.ptr(q), None, 0, None, None, None, L.stream_ptr())
    assert L.launch_count() == before
