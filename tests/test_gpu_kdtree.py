"""GPU: the KDTree drop-in of the label transfers (toothgroupnetwork_b200.neighbors) against scikit-learn's KDTree with the same
leaf_size -- indices equal, distances bitwise equal, exact ties resolved by the host tree -- the tie flag of csrc/knn_f64.cu
against a float64 brute force of its definition, the refusals, and the reference's own get_boundary_sampled_feats(...,
sample_output_features) with its KDTree swapped (skipped without the staged reference snapshot)."""
import numpy as np
import pytest
import torch
from sklearn.neighbors import KDTree as SkKDTree

from toothgroupnetwork_b200 import _lib as L
from toothgroupnetwork_b200 import clouds, dropin, neighbors

pytestmark = pytest.mark.gpu


def arch(n, seed):
    """float64 arch vertices with float64 jitter: coordinates that are not float32 values, so distances do not tie"""
    return clouds.dental_arch(n, seed)[0].double().numpy() + np.random.default_rng(seed).normal(0.0, 1e-4, (n, 3))


def lattice(seed):
    """a shuffled 12^3 lattice in steps of 1/8: every d2 to a query in steps of 1/16 is exact, and ties are everywhere"""
    pts = np.stack(np.meshgrid(*[np.arange(12) / 8.0] * 3, indexing="ij"), -1).reshape(-1, 3)
    return pts[np.random.default_rng(seed).permutation(pts.shape[0])]


def same(points, queries, k, leaf_size, host_rows=None, **kw):
    """our KDTree against scikit-learn's: the same return structure, indices equal, distances bitwise equal"""
    ours = neighbors.KDTree(points, leaf_size=leaf_size)
    got = ours.query(queries, k=k, **kw)
    want = SkKDTree(points, leaf_size=leaf_size).query(queries, k=k, **kw)
    if kw.get("return_distance", True):
        assert got[0].dtype == np.float64 and got[1].dtype == np.intp and got[1].shape == want[1].shape
        assert np.array_equal(got[1], want[1]), f"{int((got[1] != want[1]).any(1).sum())} rows differ"
        assert np.array_equal(got[0], want[0])
    else:
        assert isinstance(got, np.ndarray) and got.dtype == np.intp and got.shape == want.shape
        assert np.array_equal(got, want)
    if host_rows == 0:
        assert ours.host_rows == 0
    elif host_rows == ">0":
        assert ours.host_rows > 0
    return ours


@pytest.mark.parametrize("leaf_size", [2, 40])
@pytest.mark.parametrize("k", [1, 3, 10, 40, 63])
def test_arch_without_ties_never_reaches_the_host(k, leaf_size):
    same(arch(24000, 1), arch(20000, 2), k, leaf_size, host_rows=0)


@pytest.mark.parametrize("leaf_size", [2, 40])
def test_far_queries_n_equals_k_and_a_single_point(leaf_size):
    pts, base = arch(24000, 3), arch(3000, 4)
    far = np.concatenate([base * 40.0 + 3.0, base - np.array([0.0, 0.0, 25.0]), np.array([[1e6, -1e6, 5e5], [-3.0, 0.1, 0.0]])])
    same(pts, far, 40, leaf_size, host_rows=0)
    same(arch(40, 5), arch(2000, 6), 40, leaf_size)
    same(arch(63, 7), arch(2000, 8), 63, leaf_size)
    same(arch(1, 9), arch(500, 10), 1, leaf_size, host_rows=0)


def tgn_final_transfer(m, seed):
    """the final tree of inference_pipeline_tgn.py:137-140: float32 copies of 24 000 first-network samples and up to 20 000
    boundary vertices, both drawn from the mesh's float32 vertices, so a vertex in both parts is in the tree twice; the queries
    are every mesh vertex"""
    verts = clouds.dental_arch(m, seed)[0].numpy()
    rng = np.random.default_rng(seed)
    first = verts[rng.choice(m, 24000, replace=False)]
    bdl = verts[rng.choice(m, min(20000, m // 5), replace=False)]
    return np.concatenate([first, bdl]).astype(np.float32), verts.astype(np.float64), first, bdl


@pytest.mark.parametrize("leaf_size", [2, 40])
def test_tgn_final_transfer_with_duplicates_resolves_ties_on_the_host(leaf_size):
    final, verts, _, _ = tgn_final_transfer(100000, 11)
    same(final, verts, 1, leaf_size, host_rows=">0", return_distance=False)
    same(final, verts, 1, leaf_size, host_rows=">0")


@pytest.mark.parametrize("k", [1, 8, 40])
def test_clouds_with_duplicates_queried_with_their_own_points(k):
    pts = clouds.with_duplicates(clouds.dental_arch(12000, 12)[0], 12).double().numpy()
    for leaf_size in (2, 40):
        same(pts, pts, k, leaf_size, host_rows=">0")


@pytest.mark.parametrize("k", [1, 8])
def test_lattice_ties_inside_k(k):
    pts = lattice(13)
    q = np.concatenate([pts[:800] + np.array([1.0, 0.5, 0.0]) / 16.0, np.random.default_rng(14).integers(-8, 200, (800, 3)) / 128.0])
    for leaf_size in (2, 40):
        same(pts, q, k, leaf_size, host_rows=">0")


def test_one_tree_queried_in_a_loop_of_cluster_subsets():
    """inference_pipeline_tgn.py:107-114: one tree on the first network's points, one k = 1 query per boundary cluster"""
    _, _, first, bdl = tgn_final_transfer(100000, 15)
    clusters = np.random.default_rng(15).integers(0, 17, bdl.shape[0])
    ours, sk = neighbors.KDTree(first, leaf_size=2), SkKDTree(first, leaf_size=2)
    for c in np.unique(clusters):
        sel = bdl[clusters == c]
        assert np.array_equal(ours.query(sel, k=1, return_distance=False), sk.query(sel, k=1, return_distance=False))
    d, i = ours.query(bdl, k=3)                   # the built grid is still intact after the loop
    wd, wi = sk.query(bdl, k=3)
    assert np.array_equal(i, wi) and np.array_equal(d, wd)


def test_float32_and_list_inputs():
    pts, q = arch(3000, 16).astype(np.float32), arch(500, 17).astype(np.float32)
    same(pts, q, 5, 40)
    same(pts.tolist(), q.tolist(), 5, 2, return_distance=False)


def brute(points: torch.Tensor, queries: torch.Tensor, k: int):
    """float64 brute force in the kernel's operation order, stably sorted by (d2, index), and the tie flag's definition: two
    adjacent equal d2 among the min(k+1, n) smallest keys"""
    dx, dy, dz = (queries[:, None, a] - points[None, :, a] for a in range(3))
    d2s, order = torch.sort((dx * dx + dy * dy) + dz * dz, dim=1, stable=True)
    keep = d2s[:, :min(k + 1, points.shape[0])]
    return order[:, :k], torch.sqrt(d2s[:, :k]), (keep[:, 1:] == keep[:, :-1]).any(1)


@pytest.mark.parametrize("k", [1, 8, 31, 32, 63])
def test_query_device_tie_flag_against_brute_force(k):
    pts = np.concatenate([lattice(18)[:1200], arch(800, 19), arch(800, 19)[:20]])      # exact ties, jittered points, duplicates
    q = np.concatenate([pts[::3] + 1.0 / 32.0, arch(1500, 20), pts[:400]])
    tree = neighbors.KDTree(pts)
    gi, gd, gt = tree.query_device(torch.from_numpy(q).cuda(), k)
    wi, wd, wt = brute(torch.from_numpy(pts).cuda(), torch.from_numpy(q).cuda(), k)
    assert gi.dtype == torch.int64 and gd.dtype == torch.float64 and gt.dtype == torch.uint8 and gt.shape == (q.shape[0],)
    assert torch.equal(gi, wi) and torch.equal(gd, wd)
    assert torch.equal(gt.bool(), wt)
    assert int(gt.sum()) > 0 and (k > 8 or not bool(gt.all()))
    # n = k: the flag looks at all n entries
    small = neighbors.KDTree(pts[:k])
    _, _, st = small.query_device(torch.from_numpy(q).cuda(), k)
    assert torch.equal(st.bool(), brute(torch.from_numpy(pts[:k]).cuda(), torch.from_numpy(q).cuda(), k)[2])


def test_refusals():
    pts = arch(100, 21)
    tree = neighbors.KDTree(pts)
    q = arch(10, 22)
    for bad_value in (np.nan, np.inf):
        bad = q.copy()
        bad[3, 1] = bad_value
        with pytest.raises(ValueError):
            tree.query(bad, k=1)
        with pytest.raises(ValueError):
            SkKDTree(pts).query(bad, k=1)
    with pytest.raises(ValueError, match="k must be less"):
        neighbors.KDTree(pts[:5]).query(q, k=6)
    with pytest.raises(ValueError, match="dimension"):
        tree.query(np.zeros((4, 2)), k=1)
    with pytest.raises(ValueError):
        tree.query(np.zeros(3), k=1)
    with pytest.raises(L.TgnError, match="metric"):
        neighbors.KDTree(pts, metric="chebyshev")
    with pytest.raises(L.TgnError, match="k <= 63"):
        tree.query(q, k=64)
    with pytest.raises(L.TgnError):
        tree.query(q, k=0)
    for kw in ({"dualtree": True}, {"breadth_first": True}, {"sort_results": False}):
        with pytest.raises(L.TgnError):
            tree.query(q, k=1, **kw)
    qd = torch.from_numpy(q).cuda()
    with pytest.raises(L.TgnError):
        tree.query_device(qd, 64)
    with pytest.raises(L.TgnError):
        tree.query_device(qd.float(), 1)
    with pytest.raises(L.TgnError):
        tree.query_device(torch.from_numpy(q), 1)
    nanq = qd.clone()
    nanq[0, 0] = float("nan")
    with pytest.raises(L.TgnError, match="non-finite"):
        tree.query_device(nanq, 1)
    # the C entry point refuses k = 64 with the tie flag and keeps k = 64 without it
    out = torch.empty((10, 64), dtype=torch.int64, device="cuda")
    tie = torch.empty(10, dtype=torch.uint8, device="cuda")
    with pytest.raises(L.TgnError, match="63"):
        L.call("tgn_knn_f64_query", 100, 10, 64, L.ptr(tree._xyz), L.ptr(qd), L.ptr(tree._ws), None, L.ptr(out), None, None, None,
               L.ptr(tie), L.stream_ptr())
    L.call("tgn_knn_f64_query", 100, 10, 64, L.ptr(tree._xyz), L.ptr(qd), L.ptr(tree._ws), None, L.ptr(out), None, None, None,
           None, L.stream_ptr())
    assert np.array_equal(out.cpu().numpy(), SkKDTree(pts).query(q, k=64)[1])


# ------------------------------------------------------------------------------------ the reference method itself
def _reference_tgn_module():
    """inference_pipelines.inference_pipeline_tgn imported inside a reference world (bound to that world's gen_utils, models and
    pointops), then taken back out of sys.modules so that nothing outside the world sees it"""
    import importlib
    import sys
    from oracle import ref_cuda, ref_models
    if not (ref_models.available() and ref_cuda.available()):
        pytest.skip("reference snapshot not staged")
    w = ref_models.World("reference")
    mine = lambda: [n for n in sys.modules if n.split(".")[0] == "inference_pipelines"]
    with w:
        saved = {n: sys.modules.pop(n) for n in mine()}
        try:
            mod = importlib.import_module("inference_pipelines.inference_pipeline_tgn")
        finally:
            for n in mine():
                del sys.modules[n]
            sys.modules.update(saved)
    return w, mod


def test_reference_sample_output_features_branch_with_the_kdtree_swapped():
    """the original get_boundary_sampled_feats with sample_output_features (KDTree k = 40 and k = 1 without distances, k = 3 with):
    its own scikit-learn KDTree, then ours after accelerate_label_transfer -- the four arrays bitwise equal, the same RNG state"""
    import types
    w, mod = _reference_tgn_module()
    org, sampled, labels = clouds.boundary_inputs(100000, 23)
    me = types.SimpleNamespace(config={"boundary_sampling_info": {"bdl_ratio": 0.7, "num_of_bdl_points": 20000,
                                                                  "num_of_all_points": 24000}})
    feats = torch.from_numpy(np.random.default_rng(23).standard_normal((1, 16, sampled.shape[0])).astype(np.float32))
    method = mod.InferencePipeLine.get_boundary_sampled_feats
    runs = []
    for swap in (False, True):
        if swap:
            dropin.accelerate_label_transfer(mod)
            assert mod.KDTree is neighbors.KDTree
        np.random.seed(4321)
        with w:
            out = method(me, labels, org, sampled, feats)
        runs.append((out, np.random.get_state()))
    (want, want_state), (got, got_state) = runs
    assert want_state[0] == got_state[0] and np.array_equal(want_state[1], got_state[1]) and want_state[2:] == got_state[2:]
    assert want[0].shape == (24000, 6 + 16)
    for g, r in zip(got, want):
        assert g.dtype == r.dtype and g.shape == r.shape
        assert np.array_equal(g, r)
