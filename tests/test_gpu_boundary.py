"""GPU: the float64 grid kNN with the fused label vote (csrc/knn_f64.cu) against a float64 brute force and scikit-learn's KDTree,
and the boundary resampling drop-in against the reference's own InferencePipeLine.get_boundary_sampled_feats (skipped without the
staged reference snapshot)."""
import types

import numpy as np
import pytest
import torch

from toothgroupnetwork_b200 import _lib as L
from toothgroupnetwork_b200 import boundary, clouds

pytestmark = pytest.mark.gpu


def brute(points: torch.Tensor, queries: torch.Tensor, k: int, chunk: int = 2048):
    """float64 brute force, (dx*dx + dy*dy) + dz*dz with every operation rounded on its own (one torch op each), neighbours
    ordered by (d2, index) through a stable sort."""
    idx, dist = [], []
    for s in range(0, queries.shape[0], chunk):
        q = queries[s:s + chunk]
        dx = q[:, None, 0] - points[None, :, 0]
        dy = q[:, None, 1] - points[None, :, 1]
        dz = q[:, None, 2] - points[None, :, 2]
        d2 = (dx * dx + dy * dy) + dz * dz
        d2s, order = torch.sort(d2, dim=1, stable=True)
        idx.append(order[:, :k])
        dist.append(torch.sqrt(d2s[:, :k]))
    return torch.cat(idx), torch.cat(dist)


def arch64(n, seed):
    g = np.random.default_rng(seed)
    return torch.from_numpy(clouds.dental_arch(n, seed)[0].double().numpy() + g.normal(0.0, 1e-4, (n, 3))).cuda()


def check(points, queries, k):
    gi, gd = boundary.knn_f64(points, queries, k)
    wi, wd = brute(points, queries, k)
    assert gi.dtype == torch.int64 and gd.dtype == torch.float64 and gi.shape == (queries.shape[0], k)
    bad = int((gi != wi).any(1).sum())
    assert bad == 0, f"{bad} of {queries.shape[0]} queries differ"
    assert torch.equal(gd, wd)


def test_arch_24000_points_100000_queries():
    check(arch64(24000, 1), arch64(100000, 2), 40)


@pytest.mark.parametrize("k", [1, 3, 40, 64])
def test_k_values(k):
    check(arch64(24000, 3), arch64(20000, 4), k)


@pytest.mark.parametrize("k", [1, 3, 40, 64])
def test_exact_ties_at_every_rank(k):
    """every point twice: each distance is tied, including at the k-th rank (odd k splits a pair); the lower index wins"""
    pts = clouds.with_duplicates(clouds.dental_arch(12000, 5)[0], 5).double().cuda()
    q = torch.cat([pts[:3000], arch64(7000, 6)])
    check(pts, q, k)


def test_queries_far_outside_the_box():
    pts = arch64(24000, 7)
    base = arch64(4000, 8)
    q = torch.cat([base * 40.0 + 3.0, base - torch.tensor([0.0, 0.0, 25.0], dtype=torch.float64, device="cuda"),
                   torch.tensor([[1e6, -1e6, 5e5], [-3.0, 0.1, 0.0]], dtype=torch.float64, device="cuda")])
    check(pts, q, 40)


def test_planar_cloud():
    pts = arch64(20000, 9)
    pts[:, 2] = 0.25
    check(pts, arch64(10000, 10), 40)


def test_identical_points():
    pts = torch.full((300, 3), 0.125, dtype=torch.float64, device="cuda")
    check(pts, arch64(2000, 11), 64)


def test_n_equals_k():
    check(arch64(40, 12), arch64(3000, 13), 40)
    check(arch64(64, 14), arch64(3000, 15), 64)


def test_rejected_arguments():
    pts, q = arch64(50, 16), arch64(10, 17)
    for k in (0, 51, 65):
        with pytest.raises(L.TgnError):
            boundary.knn_f64(pts, q, k)
    with pytest.raises(L.TgnError):
        boundary.knn_f64(arch64(100, 18), q, 65)
    with pytest.raises(L.TgnError):
        boundary.knn_f64(pts.float(), q.float(), 4)
    bad = q.clone()
    bad[3, 1] = float("nan")
    with pytest.raises(L.TgnError):
        boundary.knn_f64(pts, bad, 4)


def test_against_sklearn_kdtree_200000_queries():
    from sklearn.neighbors import KDTree
    org, sampled, labels = clouds.boundary_inputs(200000, 21)
    pts, q = sampled[:, :3], org[:, :3]
    want_d, want_i = KDTree(pts, leaf_size=40).query(q, k=40)
    gi, gd = boundary.knn_f64(torch.from_numpy(pts).cuda(), torch.from_numpy(q).cuda(), 40)
    assert np.array_equal(gi.cpu().numpy(), want_i)
    assert np.array_equal(gd.cpu().numpy(), want_d)
    codes = boundary.label_codes(torch.from_numpy(labels).cuda())
    nn0, agree = boundary.neighbour_vote(torch.from_numpy(pts).cuda(), torch.from_numpy(q).cuda(), codes, 40)
    assert np.array_equal(nn0.cpu().numpy(), want_i[:, 0])
    assert np.array_equal(agree.cpu().numpy(), (labels[want_i] == labels[want_i[:, :1]]).sum(1))


def test_boundary_sample_device_path_matches_its_own_steps():
    org, sampled, labels = clouds.boundary_inputs(30000, 22, label_noise=0.1)
    dev = torch.device("cuda")
    perm = np.random.default_rng(0).permutation
    drawn = {}

    def draw(n):
        drawn["perm"] = perm(n)
        return drawn["perm"]

    feats, lab, bd_feats, bd_lab = boundary.boundary_sample(torch.from_numpy(sampled[:, :3]).to(dev), torch.from_numpy(labels).to(dev),
                                                            torch.from_numpy(org).to(dev), bdl_ratio=0.7, num_bdl=2000, num_all=6000,
                                                            perm=draw)
    idx, _ = boundary.knn_f64(torch.from_numpy(sampled[:, :3]).to(dev), torch.from_numpy(org[:, :3]).to(dev), 40)
    idx = idx.cpu().numpy()
    bd = (labels[idx] == labels[idx[:, :1]]).sum(1) / 40.0 < 0.7
    keep = np.flatnonzero(bd)[drawn["perm"][:2000]]
    assert bd_feats.dtype == torch.float64 and lab.dtype == torch.float64 and feats.shape == (6000, 6) and lab.shape == (6000, 1)
    assert np.array_equal(bd_feats.cpu().numpy(), org[keep])
    assert np.array_equal(bd_lab.cpu().numpy()[:, 0], labels[idx[keep, 0]])
    assert torch.equal(feats[:bd_feats.shape[0]], bd_feats)


# ------------------------------------------------------------------------------------ the reference method itself
def _reference_method():
    from oracle import ref_cuda, ref_models
    if not (ref_models.available() and ref_cuda.available()):
        pytest.skip("reference snapshot not staged")
    w = ref_models.World("reference")
    return w, import_in_world(w, "inference_pipelines.inference_pipeline_tgn").InferencePipeLine.get_boundary_sampled_feats


def import_in_world(world, name):
    """Import a reference module that the world does not preload, bound to that world's modules (gen_utils, ops_utils, models,
    the reference's pointops), and take its package back out of sys.modules so that nothing outside the world can see it."""
    import importlib
    import sys
    top = name.split(".")[0]
    mine = lambda: [n for n in sys.modules if n.split(".")[0] == top]
    with world:
        saved = {n: sys.modules.pop(n) for n in mine()}
        try:
            mod = importlib.import_module(name)
        finally:
            for n in mine():
                del sys.modules[n]
            sys.modules.update(saved)
    return mod


_REF = {}


def reference():
    if "m" not in _REF:
        _REF["m"] = _reference_method()
    return _REF["m"]


def _stand_in(bdl_ratio=0.7, num_bdl=20000, num_all=24000):
    return types.SimpleNamespace(config={"boundary_sampling_info": {"bdl_ratio": bdl_ratio, "num_of_bdl_points": num_bdl,
                                                                    "num_of_all_points": num_all}})


def _same_state(a, b):
    return a[0] == b[0] and np.array_equal(a[1], b[1]) and a[2:] == b[2:]


@pytest.mark.parametrize("m,noise,bdl_ratio,fewer", [(100000, 0.0, 0.7, True), (100000, 0.25, 0.7, False), (100000, 0.0, 0.0, True),
                                                     (200000, 0.0, 0.7, False)])
def test_drop_in_bitwise_equal_to_the_reference_method(m, noise, bdl_ratio, fewer):
    w, ref_method = reference()
    org, sampled, labels = clouds.boundary_inputs(m, 31, label_noise=noise)
    me = _stand_in(bdl_ratio)
    np.random.seed(1234)
    with w:
        want = ref_method(me, labels, org, sampled, None)
    want_state = np.random.get_state()
    np.random.seed(1234)
    got = boundary.get_boundary_sampled_feats(me, labels, org, sampled, None)
    assert _same_state(np.random.get_state(), want_state)
    assert (want[2].shape[0] < 20000) == fewer
    if bdl_ratio == 0.0:
        assert want[2].shape[0] == 0
    for g, r in zip(got, want):
        assert g.dtype == r.dtype and g.shape == r.shape
        assert np.array_equal(g, r)


def test_too_few_non_boundary_vertices_raise_in_both():
    w, ref_method = reference()
    org, sampled, labels = clouds.boundary_inputs(30000, 32)
    me = _stand_in(1.01)                          # every vertex is a boundary vertex: FPS has nothing to sample from
    with w, pytest.raises(Exception):
        ref_method(me, labels, org, sampled, None)
    with pytest.raises(L.TgnError):
        boundary.get_boundary_sampled_feats(me, labels, org, sampled, None)
