"""DBSCAN (csrc/dbscan.cu) one launch at a time, against an independent float64 reference of the same definition:

* neighbours: (dx*dx + dy*dy) + dz*dz <= eps*eps in float64, the point itself included (the predicate of scikit-learn's KD-tree
  search, which the kernel restates at every n);
* core: at least min_samples neighbours;
* clusters: connected components of the core-core edges, numbered in the order of their smallest member index;
* a border point takes the smallest label among its core neighbours; everything else is -1.

Every launch writes into sentinel-filled outputs and must leave no sentinel, give labels and core flags equal to the reference
and a device-side cluster count equal to labels.max() + 1.  The cases sit where the kernel could go wrong: lattice shells
exactly at eps (and one ulp inside), min_samples exactly at a neighbour count, border points between clusters whose numbering
disagrees with distance and with the cell scan, a 20 000-link chain for the union-find, 3 000 clusters for the numbering scan's
carry, grids wider than 64 eps, flat, inside one cell, far from the origin and tiny, thousands of coincident points, sizes
around the warp and block widths, reuse of the cached workspace, non-finite coordinates and the refusals.  Where scikit-learn
is importable the cases of 12 points or more are also compared with ``sklearn.cluster.DBSCAN`` itself."""
import itertools
import os

import numpy as np
import pytest
import torch
from scipy.sparse import coo_matrix
from scipy.sparse.csgraph import connected_components
from scipy.spatial import cKDTree

from toothgroupnetwork_b200 import _lib as L
from toothgroupnetwork_b200 import clouds, clustering

pytestmark = pytest.mark.gpu

try:
    from sklearn.cluster import DBSCAN as SkDBSCAN
except ImportError:
    SkDBSCAN = None

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SENTINEL = -0x21524111                 # never a label: shows an entry the kernel did not write
CORE_SENTINEL = 0xA5                   # neither 0 nor 1
INT_MAX = np.iinfo(np.int64).max


def reference(pts, eps: float, min_samples: int):
    """(n,3) float32 -> (labels int64, core bool) by the definition above, in float64 numpy.  Coincident points share their
    neighbourhood, so the pairs are evaluated once per distinct point, weighted by its multiplicity.  scipy's KD tree only
    proposes the candidate pairs, within eps (1 + 1e-6), a margin far wider than any rounding; numpy's predicate decides each
    one.  A point with a non-finite coordinate fails the predicate against every point, itself included: it is noise."""
    x = np.asarray(pts, np.float64)
    n = x.shape[0]
    labels, core = np.full(n, -1, np.int64), np.zeros(n, bool)
    fin = np.flatnonzero(np.isfinite(x).all(1))
    if fin.size == 0:
        return labels, core
    u, first, inv, mult = np.unique(x[fin], axis=0, return_index=True, return_inverse=True, return_counts=True)
    inv = inv.reshape(-1)
    smallest = fin[first]                                             # smallest index holding each distinct point
    m, r2 = u.shape[0], eps * eps
    cand = cKDTree(u).query_pairs(eps * (1 + 1e-6), output_type="ndarray")       # i < j
    d = u[cand[:, 0]] - u[cand[:, 1]]
    cand = cand[(d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2] <= r2]
    rows, cols = np.concatenate([cand[:, 0], cand[:, 1]]), np.concatenate([cand[:, 1], cand[:, 0]])
    counts = mult + np.bincount(rows, weights=mult[cols], minlength=m).astype(np.int64)   # the point's copies, then the others
    core_u = counts >= min_samples
    cc = core_u[rows] & core_u[cols]
    ncomp, comp = connected_components(coo_matrix((np.ones(int(cc.sum()), np.int8), (rows[cc], cols[cc])), shape=(m, m)),
                                       directed=False)
    cu = np.flatnonzero(core_u)
    key = np.full(ncomp, INT_MAX)
    np.minimum.at(key, comp[cu], smallest[cu])
    used = np.unique(comp[cu])
    rank = np.full(ncomp, -1, np.int64)
    rank[used[np.argsort(key[used])]] = np.arange(used.size)
    lab_u = np.full(m, -1, np.int64)
    lab_u[cu] = rank[comp[cu]]
    nb = ~core_u[rows] & core_u[cols]
    best = np.full(m, INT_MAX)
    np.minimum.at(best, rows[nb], lab_u[cols[nb]])
    border = ~core_u & (best < INT_MAX)
    lab_u[border] = best[border]
    labels[fin], core[fin] = lab_u[inv], core_u[inv]
    return labels, core


def launch(pts, eps: float, min_samples: int):
    """one tgn_dbscan on the current stream, into sentinel-filled outputs and a garbage-filled workspace -> (labels int32,
    core uint8, n_clusters) on the host"""
    x = torch.as_tensor(np.ascontiguousarray(pts, np.float32)).cuda()
    n = x.shape[0]
    labels = torch.full((n,), SENTINEL, dtype=torch.int32, device="cuda")
    core = torch.full((n,), CORE_SENTINEL, dtype=torch.uint8, device="cuda")
    nc = torch.full((1,), SENTINEL, dtype=torch.int32, device="cuda")
    ws = torch.full((int(L.load().tgn_dbscan_bytes(n)),), 0xA5, dtype=torch.uint8, device="cuda")
    L.call("tgn_dbscan", n, L.ptr(x), float(eps), int(min_samples), L.ptr(ws), L.ptr(labels), L.ptr(core), L.ptr(nc),
           L.stream_ptr())
    return labels.cpu().numpy(), core.cpu().numpy(), int(nc.cpu()[0])


def sklearn_agrees(pts, eps: float, min_samples: int, labels: np.ndarray, core: np.ndarray) -> None:
    if SkDBSCAN is None or len(pts) < 12 or not np.isfinite(pts).all():
        return
    ref = SkDBSCAN(eps=eps, min_samples=min_samples).fit(pts)
    assert np.array_equal(ref.core_sample_indices_, np.flatnonzero(core)), "reference core points differ from scikit-learn's"
    assert np.array_equal(ref.labels_, labels), "reference labels differ from scikit-learn's"


def check(pts, eps: float, min_samples: int, sklearn: bool = True):
    """one launch against the reference (and scikit-learn) -> the reference's (labels, core)"""
    pts = np.ascontiguousarray(pts, np.float32)
    want_l, want_c = reference(pts, eps, min_samples)
    got_l, got_c, nc = launch(pts, eps, min_samples)
    assert not (got_l == SENTINEL).any() and np.isin(got_c, (0, 1)).all(), "an output entry was not written"
    bad = np.flatnonzero(got_c != want_c)
    assert bad.size == 0, f"core flags differ at {bad.size} points, first {bad[:8].tolist()}"
    bad = np.flatnonzero(got_l != want_l)
    assert bad.size == 0, f"labels differ at {bad.size} points, first {bad[:8].tolist()}: {got_l[bad[:8]].tolist()} vs {want_l[bad[:8]].tolist()}"
    assert nc == int(want_l.max()) + 1
    if sklearn:
        sklearn_agrees(pts, eps, min_samples, want_l, want_c)
    return want_l, want_c


# ------------------------------------------------------------------------------------------------------- lattice shells at eps
def interior_count(k: int, strict: bool = False) -> int:
    """neighbours of an interior point of the 1/8 lattice at eps = k/8 (strict: just inside eps)"""
    return sum(1 for v in itertools.product(range(-k, k + 1), repeat=3) if (sum(t * t for t in v) < k * k if strict else sum(t * t for t in v) <= k * k))


@pytest.mark.parametrize("k", [1, 2, 3])
def test_lattice_shells_exactly_at_eps(k):
    """shuffled 1/8 lattice, |i| <= 12: every float64 distance and eps^2 are exact, so the shell at eps is in, and one ulp below
    eps it is out (tests/test_cpu_dbscan_edges.py checks the exactness)"""
    pts = clouds.lattice(12, seed=k).numpy()
    eps = k / 8.0
    full, inner = interior_count(k), interior_count(k, strict=True)
    for e in (eps, float(np.nextafter(eps, 0.0))):
        for ms in (2, full):
            labels, core = check(pts, e, ms)
            if ms == full:              # the interior (|i| <= 12 - k on every axis) reaches min_samples only with the shell
                assert int(core.sum()) == ((25 - 2 * k) ** 3 if e == eps else 0)
            elif k == 1:                # at eps = 1/8 the first shell is all there is: one cluster, or nothing at all
                assert (labels == 0).all() if e == eps else (labels == -1).all()
    assert (full, inner) == ((7, 1), (33, 27), (123, 93))[k - 1]


@pytest.mark.parametrize("min_samples", [32, 33, 34])
def test_min_samples_at_the_neighbour_count(min_samples):
    """eps = 1/4: an interior lattice point has exactly 33 neighbours (1 + 6 + 12 + 8 + 6), so pass 0 stops exactly at the
    threshold there, the faces and corners fall below it, and one step inside a face a point has 32"""
    pts = clouds.lattice(12, seed=7).numpy()
    labels, core = check(pts, 0.25, min_samples)
    depth = 12 - np.abs(pts * 8).round().max(1)                      # lattice steps to the nearest face
    one_face = (np.abs(pts * 8).round() == 11).sum(1) == 1          # one step inside exactly one face: only (2, 0, 0) is missing
    if min_samples == 33:
        assert np.array_equal(core, depth >= 2)
    elif min_samples == 34:
        assert not core.any() and (labels == -1).all()
    else:
        assert np.array_equal(core, (depth >= 2) | ((depth == 1) & one_face))


# ------------------------------------------------------------------------------------------------------------ border ties
def _cluster(at, u, contact, perp):
    """six points along direction u from `at`, the first at distance `contact`; all within 0.85 of each other"""
    u, p1, p2 = np.asarray(u, float), np.asarray(perp[0], float), np.asarray(perp[1], float)
    steps = [(0.0, 0, 0), (0.25, 0.1, 0), (0.45, -0.1, 0), (0.6, 0, 0.1), (0.7, 0, -0.1), (0.8, 0, 0)]
    return [at + u * (contact + a) + p1 * b + p2 * c for a, b, c in steps]


def border_cloud(shuffle_seed=None):
    """eps = 1, min_samples = 5, six-point clusters.  Each star: a point P within eps of the first (contact) point of two or
    three clusters and of nothing else of theirs, so P has at most 4 neighbours and is a border point.  The cluster P must join
    (smallest label = smallest member index) is the one met last in the kernel's cell order (+z) and the farthest (contact at
    0.99), not the nearest (+x, 0.90) nor the first in cell order (-z, 0.95).  A second kind of star adds a point Q within eps
    of P only: Q's one neighbour is not core, so Q is noise.  Returns points, the index of each P, its clusters' first
    indices in (+z or +y, -z or -y, +x) order, and the Q indices."""
    X, Y, Z = np.eye(3)
    first, later, stars = [], [], []
    groups = {"far": [], "mid": [], "near": []}
    for s in range(6):
        at = np.array([10.0 * s + 0.37, 0.21, 0.13])
        if s % 2 == 0:       # three clusters
            spec = (("far", Z, 0.99, (X, Y)), ("mid", -Z, 0.95, (X, Y)), ("near", X, 0.90, (Y, Z)))
        else:                # two clusters on the y axis, and Q on -x
            spec = (("far", Y, 0.97, (X, Z)), ("mid", -Y, 0.90, (X, Z)))
        members = []
        for kind, u, contact, perp in spec:
            c = _cluster(at, u, contact, perp)
            groups[kind].append(c[::-1])                             # the contact point gets the largest index of its cluster
            members.append((kind, len(groups[kind]) - 1))
        first.append(at)
        if s % 2:
            later.append(at + np.array([-0.5, 0.0, 0.0]))
        stars.append(members)
    far_pair = [np.array([200.0, 0.0, 0.0]), np.array([200.5, 0.0, 0.0])]   # two non-core points with each other only
    pts = first + [p for kind in ("far", "mid", "near") for c in groups[kind] for p in c] + later + far_pair
    pts = np.array(pts, np.float32)
    base = {"far": len(first)}
    base["mid"] = base["far"] + 6 * len(groups["far"])
    base["near"] = base["mid"] + 6 * len(groups["mid"])
    q0 = base["near"] + 6 * len(groups["near"])
    star_clusters = [[base[kind] + 6 * j for kind, j in members] for members in stars]
    qs = list(range(q0, q0 + len(later))) + [q0 + len(later), q0 + len(later) + 1]
    p_idx = list(range(len(first)))
    if shuffle_seed is not None:
        perm = np.random.default_rng(shuffle_seed).permutation(len(pts))
        new_of = np.argsort(perm)
        pts = pts[perm]
        p_idx = [int(new_of[i]) for i in p_idx]
        star_clusters = [[int(new_of[i]) for i in c] for c in star_clusters]
        qs = [int(new_of[i]) for i in qs]
    return pts, p_idx, star_clusters, qs


@pytest.mark.parametrize("shuffle_seed", [None, 3, 4])
def test_border_points_take_the_smallest_label(shuffle_seed):
    pts, p_idx, star_clusters, qs = border_cloud(shuffle_seed)
    labels, core = check(pts, 1.0, 5)
    for p, clusters in zip(p_idx, star_clusters):
        assert not core[p] and all(core[c] for c in clusters)
        their = [int(labels[c]) for c in clusters]
        assert len(set(their)) == len(their) and labels[p] == min(their)
        if shuffle_seed is None:        # the label P takes is neither the nearest cluster's nor the first met in cell order
            assert labels[p] == their[0] and labels[p] < min(their[1:])
    assert (labels[qs] == -1).all() and not core[qs].any()


# ------------------------------------------------------------------------------------------------------- deep union-find
def helix(n: int, step: float, cuts=(), gap: float = 0.0, seed: int = 0) -> np.ndarray:
    """n points along a helix of radius 1 and pitch 0.05 at arc-length spacing `step` (`gap` after the points in `cuts`), shuffled"""
    t = np.full(n - 1, step)
    t[list(cuts)] = gap
    s = np.concatenate([[0.0], np.cumsum(t)])
    c = 0.05 / (2 * np.pi)
    theta = s / np.sqrt(1.0 + c * c)
    pts = np.stack([np.cos(theta), np.sin(theta), c * theta], 1).astype(np.float32)
    return pts[np.random.default_rng(seed).permutation(n)]


@pytest.mark.parametrize("min_samples", [2, 3])
def test_deep_union_find_on_a_chain(min_samples):
    """20 000 points at 0.9 eps along a helix, shuffled: one component whose every union crosses the index order.  Cut at 7
    places with 1.1 eps gaps, the 8 pieces are numbered by their smallest index.  The same input three times, once on a
    second stream, gives the same outputs."""
    eps = 0.01
    pts = helix(20000, 0.9 * eps, seed=min_samples)
    labels, core = check(pts, eps, min_samples)
    assert (labels == 0).all() and int(core.sum()) == (20000 if min_samples == 2 else 19998)
    cuts = np.random.default_rng(10 + min_samples).choice(np.arange(100, 19900), 7, replace=False)
    pts = helix(20000, 0.9 * eps, cuts, 1.1 * eps, seed=20 + min_samples)
    labels, _ = check(pts, eps, min_samples)
    assert labels.max() == 7 and (labels >= 0).all()
    firsts = [int(np.flatnonzero(labels == k)[0]) for k in range(8)]
    assert firsts == sorted(firsts)
    runs = [launch(pts, eps, min_samples)]
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        runs.append(launch(pts, eps, min_samples))
    runs.append(launch(pts, eps, min_samples))
    for r in runs[1:]:
        assert np.array_equal(r[0], runs[0][0]) and np.array_equal(r[1], runs[0][1]) and r[2] == runs[0][2] == 8
    assert np.array_equal(runs[0][0], labels)


# ------------------------------------------------------------------------------------------------------------ many clusters
@pytest.mark.parametrize("min_samples", [2, 4, 5])
def test_three_thousand_clusters(min_samples):
    """3 000 four-point clusters on a 3-D grid of step 1, eps = 0.1, shuffled: the roots spread over every 1 024-point block of
    the numbering scan, whose carry must count 3 000 clusters; min_samples = 4 is exactly the count, 5 leaves only noise"""
    rng = np.random.default_rng(30)
    nodes = np.stack(np.meshgrid(np.arange(15), np.arange(15), np.arange(14), indexing="ij"), -1).reshape(-1, 3)
    nodes = nodes[rng.choice(len(nodes), 3000, replace=False)].astype(np.float64) + 0.3
    tetra = np.array([[1, 1, 1], [1, -1, -1], [-1, 1, -1], [-1, -1, 1]]) * 0.02
    pts = (nodes[:, None, :] + tetra[None]).reshape(-1, 3)
    pts = pts[rng.permutation(len(pts))].astype(np.float32)
    labels, core = check(pts, 0.1, min_samples)
    if min_samples == 5:
        assert (labels == -1).all()
    else:
        assert labels.max() == 2999 and core.all()
        assert np.array_equal(np.bincount(labels), np.full(3000, 4))


# ------------------------------------------------------------------------------------------------------------ grid geometry
def blobs(n: int, seed: int, box: float = 1.0, sigma: float = 0.02) -> np.ndarray:
    """half the points in n // 60 + 1 Gaussian blobs of deviation sigma, half uniform in the box: cores, borders and noise"""
    rng = np.random.default_rng(seed)
    centres = rng.uniform(0, box, (n // 60 + 1, 3))
    pts = np.concatenate([centres[rng.integers(0, len(centres), n // 2)] + rng.normal(0, sigma, (n // 2, 3)),
                          rng.uniform(0, box, (n - n // 2, 3))])
    return pts[rng.permutation(n)].astype(np.float32)


def kernel_cells(pts: np.ndarray, eps: float):
    """the kernel's grid (db_setup_kernel): per axis (cells, cell of the largest coordinate before the clamp)"""
    out = []
    for a in range(3):
        lo, hi = float(pts[:, a].min()), float(pts[:, a].max())
        h = max(eps * (1.0 + 1e-9), (hi - lo) / 63) or 1.0
        out.append((min(64, int((hi - lo) / h) + 1), int((hi - lo) / h)))
    return out


def geometry_case(name: str):
    rng = np.random.default_rng(40)
    if name == "wide_x":            # x extent 100 eps: cells wider than eps on x only, 64 of them
        pts = (rng.uniform(0, 1, (20000, 3)) * [1.0, 0.04, 0.04]).astype(np.float32)
        return pts, 0.01, 30
    if name == "planar":            # zero extent on z
        pts = np.concatenate([rng.uniform(0, 1, (20000, 2)), np.zeros((20000, 1))], 1).astype(np.float32)
        return pts, 0.01, 6
    if name == "one_cell":          # eps wider than the extent: one cell, but not every pair within eps
        return rng.uniform(0, 1, (1500, 3)).astype(np.float32), 1.2, 1450
    if name == "offset":            # far from the origin: coordinates round to 2^-14 around 1000
        return blobs(24000, 41) + np.float32(1000.0), 0.02, 10
    if name == "scaled":
        return blobs(24000, 41) * np.float32(1e-3), 0.02e-3, 10
    if name in ("last_cell_face", "last_cell_edge"):
        # x from 0 to 8 (resp. 8.125) at eps = 1/8: cells of extent / 63; the largest x lands exactly on the lower face of cell
        # 63 of 64 (resp. one rounding below the upper edge of cell 62 of 63), with points around it
        top = 8.0 if name == "last_cell_face" else 8.125
        pts = rng.uniform(0, 1, (6000, 3)) * [top, 1.0, 1.0]
        pts[:300, 0] = top - rng.uniform(0, 0.2, 300)
        pts[0, 0], pts[1, 0], pts[2:6, 0] = 0.0, top, top
        return pts.astype(np.float32), 0.125, 5
    raise KeyError(name)


@pytest.mark.parametrize("name", ["wide_x", "planar", "one_cell", "offset", "scaled", "last_cell_face", "last_cell_edge"])
def test_grid_geometry(name):
    pts, eps, ms = geometry_case(name)
    cells = kernel_cells(pts, eps)
    if name == "wide_x":
        assert cells[0][0] == 64 and (pts[:, 0].max() - pts[:, 0].min()) > 63 * eps and cells[1][0] < 64 and cells[2][0] < 64
    if name == "planar":
        assert cells[2][0] == 1
    if name == "one_cell":
        assert all(c[0] == 1 for c in cells)
    if name == "last_cell_face":
        assert cells[0] == (64, 63)
    if name == "last_cell_edge":
        assert cells[0] == (63, 62)
    labels, core = check(pts, eps, ms)
    assert core.any() and not core.all()


# ------------------------------------------------------------------------------------------------------------ duplicates
@pytest.mark.parametrize("min_samples", [3, 5])
def test_coincident_copies_at_min_samples(min_samples):
    """exactly min_samples copies at one location (core), min_samples - 1 at another (noise), and both inside a sparse cloud"""
    rng = np.random.default_rng(50)
    bg = rng.uniform(0, 1, (600, 3))
    a, b, c, d = np.array([2.0, 2.0, 2.0]), np.array([3.0, 3.0, 3.0]), bg[10], bg[20]
    pts = np.concatenate([bg, np.repeat([a], min_samples, 0), np.repeat([b], min_samples - 1, 0),
                          np.repeat([c], min_samples - 1, 0), np.repeat([d], min_samples - 2, 0)])
    perm = rng.permutation(len(pts))
    pts = pts[perm].astype(np.float32)
    labels, core = check(pts, 0.05, min_samples)
    at_a = np.flatnonzero((pts == a.astype(np.float32)).all(1))
    at_b = np.flatnonzero((pts == b.astype(np.float32)).all(1))
    assert core[at_a].all() and len(set(labels[at_a].tolist())) == 1 and labels[at_a][0] >= 0
    assert not core[at_b].any() and (labels[at_b] == -1).all()


@pytest.mark.parametrize("min_samples", [4000, 5000, 5001])
def test_five_thousand_copies(min_samples):
    """5 000 copies of one point, and isolated points 1.4 eps away in all 26 surrounding cells: the ballot count of pass 0 runs
    over 157 warp-wide chunks after the cells before it in scan order, and stops early at 4 000, exactly at the last copy at
    5 000, and not at all at 5 001"""
    eps = 0.1
    ring = np.array([v for v in itertools.product((-1, 0, 1), repeat=3) if any(v)], np.float64) * 0.14
    pts = np.concatenate([np.zeros((5000, 3)), np.repeat(ring, 3, 0)])
    pts = pts[np.random.default_rng(51).permutation(len(pts))].astype(np.float32)
    assert kernel_cells(pts, eps) == [(3, 2)] * 3
    labels, core = check(pts, eps, min_samples, sklearn=min_samples == 5000)
    copies = (pts == 0).all(1)
    assert core[copies].all() == (min_samples <= 5000) and not core[~copies].any()
    assert (labels[copies] == (0 if min_samples <= 5000 else -1)).all() and (labels[~copies] == -1).all()


# ------------------------------------------------------------------------------------------------------------ sizes
SIZES = [1, 2, 11, 12, 31, 32, 33, 255, 256, 257, 1023, 1024, 1025, 24000]


@pytest.mark.parametrize("n", SIZES)
def test_sizes(n):
    """around the warp (32), block (256 threads, 8 warps) and numbering-scan (1 024) widths; min_samples above n leaves only
    noise and min_samples = 1 makes every point core (the components of the eps-graph).  The kernel applies the direct
    predicate below 12 points too."""
    pts = blobs(n, 60 + n, box=0.1 * max(n, 8) ** (1 / 3), sigma=0.05)
    for ms in (4, n + 1, 1):
        labels, core = check(pts, 0.1, ms)
        if ms == n + 1:
            assert (labels == -1).all() and not core.any()
        if ms == 1:
            assert core.all()


def test_cached_workspace_across_sizes():
    """clustering.dbscan_device's per-stream workspace: 24 000 points, then 100 in the same buffer, then 24 000 again"""
    clustering._ws.clear()
    bufs = []
    for n, seed in ((24000, 70), (100, 71), (24000, 72)):
        pts = blobs(n, seed, box=0.1 * n ** (1 / 3), sigma=0.05)
        want_l, want_c = reference(pts, 0.1, 5)
        labels, core = clustering.dbscan_device(torch.from_numpy(pts).cuda(), 0.1, 5)
        assert np.array_equal(labels.cpu().numpy(), want_l) and np.array_equal(core.cpu().numpy(), want_c)
        bufs.append(next(iter(clustering._ws.values())).data_ptr())
    assert len(set(bufs)) == 1


def test_non_finite_points_are_noise():
    """the kernel and dbscan_device take non-finite coordinates (the public functions refuse them): such a point is within eps
    of nothing, itself included, and the rest cluster as if it were absent"""
    pts = blobs(3000, 80, box=1.4, sigma=0.05)
    bad = np.random.default_rng(81).choice(3000, 40, replace=False)
    for k, i in enumerate(bad):
        pts[i, k % 3] = (np.nan, np.inf, -np.inf)[k % 3]
    labels, core = check(pts, 0.1, 5)
    assert (labels[bad] == -1).all() and not core[bad].any()
    keep = np.setdiff1d(np.arange(3000), bad)
    l_keep, c_keep = reference(pts[keep], 0.1, 5)
    assert np.array_equal(labels[keep], l_keep) and np.array_equal(core[keep], c_keep)
    d_l, d_c = clustering.dbscan_device(torch.from_numpy(pts).cuda(), 0.1, 5)
    assert np.array_equal(d_l.cpu().numpy(), labels) and np.array_equal(d_c.cpu().numpy(), core)
    with pytest.raises(ValueError, match="^Input X contains NaN"):
        clustering.dbscan(pts, 0.1, 5)


def test_refusals_leave_the_outputs_untouched():
    x = torch.from_numpy(blobs(64, 90)).cuda()
    labels = torch.full((64,), SENTINEL, dtype=torch.int32, device="cuda")
    core = torch.full((64,), CORE_SENTINEL, dtype=torch.uint8, device="cuda")
    nc = torch.full((1,), SENTINEL, dtype=torch.int32, device="cuda")
    ws = torch.empty(int(L.load().tgn_dbscan_bytes(64)), dtype=torch.uint8, device="cuda")
    ok = (64, L.ptr(x), 0.1, 5, L.ptr(ws), L.ptr(labels), L.ptr(core), L.ptr(nc), L.stream_ptr())

    def untouched():
        torch.cuda.synchronize()
        return (labels == SENTINEL).all() and (core == CORE_SENTINEL).all() and int(nc[0]) == SENTINEL

    for pos, value in ((2, 0.0), (2, -0.1), (2, float("nan")), (3, 0), (3, -1), (0, -1), (5, None), (6, None), (1, None), (4, None)):
        args = list(ok)
        args[pos] = value
        with pytest.raises(L.TgnError, match="dbscan"):
            L.call("tgn_dbscan", *args)
        assert untouched(), f"argument {pos} = {value!r}"
    L.call("tgn_dbscan", 0, *ok[1:])                                 # n = 0: nothing to do, nothing written
    assert untouched()
    L.call("tgn_dbscan", 0, None, 0.1, 5, None, None, None, None, L.stream_ptr())
    L.call("tgn_dbscan", *ok[:7], None, L.stream_ptr())               # the cluster count is optional
    want_l, want_c = reference(x.cpu().numpy(), 0.1, 5)
    assert np.array_equal(labels.cpu().numpy(), want_l) and np.array_equal(core.cpu().numpy(), want_c)
    assert int(nc[0]) == SENTINEL


# ------------------------------------------------------------------------------------------------------------ public functions
def test_public_functions_equal_the_sklearn_edges_fixture():
    """tests/golden/ref_sklearn_dbscan_edges.npz: eps within one ulp of a pair's distance.  Below 12 points dbscan and DBSCAN are
    scikit-learn's brute-force answer (host_fits counts them), while the kernel keeps the direct predicate; from 12 points the
    kernel is scikit-learn's answer"""
    fix = np.load(os.path.join(ROOT, "tests", "golden", "ref_sklearn_dbscan_edges.npz"))
    off = fix["offsets"]
    kernel_differs = 0
    for k, name in enumerate(fix["names"].tolist()):
        pts, eps, ms = fix["points"][off[k]:off[k + 1]], float(fix["eps"][k]), int(fix["min_samples"][k])
        want_l, want_core = fix["labels"][off[k]:off[k + 1]], np.flatnonzero(fix["core"][off[k]:off[k + 1]])
        before = clustering.DBSCAN.host_fits
        got = clustering.DBSCAN(eps=eps, min_samples=ms).fit(pts)
        assert clustering.DBSCAN.host_fits - before == (1 if len(pts) < 12 else 0), name
        assert np.array_equal(got.labels_, want_l) and np.array_equal(got.core_sample_indices_, want_core), name
        labels, core = check(pts, eps, ms, sklearn=False)
        if len(pts) >= 12:
            assert np.array_equal(labels, want_l) and np.array_equal(np.flatnonzero(core), want_core), name
        else:
            kernel_differs += not np.array_equal(labels, want_l)
    assert kernel_differs > 0


def test_clustering_labels_below_twelve_points():
    """get_clustering_labels runs the kernel at every size: with min_samples = 30 no point of a cloud under 12 points is core
    under either distance form, so it finds no cluster, and like the reference function it then raises IndexError"""
    fix = np.load(os.path.join(ROOT, "tests", "golden", "ref_sklearn_dbscan_edges.npz"))
    off = fix["offsets"]
    for k in range(len(fix["names"])):
        pts = fix["points"][off[k]:off[k + 1]] * np.float32(0.01)    # within 0.03 of each other
        if len(pts) >= 12:
            continue
        labels, core = clustering.dbscan_device(torch.from_numpy(pts).cuda(), 0.03, 30)
        assert (labels.cpu().numpy() == -1).all() and not core.cpu().numpy().any()
        if SkDBSCAN is not None:
            assert (SkDBSCAN(eps=0.03, min_samples=30).fit(pts).labels_ == -1).all()
        with pytest.raises(IndexError):
            clustering.get_clustering_labels(pts, np.ones(len(pts), np.int64))
