"""Ball query through the index-windowed grid: every case through the grid kernel, the tile scan and the automatic choice,
bitwise against the CPU oracle, int64 and int32 outputs.  The cases aim at the windows: clouds that are not a multiple of
the window size or smaller than one window, balls whose members are spread over several windows (full in a later one, or
never full), K from 1 to 128, duplicated vertices, clouds far from the origin, and clouds whose window grows to keep the
(window, cell) table within bounds."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import oracle
from toothgroupnetwork_b200 import _lib as L
from toothgroupnetwork_b200 import clouds
from toothgroupnetwork_b200 import pointnet2_utils as pn2

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _reference_on_cpu():
    """The oracle restates the reference on CPU tensors (index-order |p|^2 rounding)."""
    pn2.set_reference_device("cpu")
    yield
    pn2.set_reference_device("cuda")


def check_all_paths(xyz, new, r, K):
    want = oracle.query_ball_point(r, K, xyz.numpy(), new.numpy())
    x, q = xyz.cuda(), new.cuda()
    for path in (pn2.BALL_GRID, pn2.BALL_TILE, pn2.BALL_AUTO):
        got64 = pn2._ball_query(r, K, x, q, True, path)
        got32 = pn2._ball_query(r, K, x, q, False, path)
        assert np.array_equal(got64.cpu().numpy(), want), f"path {path}, int64"
        assert np.array_equal(got32.cpu().numpy().astype(np.int64), want), f"path {path}, int32"
    return want


def arch_batch(N, S, r, offset=0.0, scale=1.0, seeds=(4, 5), dup=False):
    xs = [clouds.dental_arch(N // 2 if dup else N, s)[0] for s in seeds]
    if dup:
        xs = [clouds.with_duplicates(x, s) for x, s in zip(xs, seeds)]
    xs = [x * scale + offset for x in xs]
    n = xs[0].shape[0]
    g = torch.Generator().manual_seed(n + S)
    news = []
    for x in xs:
        q = x[torch.randperm(n, generator=g)[:S]].clone()
        q[: S // 8] += (torch.rand(S // 8, 3, generator=g) - 0.5) * 4 * r * scale    # queries off the surface
        q[0] = x.max(0).values + 3 * r * scale + 1.0                                 # outside the bounding box: empty ball
        news.append(q)
    return torch.stack(xs).contiguous(), torch.stack(news).contiguous()


CASES = [
    # (N, S, r, K, offset, scale, duplicated vertices)
    (24000, 1024, 0.1, 32, 0.0, 1.0, False),     # bench shape
    (24000, 512, 0.4, 32, 0.0, 1.0, False),      # dense balls
    (24000, 512, 0.01, 16, 0.0, 1.0, False),     # mostly empty balls
    (9000, 300, 0.1, 64, 40.0, 1.0, False),      # far from the origin: the expanded form is noisy
    (9000, 300, 2.0, 32, 0.0, 25.0, False),      # millimetre-like coordinates
    (1000, 64, 0.15, 8, 0.0, 1.0, False),        # smaller than one window
    (70000, 256, 0.05, 32, 0.0, 1.0, False),     # the window grows to the largest size to keep the table in bounds
    (5000, 100, 5.0, 32, 0.0, 1.0, False),       # radius larger than the cloud: one cell
    (3001, 200, 0.15, 32, 0.0, 1.0, False),      # not a multiple of any window size
    (700, 64, 0.2, 16, 0.0, 1.0, False),         # N < the smallest window
    (24000, 512, 0.075, 32, 0.0, 1.0, False),    # cells that need a 4096-point window
    (24000, 256, 0.1, 1, 0.0, 1.0, False),       # K = 1
    (24000, 256, 0.1, 64, 0.0, 1.0, False),      # K = 64
    (24000, 256, 0.1, 128, 0.0, 1.0, False),     # K = 128: most queries need several windows
    (24000, 512, 0.1, 32, 0.0, 1.0, True),       # every vertex twice
    (16000, 256, 0.05, 32, 1000.0, 1.0, False),  # far from the origin, sparse balls
]


@pytest.mark.parametrize("N,S,r,K,offset,scale,dup", CASES)
def test_windowed_grid_matches_oracle(N, S, r, K, offset, scale, dup):
    xyz, new = arch_batch(N, S, r, offset, scale, dup=dup)
    check_all_paths(xyz, new, r, K)


def ball_float64(xyz, new, r, K):
    """query_ball_point in float64, exact on the 1/8 lattice (tests/test_cpu_lattice_exact.py): the first K indices with
    d2 <= r^2, padded with the first, N for an empty ball; and how many (query, point) pairs lie exactly on a sphere."""
    x, q = xyz.double().numpy(), new.double().numpy()
    B, N, _ = x.shape
    out = np.full((B, q.shape[1], K), N, np.int64)
    on_sphere = 0
    for b in range(B):
        for c in range(0, q.shape[1], 128):
            d = q[b, c:c + 128, None, :] - x[b][None, :, :]
            d2 = (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]
            on_sphere += int((d2 == r * r).sum())
            for s, inside in enumerate(d2 <= r * r):
                m = np.nonzero(inside)[0][:K]
                if len(m):
                    out[b, c + s, :] = m[0]
                    out[b, c + s, :len(m)] = m
    return out, on_sphere


def lattice_batch(half, N, S, seed, B=2):
    """B shuffled 1/8 lattices (N points of the box |i| <= half each) and S queries per cloud: a quarter on points of the
    cloud, a quarter on lattice sites the cloud may lack, a quarter in the middle of cells, the rest half-way along a cell edge."""
    g = torch.Generator().manual_seed(seed)
    xs = [clouds.lattice(half, seed + b, N) for b in range(B)]
    news = []
    for x in xs:
        q = S // 4
        on = x[torch.randperm(N, generator=g)[:q]]
        site = torch.randint(-half, half + 1, (q, 3), generator=g).float() / 8.0
        mid = (2 * torch.randint(-half, half, (q, 3), generator=g) + 1).float() / 16.0
        edge = torch.randint(-half, half, (S - 3 * q, 3), generator=g).float() / 8.0
        edge[:, 0] += 1.0 / 16.0
        news.append(torch.cat([on, site, mid, edge]))
    return torch.stack(xs).contiguous(), torch.stack(news).contiguous()


LATTICE_CASES = [
    # (half-width of the lattice box, points per cloud, queries, r, K): r = 0.25 puts 6 lattice points of a full shell at
    # exactly r (d2 = float32(r^2) = 1/16) and 33 in a ball around a lattice point, 32 around a cell centre
    (10, 9261, 512, 0.25, 32),           # every point of the box: full balls, K one below the 33 members
    (10, 9261, 512, 0.25, 33),           # K = the members of an interior ball
    (10, 9261, 512, 0.25, 34),           # K one above: padded with the first
    (10, 9261, 256, 0.25, 1),
    (10, 9261, 256, 0.375, 128),         # 123 / 136 members at r = 3/8 (shell i^2 + j^2 + l^2 = 9 at exactly r)
    (40, 24000, 1024, 0.25, 8),          # 4.5 % of a larger box: sparse balls, the grid's case
    (40, 24000, 1024, 0.5, 16),          # ~12 members: 4.5 % of the 257 sites within r = 0.5
    (6, 2197, 300, 0.25, 32),            # below the grid's automatic size: the tile kernel, and the grid when forced
]


@pytest.mark.parametrize("half,N,S,r,K", LATTICE_CASES)
def test_lattice_balls_match_oracle_and_float64(half, N, S, r, K):
    xyz, new = lattice_batch(half, N, S, seed=half + N + K)
    want = check_all_paths(xyz, new, r, K)
    exact, on_sphere = ball_float64(xyz, new, r, K)
    assert np.array_equal(want, exact)
    assert on_sphere > 0, "no point exactly on a sphere"


SENTINEL = -0x21524111                 # never an index: shows a row that neither kernel wrote


@pytest.mark.parametrize("wide", [False, True])
def test_one_launch_mixing_grid_and_tile_clouds(wide):
    """Three clouds of one launch: two sparse ones the automatic choice sends to the grid kernel, and a copy of the arch
    shrunk until r covers it whole, left to the tile kernel (every point a member).  The per-cloud flag decides which kernel
    writes which rows, so into a sentinel-filled output every row must be written once, by either.  wide: enough queries
    that the tile kernel runs at 16 warps per CTA."""
    N, r, K = 24000, 0.1, 32
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    S = 16 * -(-2 * sms // 3) if wide else 256
    assert (3 * -(-S // 16) >= 2 * sms) == wide
    arch = clouds.dental_arch(N, 21)[0]
    dense = (arch - arch.mean(0)) * 0.02                               # extent ~0.03 < r
    sparse = clouds.lattice(40, 22, N)
    assert float((dense.max(0).values - dense.min(0).values).norm()) < r
    xyz = torch.stack([arch, dense, sparse]).contiguous()
    g = torch.Generator().manual_seed(23)
    new = torch.stack([c[torch.randperm(N, generator=g)[:S]] for c in xyz]).contiguous()
    new[2, : S // 2] += 1.0 / 16.0                                     # off-lattice queries: empty balls
    want = oracle.query_ball_point(r, K, xyz.numpy(), new.numpy())
    assert (want[1] == np.arange(K)).all()                            # the dense cloud: every ball holds the first K points
    x, q = xyz.cuda(), new.cuda()
    for idx64, dtype in ((1, torch.int64), (0, torch.int32)):
        for path in (pn2.BALL_AUTO, pn2.BALL_GRID, pn2.BALL_TILE):
            out = torch.full((3, S, K), SENTINEL, dtype=dtype, device="cuda")
            L.call("tgn_ball_query", 3, N, S, ctypes.c_float(pn2._radius_sq_f32(r)), K, L.ptr(x), L.ptr(q), L.ptr(out),
                   idx64 | path, L.stream_ptr())
            got = out.cpu().numpy().astype(np.int64)
            assert np.array_equal(got, want), f"path {path}, idx64 {idx64}: rows differ in clouds " \
                                              f"{sorted(set(np.nonzero((got != want).any(-1))[0].tolist()))}"


def planted_cloud(N, member_idx, seed):
    """Points spread over a 10-unit cube (balls of r = 0.05 around the origin are empty), except at `member_idx`, which lie
    within 0.03 of the origin: the query at the origin has exactly those members."""
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(N, 3, generator=g) * 10.0 + 1.0
    x[member_idx] = (torch.rand(len(member_idx), 3, generator=g) - 0.5) * 0.03
    return x


def test_ball_full_in_a_later_window():
    N, K, r = 12000, 32, 0.05
    idx = list(range(3, 300, 37)) + list(range(6000, 6000 + 35 * 113, 113))     # 9 early members, the 32nd near index 8600
    x = torch.stack([planted_cloud(N, idx, 1), planted_cloud(N, idx[::-1], 2)])
    q = torch.zeros(2, 4, 3)
    q[:, 1] = torch.tensor([0.01, -0.01, 0.005])
    q[:, 2:] = x[:, [5, 11000]]
    want = check_all_paths(x.contiguous(), q.contiguous(), r, K)
    assert want[0, 0, K - 1] > 8000 and want[0, 0, 0] == 3


def test_ball_never_full_over_several_windows():
    N, K, r = 12000, 32, 0.05
    idx = [7, 1500, 2100, 4500, 4501, 9000, 11999]          # 7 members in five windows of any size up to 2048
    x = torch.stack([planted_cloud(N, idx, 3)])
    q = torch.zeros(1, 2, 3)
    q[0, 1] = torch.tensor([0.005, 0.0, -0.005])
    want = check_all_paths(x.contiguous(), q.contiguous(), r, K)
    assert list(want[0, 0, :7]) == idx and (want[0, 0, 7:] == idx[0]).all()
