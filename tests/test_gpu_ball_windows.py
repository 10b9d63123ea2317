"""Ball query through the index-windowed grid: every case through the grid kernel, the tile scan and the automatic choice,
bitwise against the CPU oracle, int64 and int32 outputs.  The cases aim at the windows: clouds that are not a multiple of
the window size or smaller than one window, balls whose members are spread over several windows (full in a later one, or
never full), K from 1 to 128, duplicated vertices, clouds far from the origin, and clouds whose window grows to keep the
(window, cell) table within bounds."""
import numpy as np
import pytest
import torch

from oracle import oracle
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
