"""The crop selection (csrc/crop_knn.cu) one launch at a time, against a float64 brute force in the kernel's operation order
((dx dx + dy dy) + dz dz), ordered by (distance, index): indices bit for bit.  The inputs are tie-heavy: shuffled 1/8 lattices
(every shell of equal distance is a tie, and a centre in the middle of a cell has eight nearest points) and meshes whose
vertices coincide thousands of times.  The cases sit at the edges of the kernel: k around each padded sort size, ties split by
the k-th rank, more threshold-equal points than the padded size, k >= N and clouds smaller than one sweep of the CTA, several
clouds and centres per launch, the int32 output, centres on a point or far away, clouds far from the origin, repeated launches
and the refusals."""
import numpy as np
import pytest
import torch

from toothgroupnetwork_b200 import _lib as L
from toothgroupnetwork_b200 import clouds

pytestmark = pytest.mark.gpu

SENTINEL = -0x21524111                 # never an index: shows an entry the kernel did not write


def brute(xyz: torch.Tensor, cents: torch.Tensor, k: int):
    """(N,3), (Q,3) -> indices (Q,k) int64 (zeros past N, as the kernel pads) and the sorted float64 distances (Q,N)."""
    x, c = xyz.double().numpy(), cents.double().numpy()
    d = x[None, :, :] - c[:, None, :]
    d2 = (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]
    order = np.lexsort((np.broadcast_to(np.arange(x.shape[0]), d2.shape), d2), axis=-1)
    out = np.zeros((c.shape[0], k), np.int64)
    out[:, :min(k, x.shape[0])] = order[:, :k]
    return out, np.take_along_axis(d2, order, -1)


def launch(xyz: torch.Tensor, cents: torch.Tensor, k: int, idx64: int = 1, out: torch.Tensor = None) -> torch.Tensor:
    """xyz (B,N,3), cents (B,Q,3) -> (B,Q,k) through tgn_crop_knn into a sentinel-filled buffer, on the CPU."""
    x, c = xyz.contiguous().cuda(), cents.contiguous().cuda()
    B, N, _ = x.shape
    Q = c.shape[1]
    if out is None:
        out = torch.full((B, Q, k), SENTINEL, dtype=torch.int64 if idx64 else torch.int32, device="cuda")
    L.call("tgn_crop_knn", B, N, Q, int(k), L.ptr(x), L.ptr(c), L.ptr(out), int(idx64), L.stream_ptr())
    return out.cpu()


def check(xyz: torch.Tensor, cents: torch.Tensor, k: int, idx64: int = 1) -> torch.Tensor:
    got = launch(xyz, cents, k, idx64)
    for b in range(xyz.shape[0]):
        want, _ = brute(xyz[b], cents[b], k)
        bad = np.nonzero((got[b].numpy() != want).any(1))[0]
        assert len(bad) == 0, f"cloud {b}, k={k}: rows {bad.tolist()} differ, first at column " \
                              f"{int(np.argmax(got[b, bad[0]].numpy() != want[bad[0]]))}"
    return got


def lattice_centres(half: int, n_on: int, n_mid: int, seed: int) -> torch.Tensor:
    """n_on centres on lattice points and n_mid in the middle of lattice cells, all inside the box |i| <= half."""
    g = torch.Generator().manual_seed(seed)
    on = torch.randint(-half, half + 1, (n_on, 3), generator=g).float() / 8.0
    mid = (2 * torch.randint(-half, half, (n_mid, 3), generator=g) + 1).float() / 16.0
    return torch.cat([on, mid]).contiguous()


def lattice_cloud(seed: int) -> torch.Tensor:
    return clouds.lattice(14, seed)                       # 29^3 = 24 389 points, not a multiple of the 1024-thread sweep


def kpad(k: int) -> int:
    return max(2, 1 << (k - 1).bit_length())


@pytest.mark.parametrize("k", [1, 2, 3, 1023, 1024, 1025, 2047, 3072, 4095, 4096])
def test_k_around_every_padded_size_with_split_ties(k):
    xyz = lattice_cloud(k)
    cents = lattice_centres(12, 8, 8, seed=k)
    check(xyz[None], cents[None], k)
    _, d2 = brute(xyz, cents, k)
    split = d2[:, k - 1] == d2[:, k]
    assert split.any(), "no row has a tie split by the k-th rank"


@pytest.mark.parametrize("k", [1, 2, 3])
@pytest.mark.parametrize("half", [14, 4])
def test_more_ties_than_the_padded_size_at_cell_centres(k, half):
    """Eight corners tie at a cell centre: for k = 1, 2 (padded 2) and 3 (padded 4) more points equal the threshold than the
    padded size; the answer is still the k lowest indices among them.  half = 4: 729 points, fewer than one sweep."""
    xyz = clouds.lattice(half, 40 + k)
    cents = lattice_centres(half, 0, 64, seed=k + half)
    _, d2 = brute(xyz, cents, k)
    assert ((d2 == d2[:, k - 1:k]).sum(1) == 8).all()
    check(xyz[None], cents[None], k)


def coincident_mesh(n: int = 24000, copies: int = 20000, seed: int = 0):
    """n - copies points of an arch and `copies` copies of one vertex, interleaved at random through the index order (the
    lowest-index copies lie in several 1024-index sweeps); returns the cloud and centres at the copied vertex, beside it (so
    that the copies tie at a distance other than zero behind closer arch points) and far from it."""
    g = torch.Generator().manual_seed(seed)
    arch = clouds.dental_arch(n - copies + 1, seed)[0]
    p, arch = arch[0].clone(), arch[1:]
    where = torch.randperm(n, generator=g)[:copies]
    xyz = torch.empty(n, 3)
    is_copy = torch.zeros(n, dtype=torch.bool)
    is_copy[where] = True
    xyz[is_copy] = p
    xyz[~is_copy] = arch
    cents = torch.stack([p, p + torch.tensor([0.01, 0.0, 0.0]), p + torch.tensor([0.0, -0.003, 0.002]), p + 0.5])
    return xyz.contiguous(), cents.contiguous(), is_copy


@pytest.mark.parametrize("seed", [0, 1])
def test_more_ties_than_the_padded_size_on_coincident_vertices(seed):
    xyz, cents, is_copy = coincident_mesh(seed=seed)
    k = 3072
    want, d2 = brute(xyz, cents, k)
    eq = (d2 == d2[:, k - 1:k]).sum(1)
    assert (eq[:3] >= 20000).all() and (eq[:3] > kpad(k)).all()
    first_copies = np.nonzero(is_copy.numpy())[0][:k]
    assert first_copies[-1] >= 3 * 1024                     # the copies taken span several sweeps
    assert np.array_equal(np.sort(want[0]), first_copies)
    check(xyz[None], cents[None], k)


@pytest.mark.parametrize("n,k", [(700, 700), (700, 701), (700, 1024), (700, 4096), (1000, 1), (1024, 1024), (1025, 1025),
                                 (1025, 2048)])
def test_k_at_and_above_n_and_clouds_smaller_than_a_sweep(n, k):
    xyz = clouds.lattice(5, n, n)
    cents = lattice_centres(5, 4, 4, seed=n + k)
    got = check(xyz[None], cents[None], k)
    if k > n:
        assert (got[0, :, n:] == 0).all()


@pytest.mark.parametrize("Q", [1, 16])
@pytest.mark.parametrize("k", [1, 100, 3072])
def test_batched_clouds_equal_single_launches(Q, k):
    xs = [clouds.lattice(14, 60 + b, 20000) + 0.125 * b for b in range(2)] + [clouds.dental_arch(20000, 62)[0]]
    cs = [lattice_centres(10, Q // 2, Q - Q // 2, seed=70 + b) + 0.125 * b for b in range(2)]
    cs.append(clouds.dental_arch(20000, 62)[0][:Q] * 1.01)
    xyz, cents = torch.stack(xs), torch.stack(cs)
    full = check(xyz, cents, k)
    for b in range(3):
        assert torch.equal(full[b:b + 1], launch(xyz[b:b + 1], cents[b:b + 1], k)), f"cloud {b}"


@pytest.mark.parametrize("k", [1, 3, 1025, 4096])
def test_int32_output_equals_int64(k):
    xyz = torch.stack([lattice_cloud(80), clouds.lattice(14, 81)])
    cents = torch.stack([lattice_centres(12, 3, 5, seed=82), lattice_centres(12, 5, 3, seed=83)])
    got32 = check(xyz, cents, k, idx64=0)
    assert got32.dtype == torch.int32
    assert torch.equal(got32.long(), launch(xyz, cents, k, idx64=1))


@pytest.mark.parametrize("k", [1, 3072])
def test_centre_on_a_point_far_away_and_far_from_the_origin(k):
    arch = clouds.dental_arch(24000, 90)[0]
    for shift in (0.0, 1000.0):
        xyz = arch + shift
        cents = torch.stack([xyz[17], xyz[23999], xyz.mean(0), xyz[5] + torch.tensor([40.0, -25.0, 60.0]),
                             torch.full((3,), shift - 500.0)])
        got = check(xyz[None], cents[None], k)
        assert got[0, 0, 0] == 17 and got[0, 1, 0] == 23999


def test_two_launches_are_bitwise_equal():
    xyz, cents, _ = coincident_mesh(seed=3)
    lat = lattice_cloud(91)[:24000]
    both = torch.stack([xyz, lat])
    cc = torch.stack([cents, lattice_centres(12, 2, 2, seed=92)])
    for k in (2, 3072):
        assert torch.equal(launch(both, cc, k), launch(both, cc, k))


@pytest.mark.parametrize("B,N,Q,k,message", [(1, 500, 2, 4097, "exceeds 4096"), (1, 0, 2, 8, "bad arguments"),
                                             (1, -3, 2, 8, "bad arguments"), (2, 0, 1, 4097, "bad arguments")])
def test_refusals_leave_out_untouched(B, N, Q, k, message):
    x = clouds.cube(max(N, 1) * B, 1).reshape(B, -1, 3).cuda()
    c = torch.zeros(B, Q, 3, device="cuda")
    for idx64, dtype in ((1, torch.int64), (0, torch.int32)):
        out = torch.full((B, Q, k), SENTINEL, dtype=dtype, device="cuda")
        with pytest.raises(L.TgnError, match=message):
            L.call("tgn_crop_knn", B, N, Q, k, L.ptr(x), L.ptr(c), L.ptr(out), idx64, L.stream_ptr())
        assert bool((out == SENTINEL).all())


@pytest.mark.parametrize("B,Q,k", [(0, 2, 8), (1, 0, 8), (1, 2, 0), (1, 2, -1)])
def test_empty_calls_write_nothing(B, Q, k):
    x = clouds.cube(100, 2).cuda()
    c = torch.zeros(2, 3, device="cuda")
    out = torch.full((2, 8), SENTINEL, dtype=torch.int64, device="cuda")
    L.call("tgn_crop_knn", B, 100, Q, k, L.ptr(x), L.ptr(c), L.ptr(out), 1, L.stream_ptr())
    torch.cuda.synchronize()
    assert bool((out == SENTINEL).all())
