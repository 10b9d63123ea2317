"""CPU: the premise of the lattice tests of the neighbour selections (test_gpu_crop_knn_edges.py, the lattice cases of
test_gpu_pointops.py and test_gpu_ball_windows.py).  On points (i, j, l) / 8 with |i|, |j|, |l| <= 64 and queries on the
half-step lattice between them, every product and every partial sum of the float32 distance forms the kernels evaluate is
a float32 value, so neither a rounded nor a fused multiply-add changes it, and the float32 distance equals the float64 one:

* the expanded form of the ball query and three_nn, (-2 dot + |a|^2) + |b|^2 with dot = fma(az, bz, fma(ay, by, ax bx)) (and
  the one-column variant fma(ay, by, ax bx) + az bz), with |p|^2 in both the index order (x x + y y) + z z and the
  contiguous-reduce order (x x + z z) + y y;
* the difference form of the kNN kernels, fma(dz, dz, fma(dx, dx, dy dy)).

If this stops holding, a float64 brute force is no longer the exact reference of those tests."""
import numpy as np
import pytest

from toothgroupnetwork_b200 import clouds

HALF = clouds.LATTICE_HALF


def pairs(seed, n=200_000):
    """n (point, query) pairs: points on the 1/8 lattice, queries on it or on the half-step lattice, including the corners
    and the half-step cells just outside them (the largest magnitudes)."""
    rng = np.random.default_rng(seed)
    a = rng.integers(-HALF, HALF + 1, (n, 3)) / 8.0
    b = np.where(rng.random((n, 1)) < 0.5, rng.integers(-HALF, HALF + 1, (n, 3)) / 8.0,
                 (2 * rng.integers(-HALF - 1, HALF + 1, (n, 3)) + 1) / 16.0)
    near = a[: n // 10] + rng.integers(-2, 3, (n // 10, 3)) / 8.0            # neighbours: shells at r = 0.25 and below
    b[: n // 10] = np.clip(near, -HALF / 8.0, HALF / 8.0)
    ext = np.array([s * HALF / 8.0 for s in (-1, 1)] + [s * (2 * HALF + 1) / 16.0 for s in (-1, 1)])
    corners = np.stack(np.meshgrid(ext, ext, ext, indexing="ij"), -1).reshape(-1, 3)
    a = np.concatenate([a, np.repeat(corners, len(corners), 0)])
    b = np.concatenate([b, np.tile(corners, (len(corners), 1))])
    # every value is a float32 value to start with
    assert np.array_equal(a.astype(np.float32).astype(np.float64), a) and np.array_equal(b.astype(np.float32).astype(np.float64), b)
    return a, b


def exact_in_f32(*values):
    for v in values:
        assert np.array_equal(v.astype(np.float32).astype(np.float64), v), "a partial result is not a float32 value"


def sq_norm(p, contiguous_order):
    x, y, z = p[:, 0], p[:, 1], p[:, 2]
    first = x * x + (z * z if contiguous_order else y * y)
    exact_in_f32(x * x, y * y, z * z, first)
    return first + (y * y if contiguous_order else z * z)


def float64_d2(a, b):
    d = a - b
    return (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]


@pytest.mark.parametrize("order_a", [False, True])
@pytest.mark.parametrize("order_b", [False, True])
def test_expanded_form_is_exact(order_a, order_b):
    a, b = pairs(1 + 2 * order_a + order_b)
    an, bn = sq_norm(a, order_a), sq_norm(b, order_b)
    p = a * b
    dot = (p[:, 0] + p[:, 1]) + p[:, 2]
    one_column = (p[:, 1] + p[:, 0]) + p[:, 2]
    exact_in_f32(p[:, 0], p[:, 1], p[:, 2], p[:, 0] + p[:, 1], dot, an, bn, -2.0 * dot, -2.0 * dot + an)
    d = (-2.0 * dot + an) + bn
    exact_in_f32(d)
    assert np.array_equal(one_column, dot)
    assert np.array_equal(d, float64_d2(a, b))
    # and float32 arithmetic itself, step by step (unfused; the fused steps have the same exact results)
    a32, b32 = a.astype(np.float32), b.astype(np.float32)
    n32 = [(q[:, 0] * q[:, 0] + (q[:, 2] * q[:, 2] if o else q[:, 1] * q[:, 1])) + (q[:, 1] * q[:, 1] if o else q[:, 2] * q[:, 2])
           for q, o in ((a32, order_a), (b32, order_b))]
    dot32 = (a32[:, 0] * b32[:, 0] + a32[:, 1] * b32[:, 1]) + a32[:, 2] * b32[:, 2]
    d32 = (np.float32(-2.0) * dot32 + n32[0]) + n32[1]
    assert d32.dtype == np.float32 and np.array_equal(d32.astype(np.float64), d)
    # the ball-query radius of the lattice tests: r = 0.25 gives float32(r^2) = 1/16 exactly, and shells land on it
    assert float(np.float32(0.25 ** 2)) == 0.0625 and (d == 0.0625).any()


def test_difference_form_is_exact():
    a, b = pairs(7)
    d = b - a
    exact_in_f32(d)
    sq = d * d
    exact_in_f32(sq, sq[:, 1] + sq[:, 0])
    got = (sq[:, 1] + sq[:, 0]) + sq[:, 2]
    exact_in_f32(got)
    assert np.array_equal(got, float64_d2(a, b))
    d32 = b.astype(np.float32) - a.astype(np.float32)
    got32 = (d32[:, 1] * d32[:, 1] + d32[:, 0] * d32[:, 0]) + d32[:, 2] * d32[:, 2]
    assert got32.dtype == np.float32 and np.array_equal(got32.astype(np.float64), got)


def test_lattice_builder():
    pts = clouds.lattice(3, seed=5).numpy()
    assert pts.shape == (7 ** 3, 3) and len(np.unique(pts, axis=0)) == 7 ** 3
    assert np.array_equal(np.sort(np.unique(pts[:, 0])), np.arange(-3, 4) / 8.0)
    assert not np.array_equal(pts, clouds.lattice(3, seed=6).numpy())
    assert np.array_equal(clouds.lattice(3, seed=5, n=40).numpy(), pts[:40])
