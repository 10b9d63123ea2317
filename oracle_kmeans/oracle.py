"""oracle_kmeans/oracle.py -- numpy restatement of scikit-learn 1.9's float32 ``KMeans(init="k-means++").fit`` (TEST INFRASTRUCTURE ONLY).

Every rounding step of ``_kmeans_plusplus`` and ``_kmeans_single_lloyd`` is written out in the order that single-threaded
scikit-learn performs it on x86-64 with its bundled OpenBLAS 0.3.30 (SkylakeX kernels).  DESIGN §3.13 lists the orders and how
they were pinned.  csrc/kmeans.cu is checked against this module bit for bit.  Nothing under ``toothgroupnetwork_b200/`` may
import it.
"""
from __future__ import annotations

import numpy as np

f32, f64 = np.float32, np.float64


def prepare(X, n_clusters: int, random_state=None):
    """What ``KMeans.fit`` computes with numpy before seeding, and the draws of ``_kmeans_plusplus``, made with the same calls on
    the same generator: (X - X.mean(0), X.mean(0), tol, first index, (k-1, n_local_trials) uniforms)."""
    X = np.array(X, dtype=f32, order="C", copy=True)
    n = X.shape[0]
    # sklearn.utils.check_random_state for the three forms the tests pass
    rs = np.random.mtrand._rand if random_state is None else (
        random_state if isinstance(random_state, np.random.RandomState) else np.random.RandomState(random_state))
    sw = np.ones(n, dtype=f32)
    tol = np.mean(np.var(X, axis=0)) * 1e-4
    x_mean = X.mean(axis=0)
    X -= x_mean
    trials = 2 + int(np.log(n_clusters))
    first = int(rs.choice(n, p=sw / sw.sum()))
    u = np.stack([rs.uniform(size=trials) for _ in range(n_clusters - 1)]) if n_clusters > 1 else np.zeros((0, trials))
    return X, x_mean, f32(tol), first, u


def sdot_sum(x: np.ndarray) -> np.float32:
    """``x[None, :] @ ones`` (cblas_sdot, sdot_k_SKYLAKEX): 64 float32 lanes over the 64-blocks, folded to 32 lanes, one more
    32-block, lanes summed ((q0+q1)+q2)+q3 then pairwise within 8 and 4; the tail past the last 32-block is summed in float64
    and added to the kernel's part in float64."""
    n = x.size
    n1 = n & -32
    n64 = n1 & -64
    k = f32(0)
    if n1:
        acc = np.cumsum(x[:n64].reshape(-1, 64), axis=0, dtype=f32)[-1] if n64 else np.zeros(64, f32)
        acc = acc.reshape(4, 16)
        a = acc[:, :8] + acc[:, 8:]
        if n1 > n64:
            a = a + x[n64:n1].reshape(4, 8)
        s = ((a[0] + a[1]) + a[2]) + a[3]
        h = s[:4] + s[4:]
        k = f32(f32(h[0] + h[1]) + f32(h[2] + h[3]))
    t = 0.0
    for v in x[n1:].astype(f64):
        t = t + v
    return f32(t + f64(k))


def _block_sum(a: np.ndarray, kind: int) -> np.float32:
    """one column of sgemv_t_SKYLAKEX's sgemv_kernel_4x4 (kind 4), 4x2 (kind 2) or 4x1 (kind 1) over a block of 4m rows"""
    n = a.size
    i = 0
    if kind == 4:
        acc = np.zeros(8, f32)
        if n & 4:
            acc[:4] += a[:4]
            i = 4
        if (n - i) & 8:
            acc += a[i:i + 8]
            i += 8
        if n > i:
            acc = np.cumsum(np.concatenate([acc[None], a[i:].reshape(-1, 8)]), axis=0, dtype=f32)[-1]
        h = acc[:4] + acc[4:]
    else:
        acc = np.zeros(4, f32)
        if n & 4:
            acc += a[:4]
            i = 4
        rest = a[i:].reshape(-1, 2, 4)
        if kind == 2:
            if rest.size:
                acc = np.cumsum(np.concatenate([acc[None], rest.reshape(-1, 4)]), axis=0, dtype=f32)[-1]
        else:
            if rest.size:
                acc = np.cumsum(np.concatenate([acc[None], rest[:, 0]]), axis=0, dtype=f32)[-1] + \
                    np.cumsum(rest[:, 1], axis=0, dtype=f32)[-1]
        h = acc
    return f32(f32(h[0] + h[1]) + f32(h[2] + h[3]))


def sgemv_sum(rows: np.ndarray) -> np.ndarray:
    """``rows @ ones((n, 1))`` for 2 <= T rows (cblas_sgemv, sgemv_t_SKYLAKEX): row blocks of 4096 (the last one cut to a
    multiple of 4), each block's sum added to y in float32; columns in groups of 4, then 2, then 1, each with its kernel's lane
    order; the n % 4 trailing rows are added last as ((a0 + a1) + a2)."""
    T, m = rows.shape
    y = np.zeros(T, f32)
    m3 = m & 3
    m1 = m & -4
    m2 = (m & 4095) - m3
    NB, off = 4096, 0
    while NB == 4096:
        m1 -= NB
        if m1 < 0:
            if m2 == 0:
                break
            NB = m2
        for j in range(T):
            kind = 4 if j < (T & ~3) else (2 if j < (T & ~1) else 1)
            y[j] = f32(y[j] + _block_sum(rows[j, off:off + NB], kind))
        off += NB
    if m3:
        for j in range(T):
            s = rows[j, off]
            for q in range(1, m3):
                s = f32(s + rows[j, off + q])
            y[j] = f32(y[j] + s)
    return y


def _sq_dists64(X64: np.ndarray, xx: np.ndarray, c: int) -> np.ndarray:
    """_euclidean_distances_upcast for one centre: float32(((-2 * dot) + |c|^2) + |x|^2) in float64, clamped at 0"""
    dot = (X64[:, 0] * X64[c, 0] + X64[:, 1] * X64[c, 1]) + X64[:, 2] * X64[c, 2]
    return np.maximum(((-2.0 * dot + xx[c]) + xx).astype(f32), f32(0))


def _norms32(c: np.ndarray) -> np.ndarray:
    return (c[:, 0] * c[:, 0] + c[:, 1] * c[:, 1]) + c[:, 2] * c[:, 2]


def _fma32(a, b, c):
    """float32 fma(a, b, c) with one rounding: the product is exact in float64, the float64 sum is rounded to odd (TwoSum
    residual folded into the last bit), and rounding that to float32 is then correct."""
    p = a.astype(f64) * b.astype(f64)
    c = np.broadcast_to(c, p.shape).astype(f64)
    s = p + c
    bp = s - c
    e = (p - bp) + (c - (s - bp))
    bits = s.view(np.int64)
    odd = (e != 0) & ((bits & 1) == 0)
    bits = np.where(odd, bits + np.where((e > 0) == (s > 0), 1, -1), bits)
    return bits.view(f64).astype(f32)


def _assign(X: np.ndarray, centres: np.ndarray) -> np.ndarray:
    """_update_chunk_dense's labels: float32 ||c||^2 + (-2) * (x . c), the dot an FMA chain from x0 * c0 (the sgemm kernel),
    the first minimum winning"""
    acc = X[:, 0:1] * centres[None, :, 0]
    acc = _fma32(X[:, 1:2], centres[None, :, 1], acc)
    acc = _fma32(X[:, 2:3], centres[None, :, 2], acc)
    pd = _norms32(centres)[None, :] + f32(-2) * acc
    return np.argmin(pd, axis=1).astype(np.int32)


def _sqdist32(a: np.ndarray, b: np.ndarray) -> np.ndarray:
    """_euclidean_dense_dense with three features: ((0 + d0^2) + d1^2) + d2^2 in float32, no FMA"""
    d = a - b
    return ((f32(0) + d[:, 0] * d[:, 0]) + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]


def _shift_total(sq: np.ndarray) -> np.float32:
    """numpy's float32 ``sum`` of k values: pairwise_sum, eight lanes once k >= 8"""
    n = sq.size
    if n < 8:
        r = f32(0)
        for v in sq:
            r = f32(r + v)
        return r
    r = sq[:8].copy()
    m = n - n % 8
    for i in range(8, m, 8):
        r = r + sq[i:i + 8]
    res = f32(f32(f32(r[0] + r[1]) + f32(r[2] + r[3])) + f32(f32(r[4] + r[5]) + f32(r[6] + r[7])))
    for i in range(m, n):
        res = f32(res + sq[i])
    return res


def fit(Xc: np.ndarray, first: int, uniforms: np.ndarray, tol, max_iter: int = 300) -> dict:
    """One fit on prepared values (``prepare``): centred float32 (n, 3) points, the first seed, the per-centre uniforms and the
    float32 tolerance.  Centres are returned centred; ``relocated`` is True when a cluster emptied (scikit-learn relocates it;
    that step is not restated, and the other outputs are then meaningless)."""
    Xc = np.ascontiguousarray(Xc, dtype=f32)
    n = Xc.shape[0]
    k = uniforms.shape[0] + 1
    X64 = Xc.astype(f64)
    xx = (X64[:, 0] * X64[:, 0] + X64[:, 1] * X64[:, 1]) + X64[:, 2] * X64[:, 2]
    init = np.empty(k, np.int64)
    init[0] = first
    closest = _sq_dists64(X64, xx, first)
    pot = sdot_sum(closest)
    for c in range(1, k):
        rand_vals = uniforms[c - 1] * f64(pot)
        cum = np.cumsum(closest, dtype=f32)
        cand = np.minimum(np.searchsorted(cum.astype(f64), rand_vals), n - 1)
        dist = np.minimum(closest[None, :], np.stack([_sq_dists64(X64, xx, int(j)) for j in cand]))
        pots = sgemv_sum(dist)
        best = int(np.argmin(pots))
        pot, closest, init[c] = pots[best], dist[best], cand[best]
    centres = Xc[init].copy()

    labels_old = np.full(n, -1, np.int32)
    strict = False
    relocated = False
    for it in range(max_iter):
        labels = _assign(Xc, centres)
        new = np.zeros((k, 3), f32)
        counts = np.bincount(labels, minlength=k)
        if (counts == 0).any():
            relocated = True
            break
        order = np.argsort(labels, kind="stable")
        starts = np.concatenate([[0], np.cumsum(counts)[:-1]])
        for j in range(k):                                               # index-order float32 chain over the members
            new[j] = f32(0) + np.cumsum(Xc[order[starts[j]:starts[j] + counts[j]]], axis=0, dtype=f32)[-1]
        alpha = (1.0 / counts.astype(f32).astype(f64)).astype(f32)
        new = new * alpha[:, None]
        shift = np.sqrt(_sqdist32(new, centres).astype(f64)).astype(f32)
        centres = new
        if np.array_equal(labels, labels_old):
            strict = True
            break
        if _shift_total(shift * shift) <= tol:
            break
        labels_old = labels
    n_iter = it + 1
    if not strict and not relocated:
        labels = _assign(Xc, centres)
    inertia = f32(0)
    for v in _sqdist32(Xc, centres[labels]):
        inertia = f32(inertia + v)
    return dict(labels=labels, init=init, centers=centres, n_iter=n_iter, inertia=inertia, relocated=relocated)


def kmeans(X, n_clusters: int, random_state=None, max_iter: int = 300) -> dict:
    """``KMeans(n_clusters, random_state=random_state).fit(X)`` restated: labels, init (the k-means++ indices), centers
    (``cluster_centers_``), n_iter, inertia, relocated."""
    Xc, x_mean, tol, first, u = prepare(X, n_clusters, random_state)
    out = fit(Xc, first, u, tol, max_iter)
    out["centers"] = out["centers"] + x_mean
    return out
