"""oracle_meanshift/oracle.py -- numpy restatement of scikit-learn 1.9's float64 ``MeanShift(bandwidth).fit`` (TEST INFRASTRUCTURE ONLY).

The seed ascent of ``_mean_shift_single_seed`` is written out from the points, the ``idx_array`` of scikit-learn's
``KDTree(X, leaf_size=30)``, the bandwidth and ``max_iter``; the tree's node structure is not needed, because a radius query
returns its members in ascending tree position.  DESIGN §3.14 gives the three rules and how they were pinned:

- membership: the float64 reduced distance ((0 + dx*dx) + dy*dy) + dz*dz <= r*r, unfused;
- order: members in ascending position of ``idx_array``; ``np.mean(axis=0)`` adds them in one float64 chain from the first
  member, then divides by the count;
- stop: ``np.linalg.norm`` of the step as OpenBLAS's ddot computes it, sqrt(fma(dz,dz, fma(dy,dy, dx*dx))), ``<= 1e-3 * r``.

csrc/meanshift.cu is checked against this module bit for bit, flags included.  Nothing under ``toothgroupnetwork_b200/``
may import it.
"""
from __future__ import annotations

from fractions import Fraction
import math

import numpy as np

BAND = 2.0 ** -40           # flag margin, relative to r^2 and stop^2
CHUNK = 128                 # seeds per vectorised block


def fma(a: float, b: float, c: float) -> float:
    """a * b + c rounded once (math.fma from Python 3.13; exact rationals before)"""
    if hasattr(math, "fma"):
        return math.fma(a, b, c)
    return float(Fraction(a) * Fraction(b) + Fraction(c))


def step_sq(new: np.ndarray, old: np.ndarray) -> float:
    """the square of ``np.linalg.norm(new - old)`` in OpenBLAS ddot's order for a 3-vector"""
    d = new - old
    dx, dy, dz = float(d[0]), float(d[1]), float(d[2])
    return fma(dz, dz, fma(dy, dy, dx * dx))


def ascent(X: np.ndarray, idx_array: np.ndarray, bandwidth: float, max_iter: int = 300):
    """Every seed's ``_mean_shift_single_seed`` with seeds = X.  Returns (means (n,3) float64, counts (n) int64, iters (n) int64,
    flags (n) bool), indexed like X.  A seed is flagged when a reduced distance came within 2^-40 r^2 of r^2 or a squared step
    within 2^-40 stop^2 of stop^2."""
    X = np.asarray(X, dtype=np.float64)
    Xt = X[idx_array]
    n = X.shape[0]
    r2 = bandwidth * bandwidth
    stop = 1e-3 * bandwidth
    st2 = stop * stop
    means = Xt.copy()
    counts = np.zeros(n, np.int64)
    iters = np.zeros(n, np.int64)
    flags = np.zeros(n, bool)
    active = np.arange(n)
    it = 0
    while active.size:
        still = []
        for c0 in range(0, active.size, CHUNK):
            a = active[c0:c0 + CHUNK]
            q = means[a]
            d = q[:, None, :] - Xt[None, :, :]
            rd = (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]
            inside = rd <= r2
            flags[a] |= (np.abs(rd - r2) <= r2 * BAND).any(1)
            m = inside.sum(1)
            # -0.0 is the exact additive identity, so the chain over non-members is the chain over members from the first one
            s = np.add.accumulate(np.where(inside[..., None], Xt[None, :, :], -0.0), axis=1)[:, -1, :]
            for j, i in enumerate(a):
                if m[j] == 0:
                    continue
                counts[i] = m[j]
                new = s[j] / m[j]
                sq = step_sq(new, means[i])
                flags[i] |= abs(sq - st2) <= st2 * BAND
                means[i] = new
                if math.sqrt(sq) <= stop or it == max_iter:
                    continue
                still.append(i)
        active = np.array(still, dtype=np.int64)
        it += 1
        iters[active] = it
    out = np.empty_like(means)
    out[idx_array] = means
    res = [np.empty_like(v) for v in (counts, iters, flags)]
    for o, v in zip(res, (counts, iters, flags)):
        o[idx_array] = v
    return out, res[0], res[1], res[2]


def postprocess(X: np.ndarray, means: np.ndarray, counts: np.ndarray, iters: np.ndarray, bandwidth: float):
    """``MeanShift.fit`` after the ascent, with brute-force float64 distances: (cluster_centers_, labels_, n_iter_)."""
    intensity = {}
    for mean, c in zip(means, counts):
        if c:
            intensity[tuple(mean)] = int(c)                # -0.0 and +0.0 make the same key; the first key and last count stay
    ranked = sorted(intensity.items(), key=lambda kv: (kv[1], kv[0]), reverse=True)
    centers = np.array([kv[0] for kv in ranked])
    unique = np.ones(len(centers), bool)
    for i, c in enumerate(centers):
        if unique[i]:
            d = centers - c
            unique[np.sqrt((d * d).sum(1)) <= bandwidth] = False
            unique[i] = True
    centers = centers[unique]
    d = X[:, None, :] - centers[None, :, :]
    labels = np.argmin((d * d).sum(2), axis=1)
    return centers, labels, int(iters.max())
