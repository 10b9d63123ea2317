"""Seeded synthetic point clouds (SURVEY.md 8d): the inputs every parity test, golden
fixture and bench line is quoted on.  CPU generators (torch.Generator) so that the same
seed gives the same cloud in this container and on the GPU box.

* ``cube``  -- xyz ~ U[-1,1]^3 ("synthetic random cloud", BASELINE config C1).
* ``dental_arch`` -- half-torus tube (centre line radius 0.6, tube radius 0.18, sigma 0.002
  noise) with analytic normals: surface-like density, so balls of r <= 0.1 hold >= K points the
  way real scans normalised per ``preprocess_data.py:48-50`` do (configs C2-C5).
"""
from __future__ import annotations

import math
from typing import Tuple

import torch


def cloud_seed(rank: int, j: int) -> int:
    """Cloud j on rank r uses seed 1000*r + j (SURVEY.md 8d)."""
    return 1000 * int(rank) + int(j)


def cube(n: int, seed: int = 0) -> torch.Tensor:
    g = torch.Generator().manual_seed(int(seed))
    return (torch.rand(n, 3, generator=g, dtype=torch.float32) * 2.0 - 1.0).contiguous()


def dental_arch(n: int, seed: int = 0) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """Returns (xyz (n,3), normal (n,3), label (n,) int64).  Labels: 16 equal u-bins ("teeth")
    on the upper half of the tube (sin v > 0), -1 ("gingiva") elsewhere."""
    g = torch.Generator().manual_seed(int(seed))
    u = torch.rand(n, generator=g, dtype=torch.float32) * math.pi
    v = torch.rand(n, generator=g, dtype=torch.float32) * (2.0 * math.pi)
    noise = torch.randn(n, 3, generator=g, dtype=torch.float32) * 0.002
    cu, su, cv, sv = torch.cos(u), torch.sin(u), torch.cos(v), torch.sin(v)
    centre = torch.stack([0.6 * cu, 0.6 * su - 0.3, torch.zeros_like(u)], 1)
    e_r = torch.stack([cu, su, torch.zeros_like(u)], 1)
    e_z = torch.tensor([0.0, 0.0, 1.0]).expand(n, 3)
    normal = cv[:, None] * e_r + sv[:, None] * e_z
    xyz = (centre + 0.18 * normal + noise).contiguous()
    label = torch.where(sv > 0, torch.clamp((u / math.pi * 16).long(), max=15), torch.full_like(u, -1).long())
    return xyz, normal.contiguous(), label


def arch_features(n: int, seed: int = 0) -> torch.Tensor:
    """(1, 6, n) channel-first feature tensor [xyz; normal] as the models consume it
    (``models/modules/grouping_network_module.py:16-23``)."""
    xyz, normal, _ = dental_arch(n, seed)
    return torch.cat([xyz, normal], 1).t().contiguous().unsqueeze(0)


def boundary_inputs(m: int, seed: int = 0, n_sampled: int = 24000, label_noise: float = 0.0):
    """numpy inputs of the boundary resampling between tgnet's two networks (inference_pipeline_tgn.py:289-330):
    org_feats (m,6) float64 -- dental_arch vertices with float64 jitter (coordinates that are not float32 values, so distances do
    not tie) and their normals; sampled_feats (n_sampled,6) -- a seeded subset of those rows, as the FPS of the mesh would be;
    point_labels (n_sampled,) float64 -- the arch's tooth bins + 1 (0 = gingiva), a share ``label_noise`` of them replaced by
    random labels (a poorly trained first network)."""
    import numpy as np
    xyz, normal, label = dental_arch(m, seed)
    rng = np.random.default_rng(int(seed) + 104729)
    org = np.concatenate([xyz.double().numpy() + rng.normal(0.0, 1e-4, (m, 3)), normal.double().numpy()], 1)
    rows = np.sort(rng.choice(m, n_sampled, replace=False))
    labels = label.numpy()[rows].astype(np.float64) + 1.0
    noisy = rng.random(n_sampled) < label_noise
    labels[noisy] = rng.integers(0, 17, int(noisy.sum())).astype(np.float64)
    return org, org[rows].copy(), labels


LATTICE_STEP = 0.125
LATTICE_HALF = 64


def lattice(half: int, seed: int = 0, n: int | None = None) -> torch.Tensor:
    """The points (i, j, l) / 8 with |i|, |j|, |l| <= half (half <= LATTICE_HALF), shuffled by the seed; the first n of them when
    n is given.  On these coordinates, and on queries on the half-step lattice (2i + 1) / 16 between them, every product and
    partial sum of the float32 distance forms the kernels evaluate is exact, so their distances equal float64's and tie
    wherever the true distances do (tests/test_cpu_lattice_exact.py): the tie stress input of the neighbour selections."""
    assert 0 <= half <= LATTICE_HALF
    g = torch.Generator().manual_seed(int(seed) + 104723)
    axis = torch.arange(-half, half + 1, dtype=torch.float32) * LATTICE_STEP
    pts = torch.cartesian_prod(axis, axis, axis)
    pts = pts[torch.randperm(pts.shape[0], generator=g)]
    return (pts if n is None else pts[:n]).contiguous()


def with_duplicates(xyz: torch.Tensor, seed: int = 0) -> torch.Tensor:
    """Every vertex twice, shuffled: the FPS / kNN tie-break stress input (SURVEY.md 7.1)."""
    g = torch.Generator().manual_seed(int(seed) + 7919)
    both = torch.cat([xyz, xyz], 0)
    return both[torch.randperm(both.shape[0], generator=g)].contiguous()
