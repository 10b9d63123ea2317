"""CPU: oracle.point_transformer_layer at c = 16 -- the boundary network's first level, PointTransformerLayer(16, 16, 8, 36) --
against the reference's own blocks.py output (tests/golden/ref_torch_blocks16.npz, made by make_ref_blocks16_golden.py), in
train() and eval() BatchNorm mode; and the float64 restatement's error bounds (oracle/pt_layer.py) at c = 16, which the GPU tests
of the kernel's c = 16 schedule apply unchanged."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import oracle as O  # noqa: E402
from toothgroupnetwork_b200 import clouds  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")


@pytest.mark.parametrize("train_bn", [True, False])
def test_oracle_point_transformer_layer_matches_the_reference_layer_at_c16(train_bn):
    fix = np.load(os.path.join(GOLD, "ref_torch_blocks16.npz"))
    state = {k[len("ptl16_state_"):]: torch.from_numpy(fix[k]) for k in fix.files if k.startswith("ptl16_state_")}
    assert state["linear_w.2.weight"].shape == (2, 16)                      # c / share_planes = 2
    p, o, x = torch.from_numpy(fix["p"]), torch.from_numpy(fix["o"]), torch.from_numpy(fix["ptl16_x"])
    K = int(fix["ptl16_K"])
    assert K == 36 and x.shape == (700, 16)
    want = torch.from_numpy(fix["ptl16_out_train" if train_bn else "ptl16_out_eval"])
    got = O.point_transformer_layer(p, x, o, state, K, 8, train_bn)
    assert got.shape == want.shape
    assert float((got - want).abs().max()) <= 2e-5 * float(want.abs().max())
    exact = O.point_transformer_layer(p, x, o, state, K, 8, train_bn, dtype=torch.float64)
    assert float((exact.float() - want).abs().max()) <= 2e-5 * float(want.abs().max())


@pytest.mark.parametrize("kind", ["plain", "hard", "saturated", "uniform"])
@pytest.mark.parametrize("n_crops,per_crop", [(1, 1500), (16, 96)])
def test_restatement_bound_holds_for_float32_evaluation_at_c16(kind, n_crops, per_crop):
    """oracle/pt_layer.py's error bounds at c = 16 (c / 8 = 2 share columns, K = 36): the restatement evaluated in float32,
    conditioned on the float64 evaluation's sums, lies within the bound of every sum and every output element"""
    from oracle import pt_layer
    p = torch.cat([clouds.dental_arch(per_crop, 16 + k)[0] for k in range(n_crops)]).contiguous()
    o = torch.arange(1, n_crops + 1, dtype=torch.int32) * per_crop
    idx, _, _ = O.knnquery(36, p.numpy(), p.numpy(), o.numpy(), o.numpy())
    f = pt_layer.make_case(16, 36, p, torch.from_numpy(np.ascontiguousarray(idx)), kind, seed=52)
    f32 = {k: v.float() if torch.is_tensor(v) and v.is_floating_point() else v for k, v in f.items()}
    s64 = pt_layer.batch_sums(**f)
    cond = {"stats_" + t: s for t, (s, _) in s64.items()}
    s32 = pt_layer.batch_sums(dtype=torch.float32, **f32, **cond)
    for tag, (s, b) in s64.items():
        assert bool(((s32[tag][0] - s).abs() <= 0.999 * b).all()), tag
    out, bound = pt_layer.output(**f, **cond)
    out32, _ = pt_layer.output(dtype=torch.float32, **f32, **cond)
    assert bool(((out32.double() - out).abs() <= 0.999 * bound).all())
