"""GPU: the c = 16 schedule of the fused point-transformer layer (csrc/pt_layer.cu: two queries per warp, one per half-warp) called
through tgn_pt_layer_forward directly, one pass at a time, against its float64 restatement (oracle/pt_layer.py), with the bounds,
the 4-ulp running-statistics bar and the write guards of tests/test_gpu_pt_layer.py.

Shapes: the boundary network's first level (one cloud of 24 000 points; 16 crops of 3 072 packed), the K edges 1..64, and the n
edges of the pair loop -- n = 1 and every odd n leave one half-warp without a query, and 2 x (4 SMs x 8 warps) pairs + 1 or + 2
wrap the grid-stride loop once with one or both halves busy.  The c = 16 schedule ignores the CTA threshold."""
import pytest
import torch

from oracle import pt_layer
from test_gpu_pt_layer import CTA, DEFAULT, WARP, _all_modes, _case, _launch, _sms, _threshold

pytestmark = pytest.mark.gpu
C = 16


@pytest.mark.parametrize("K,n,crops", [(36, 24000, 1), (36, 49152, 16)])
def test_boundary_network_level(K, n, crops):
    _all_modes(_case(C, K, n, crops), DEFAULT)


@pytest.mark.parametrize("K", [1, 2, 7, 8, 9, 33, 36, 64])
def test_k_edges(K):
    _all_modes(_case(C, K, 1000), DEFAULT)


@pytest.mark.parametrize("n", [1, 2, 3, 31, 33, "grid+1", "grid+2"])
def test_n_edges(n):
    """odd n: the last warp's upper half has no query and must keep nothing while it joins the shuffles"""
    grid = 2 * 8 * 4 * _sms()                    # queries of one grid-stride step: 4 CTAs per SM x 8 warps x 2 halves
    n = {"grid+1": grid + 1, "grid+2": grid + 2}.get(n, n)
    _all_modes(_case(C, 16, n), DEFAULT)


@pytest.mark.parametrize("kind", ["plain", "saturated", "uniform"])
@pytest.mark.parametrize("crops", [1, 16])
def test_softmax_cases(kind, crops):
    """near one-hot logits (x 100) and an exactly uniform softmax (b_w = 0), next to unit-scale data"""
    _all_modes(_case(C, 36, 6144, crops, kind), DEFAULT)


def test_offset_channel():
    """the default "hard" case offsets xk by 140 on channel 0 (and 1400 on channel 4): BatchNorm_a sees
    |mean| / std ~ 100 there, and the fp64 sums must keep its variance"""
    f = _case(C, 36, 6000)
    s, _ = pt_layer.batch_sums(passes=(1,), **f)["a"]
    rows = f["n"] * f["K"]
    mean = s[0] / rows
    std = (s[C] / rows - mean * mean).sqrt()
    assert 50.0 < float(mean.abs() / std) < 200.0
    _all_modes(f, DEFAULT)


def test_cta_threshold_does_not_apply():
    """1023 and 1024 queries (either side of the default threshold), all modes under the default threshold; the output pass
    under the default, always-CTA and never-CTA thresholds is the same half-warp launch, bit for bit"""
    for n in (1023, 1024):
        f = _case(C, 36, n)
        _all_modes(f, DEFAULT)
        outs = []
        for thr in (DEFAULT, CTA, WARP):
            with _threshold(thr):
                outs.append(_launch(f, [2, 2, 2], update=0)["out"])      # no fp64 atomics: deterministic
        assert all(torch.equal(o, outs[0]) for o in outs[1:]), n
