"""CPU: the fused PointTransformerBlock's descriptors (include/tgn_b200.h against the ctypes mirror), oracle/pt_block.py against
torch's own float64 modules, and the drop-in's routing of CPU tensors.  The other routing cases (autograd, widths, a bias,
momentum=None) need CUDA tensors to reach their own check and are in tests/test_gpu_pt_block.py."""
import ctypes
import os
import shutil
import subprocess
import tempfile
import types

import pytest
import torch
import torch.nn as nn

from oracle import pt_block as B
from toothgroupnetwork_b200 import _lib as L
from toothgroupnetwork_b200 import blocks_fused

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class Layer(nn.Module):
    """blocks.PointTransformerLayer's attributes (blocks.py:15-29); forward over given neighbours idx (n, K), in torch modules"""

    def __init__(self, c, nsample, share=8):
        super().__init__()
        self.mid_planes = self.out_planes = c
        self.share_planes, self.nsample = share, nsample
        self.linear_q, self.linear_k, self.linear_v = nn.Linear(c, c), nn.Linear(c, c), nn.Linear(c, c)
        self.linear_p = nn.Sequential(nn.Linear(3, 3), nn.BatchNorm1d(3), nn.ReLU(inplace=True), nn.Linear(3, c))
        self.linear_w = nn.Sequential(nn.BatchNorm1d(c), nn.ReLU(inplace=True), nn.Linear(c, c // share), nn.BatchNorm1d(c // share),
                                      nn.ReLU(inplace=True), nn.Linear(c // share, c // share))
        self.idx = None

    def forward(self, pxo):
        p, x, _ = pxo
        idx = self.idx
        q, k, v = self.linear_q(x), self.linear_k(x), self.linear_v(x)
        rel = p[idx] - p.unsqueeze(1)
        for i, m in enumerate(self.linear_p):                       # BatchNorm over the (n, c, K) view, as blocks.py:38
            rel = m(rel.transpose(1, 2)).transpose(1, 2) if i == 1 else m(rel)
        w = k[idx] - q.unsqueeze(1) + rel
        for i, m in enumerate(self.linear_w):
            w = m(w.transpose(1, 2)).transpose(1, 2) if i % 3 == 0 else m(w)
        w = torch.softmax(w, dim=1)
        n, K, c = rel.shape
        s = self.share_planes
        return ((v[idx] + rel).view(n, K, s, c // s) * w.unsqueeze(2)).sum(1).view(n, c)


class Block(nn.Module):
    """blocks.PointTransformerBlock's attributes (blocks.py:117-125) and its forward (:127-135) around ``Layer``"""

    def __init__(self, c, nsample, bias=False):
        super().__init__()
        self.linear1 = nn.Linear(c, c, bias=bias)
        self.bn1 = nn.BatchNorm1d(c)
        self.transformer2 = Layer(c, nsample)
        self.bn2 = nn.BatchNorm1d(c)
        self.linear3 = nn.Linear(c, c, bias=False)
        self.bn3 = nn.BatchNorm1d(c)
        self.relu = nn.ReLU(inplace=True)

    def forward(self, pxo):
        p, x, o = pxo
        identity = x
        x = self.relu(self.bn1(self.linear1(x)))
        x = self.relu(self.bn2(self.transformer2([p, x, o])))
        x = self.bn3(self.linear3(x))
        x += identity
        return [p, self.relu(x), o]


def _randomise(module, gen):
    with torch.no_grad():
        for m in module.modules():
            if isinstance(m, nn.BatchNorm1d):
                m.weight.copy_(torch.randn(m.weight.shape, generator=gen))           # negative gammas too
                m.bias.copy_(torch.randn(m.bias.shape, generator=gen) * 0.2)
                m.running_mean.copy_(torch.randn(m.running_mean.shape, generator=gen) * 0.2)
                m.running_var.copy_(torch.rand(m.running_var.shape, generator=gen) + 0.5)


def test_descriptor_sizes_and_offsets_match_the_header():
    assert ctypes.sizeof(L.PtResApply) == ctypes.sizeof(L.PwApply) + 16
    assert L.PtResApply.apply.offset == 0 and L.PtResApply.identity.offset == ctypes.sizeof(L.PwApply)
    assert L.PtResApply.identity_row_stride.offset == ctypes.sizeof(L.PwApply) + 8
    assert L.PtLayerSums.layer.offset == 0 and L.PtLayerSums.out_stats.offset == ctypes.sizeof(L.PtLayer)
    assert ctypes.sizeof(L.PtLayerSums) == ctypes.sizeof(L.PtLayer) + 8
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("no C compiler for the header's own offsets")
    src = r"""
#include <stdio.h>
#include <stddef.h>
#include "tgn_b200.h"
int main(void) {
    printf("%zu %zu %zu %zu %zu %zu\n", sizeof(tgn_pt_res_apply_t), offsetof(tgn_pt_res_apply_t, identity),
           offsetof(tgn_pt_res_apply_t, identity_row_stride), sizeof(tgn_pt_layer_sums_t), offsetof(tgn_pt_layer_sums_t, out_stats),
           sizeof(tgn_pt_layer_t));
    return 0;
}
"""
    with tempfile.TemporaryDirectory() as d:
        with open(os.path.join(d, "t.c"), "w") as f:
            f.write(src)
        exe = os.path.join(d, "t")
        subprocess.run([cc, "-I", os.path.join(ROOT, "include"), os.path.join(d, "t.c"), "-o", exe], check=True)
        got = [int(v) for v in subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split()]
    assert got == [ctypes.sizeof(L.PtResApply), L.PtResApply.identity.offset, L.PtResApply.identity_row_stride.offset,
                   ctypes.sizeof(L.PtLayerSums), L.PtLayerSums.out_stats.offset, ctypes.sizeof(L.PtLayer)]
    assert {"tgn_pt_res_apply", "tgn_pt_layer_forward_sums"} <= set(L._SIGS)
    assert {"tgn_pt_res_apply_struct_size", "tgn_pt_layer_sums_struct_size"} <= set(L.EXPORTS)


@pytest.mark.parametrize("c,K,n", [(16, 36, 300), (32, 36, 257), (64, 24, 130)])
@pytest.mark.parametrize("train", [True, False])
def test_oracle_matches_torchs_float64_block(c, K, n, train):
    gen = torch.Generator().manual_seed(c * 10 + K)
    blk = Block(c, K)
    _randomise(blk, gen)
    blk = blk.double().train(train)
    p = torch.rand(n, 3, generator=gen, dtype=torch.float64)
    x = torch.randn(n, c, generator=gen, dtype=torch.float64) + 3.0 * torch.randn(1, c, generator=gen, dtype=torch.float64)
    idx = torch.argsort(torch.cdist(p, p), dim=1)[:, :K]
    blk.transformer2.idx = idx
    state = {k: v.clone() for k, v in blk.state_dict().items()}
    x0 = x.clone()
    with torch.no_grad():
        want = blk([p, x, torch.tensor([n], dtype=torch.int32)])[1]
    assert torch.equal(x, x0)                                  # the reference's += acts on bn3's output
    got, after = B.block(state, p, x, idx, train)
    assert torch.allclose(got, want, rtol=1e-10, atol=1e-10)
    sd = blk.state_dict()
    if train:
        assert len(after) == 3 * 6
        for k, v in after.items():
            assert torch.allclose(sd[k].double(), v.double(), rtol=1e-10, atol=1e-12), k
    else:
        assert after == {}


def test_res_apply_oracle_is_relu_of_bn_plus_identity():
    gen = torch.Generator().manual_seed(3)
    c, n = 8, 50
    bn = nn.BatchNorm1d(c).double()
    _randomise(bn, gen)
    y = torch.randn(c, n, generator=gen, dtype=torch.float64) * 4 + 10
    ident = torch.randn(n, c, generator=gen, dtype=torch.float64)
    state = {k: v.clone() for k, v in bn.state_dict().items()}
    for train in (False, True):                                # the train-mode call updates bn's running statistics
        got, err, after = B.res_apply(y, state, "", ident, train)
        with torch.no_grad():
            want = torch.relu(bn.train(train)(y.t().clone()) + ident)
        assert torch.allclose(got, want, rtol=1e-12, atol=1e-12)
        assert bool((err > 0).all()) and bool((err < 1e-4 * (want.abs() + 1)).all())
        assert ("running_mean" in after) == train


def test_cpu_tensors_and_wrapping_keep_the_original_forward():
    calls = []

    class PointTransformerBlock(Block):
        def forward(self, pxo):
            calls.append("original")
            return super().forward(pxo)

    mod = types.SimpleNamespace(PointTransformerBlock=PointTransformerBlock)
    blocks_fused.accelerate_blocks(mod)
    blocks_fused.accelerate_blocks(mod)                        # idempotent
    assert PointTransformerBlock._tgn_fused
    blk = PointTransformerBlock(16, 4)
    blk.transformer2.idx = torch.zeros(8, 4, dtype=torch.long)
    p, x, o = torch.rand(8, 3), torch.randn(8, 16), torch.tensor([8], dtype=torch.int32)
    assert not blocks_fused.pt_block_fusable(blk, p, x, o)
    with torch.no_grad():
        blk([p, x, o])
    assert calls == ["original"]
