"""CPU: the host side of the CUDA-graph replay of the point-transformer network's forward (toothgroupnetwork_b200/graphs.py) on the
reference's module built on the CPU: every change the graph key must cover changes it, an unchanged module keeps it, and a CPU
input is not eligible and runs the class's previous forward."""
import pytest
import torch

from oracle import ref_models
from toothgroupnetwork_b200 import _lib as L
from toothgroupnetwork_b200 import blocks_fused, dropin, graphs, pointops
from toothgroupnetwork_b200 import pointnet2_utils as pn2

needs_reference = pytest.mark.skipif(not ref_models.available(), reason="reference snapshot not staged")
FIRST = {"stride": [1, 4, 4, 4, 4], "nsample": [36, 24, 24, 24, 24], "blocks": [2, 3, 4, 6, 3], "block_num": 5,
         "planes": [32, 64, 128, 256, 512]}
CPM = "models.modules.cbl_point_transformer.cbl_point_transformer_module"


@pytest.fixture(scope="module")
def world():
    w = ref_models.World("b200")
    dropin.accelerate_decoder(w.mod("models.modules.cbl_point_transformer.blocks"), w.mod("models.modules.cbl_point_transformer.heads"))
    dropin.accelerate_transformer_blocks(w.mod("models.modules.cbl_point_transformer.blocks"))
    dropin.accelerate_graphs(w.mod(CPM))
    return w


@pytest.fixture
def model(world):
    torch.manual_seed(0)
    with world:
        return world.mod(CPM).get_model(c=6, k=17, **FIRST)


def _key(m, x):
    return graphs.graph_key(m, x)[0]


def _flip(setter, getter):
    old = getter()
    setter(not old)
    return lambda: setter(old)


@needs_reference
def test_the_key_covers_every_input_it_must(model):
    x = torch.zeros(1, 6, 64)
    base = _key(model, x)
    assert _key(model, x) == base                                       # nothing changed
    assert _key(model, torch.zeros(2, 6, 64)) != base                     # a new B
    assert _key(model, torch.zeros(1, 6, 96)) != base                     # a new N
    assert _key(model, torch.zeros(1, 6, 64, dtype=torch.float64)) != base
    with torch.no_grad():
        model.cls_head.cls.weight.mul_(1.0)                              # an in-place update bumps the version
    k1 = _key(model, x)
    assert k1 != base
    lin = model.enc2[0].linear
    lin.weight = torch.nn.Parameter(lin.weight.detach().clone())           # a replaced parameter
    k2 = _key(model, x)
    assert k2 != k1
    bn = model.enc3[1].bn1
    bn.running_mean = bn.running_mean.clone()                              # a replaced buffer
    k3 = _key(model, x)
    assert k3 != k2
    bn.train(False)                                                        # one BatchNorm's mode
    assert _key(model, x) != k3
    bn.train(True)
    assert _key(model, x) == k3
    bn.momentum = 0.3                                                      # a hyperparameter the launches carry
    assert _key(model, x) != k3
    bn.momentum = 0.1
    assert _key(model, x) == k3

    def switch(name, undo):
        assert _key(model, x) != k3, name
        undo()
        assert _key(model, x) == k3, name

    switch("blocks_fused", _flip(blocks_fused.set_enabled, lambda: blocks_fused._enabled))
    switch("layer chain", _flip(pn2.set_pw_enabled, lambda: pn2._pw_enabled))
    switch("kNN grid", _flip(pointops.set_knn_grid, lambda: pointops._knn_grid_enabled))
    old = blocks_fused.BLOCK_FUSED_MAX_C
    blocks_fused.BLOCK_FUSED_MAX_C = 512
    switch("block width", lambda: setattr(blocks_fused, "BLOCK_FUSED_MAX_C", old))
    prev = L.load().tgn_pt_layer_set_cta_threshold(1 << 30)
    assert L.load().tgn_pt_layer_cta_threshold() == 1 << 30
    switch("pt_layer CTA threshold", lambda: L.load().tgn_pt_layer_set_cta_threshold(prev))
    forward = type(model.enc2[0]).forward                                   # a forward installed on a class of the tree
    type(model.enc2[0]).forward = lambda self, pxo: forward(self, pxo)
    switch("installed forward", lambda: setattr(type(model.enc2[0]), "forward", forward))


@needs_reference
def test_a_cpu_input_is_not_eligible(model):
    assert not graphs.eligible(model, 1, torch.device("cpu"))
    calls = []

    def previous(m, inputs):
        calls.append(inputs)
        return "previous"

    before = graphs.counters["eager"]
    with torch.no_grad():
        assert graphs.forward(model, previous, [torch.zeros(1, 6, 64)]) == "previous"
    assert graphs.counters["eager"] == before + 1 and len(calls) == 1
    assert graphs.graph_entries(model) == {}
