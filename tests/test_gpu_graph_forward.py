"""GPU: CUDA-graph replay of the point-transformer network's no-grad forward (toothgroupnetwork_b200/graphs.py) against the same
network run eagerly: outputs and BatchNorm buffers over eager, capture + replay and replay calls, at tgnet's first network (1 x 24 000
and the crop batch at two B) and the boundary network, in both BatchNorm modes; that a replay launches nothing itself and does not
synchronise; that every change the key covers leads to a warm-up and a new capture; routing of the calls that are not graphed."""
import pytest
import torch

from oracle import ref_models
from toothgroupnetwork_b200 import _lib as L
from toothgroupnetwork_b200 import blocks_fused, clouds, graphs

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not ref_models.available(), reason="reference snapshot not staged")]

FIRST = {"stride": [1, 4, 4, 4, 4], "nsample": [36, 24, 24, 24, 24], "blocks": [2, 3, 4, 6, 3], "block_num": 5,
         "planes": [32, 64, 128, 256, 512]}
BOUNDARY = {"stride": [1, 1], "nsample": [36, 24], "blocks": [2, 3], "block_num": 2, "planes": [16, 32]}
CPM = "models.modules.cbl_point_transformer.cbl_point_transformer_module"
BLOCKS, HEADS = "models.modules.cbl_point_transformer.blocks", "models.modules.cbl_point_transformer.heads"


def _world(decoder=True, graphed=True):
    w = ref_models.World("b200")                       # the fused layers and TransitionDowns are on in every world
    if decoder:
        blocks_fused.accelerate_decoder(w.mod(BLOCKS), w.mod(HEADS))
        blocks_fused.accelerate_blocks(w.mod(BLOCKS))
    if graphed:
        graphs.accelerate(w.mod(CPM))
    return w


@pytest.fixture(scope="module")
def worlds():
    return {"eager": _world(graphed=False), "graphed": _world()}


def _models(worlds, params, train, copies=("eager", "eager", "graphed")):
    torch.manual_seed(0)
    with worlds["eager"]:
        base = worlds["eager"].mod(CPM).get_model(c=6, k=17, **params)
    gen = torch.Generator().manual_seed(1)
    for m in base.modules():                           # running statistics away from 0 / 1, so that eval mode uses them
        if isinstance(m, torch.nn.BatchNorm1d):
            m.running_mean.copy_(torch.randn(m.running_mean.shape, generator=gen) * 0.1)
            m.running_var.copy_(torch.rand(m.running_var.shape, generator=gen) + 0.5)
    out = []
    for c in copies:
        with worlds[c]:
            m = worlds[c].mod(CPM).get_model(c=6, k=17, **params)
        m.load_state_dict(base.state_dict())
        out.append(m.cuda().train(train))
    return out


def _input(B, N, seed):
    p = torch.stack([clouds.dental_arch(N, seed + b)[0] for b in range(B)]).cuda()
    nrm = torch.nn.functional.normalize(torch.randn(p.shape, generator=torch.Generator().manual_seed(seed)), dim=-1).cuda()
    return torch.cat([p, nrm], -1).permute(0, 2, 1).contiguous()


def _call(world, model, x):
    with world, torch.no_grad():
        return model([x])


def _tensors(model, out):
    """the outputs (cls, offset, x1) and every BatchNorm buffer of model, by name"""
    t = {"cls_results": out[0], "offset_results": out[1], "x1": out[3]}
    t.update({k: v for k, v in model.state_dict().items() if "running_" in k or "num_batches" in k})
    return t


def _close(got, want, floor=0.05):
    got, want = got.double(), want.double()
    return float(((got - want).abs() / want.abs().clamp(min=floor * float(want.abs().max()))).max())


def _compare(graphed, eager, eager2=None):
    """bitwise where the two eager runs are bitwise equal (or everywhere, without a second eager run to compare); elsewhere
    within the fused path's bound.  Returns the names that needed the bound."""
    loose = []
    for k, want in eager.items():
        got = graphed[k]
        if want is None:
            assert got is None, k
            continue
        if eager2 is not None and not torch.equal(want, eager2[k]):
            loose.append(k)
            assert _close(got, want) < 1e-4, (k, _close(got, want))
        else:
            assert torch.equal(got, want), (k, _close(got, want))
    return loose


def _counts():
    return dict(graphs.counters)


def _delta(before, **want):
    now = _counts()
    got = {k: now.get(k, 0) - before.get(k, 0) for k in ("eager", "warmup", "capture", "replay")}
    assert got == {k: want.get(k, 0) for k in got}, got


CASES = {
    "first_1x24000": (FIRST, 1, 24000),
    "first_2x3072": (FIRST, 2, 3072),
    "first_5x3072": (FIRST, 5, 3072),
    "boundary_1x24000": (BOUNDARY, 1, 24000),
}


@pytest.mark.parametrize("case", list(CASES))
@pytest.mark.parametrize("train", [True, False], ids=["train_bn", "eval_bn"])
def test_graphed_calls_match_eager_calls(worlds, case, train):
    params, B, N = CASES[case]
    a1, a2, g = _models(worlds, params, train)
    loose = set()
    for step, want in enumerate(({"warmup": 1}, {"capture": 1}, {"replay": 1})):
        x = _input(B, N, 10 * step)
        before = _counts()
        got = _tensors(g, _call(worlds["graphed"], g, x))
        _delta(before, **want)
        e1 = _tensors(a1, _call(worlds["eager"], a1, x))
        e2 = _tensors(a2, _call(worlds["eager"], a2, x))
        loose |= set(_compare(got, e1, e2))
    # what the fused kernels' fp64 atomics leave unreproducible between two eager runs is reported, not hidden
    print(case, "train" if train else "eval", "within the bound:", sorted(loose))
    graphs.release_graphs(g)
    assert graphs.graph_entries(g) == {}


def test_replay_launches_nothing_and_does_not_synchronise(worlds):
    a, g = _models(worlds, BOUNDARY, True, copies=("eager", "graphed"))
    xs = [_input(2, 3072, s) for s in range(4)]
    for x in xs[:2]:
        _call(worlds["graphed"], g, x)
        _call(worlds["eager"], a, x)
    launches = L.launch_count()
    before = _counts()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = _call(worlds["graphed"], g, xs[2])
    finally:
        torch.cuda.set_sync_debug_mode(0)
    _delta(before, replay=1)
    assert L.launch_count() == launches
    _compare(_tensors(g, out), _tensors(a, _call(worlds["eager"], a, xs[2])))
    # no aliasing: the next call leaves this call's outputs as they were
    kept = [None if t is None else t.clone() for t in out]
    _call(worlds["graphed"], g, xs[3])
    assert all(k is None and t is None or torch.equal(k, t) for k, t in zip(kept, out))
    graphs.release_graphs()
    assert graphs.graph_entries(g) == {}


def _in_place(m):
    with torch.no_grad():
        m.cls_head.cls.weight.mul_(1.5)


def _replace(m):
    lin = m.enc2[0].linear
    lin.weight = torch.nn.Parameter(lin.weight.detach() * 0.75)


def _eval(m):
    m.eval()


CHANGES = {"in_place_weight": _in_place, "replaced_parameter": _replace, "train_to_eval": _eval}


@pytest.mark.parametrize("change", list(CHANGES) + ["new_B", "switch"])
def test_every_change_the_key_covers_warms_up_and_captures_again(worlds, change):
    a, g = _models(worlds, FIRST, True, copies=("eager", "graphed"))
    B = 2
    for s in range(3):
        _call(worlds["graphed"], g, _input(B, 3072, s))
        _call(worlds["eager"], a, _input(B, 3072, s))
    old_max_c = blocks_fused.BLOCK_FUSED_MAX_C
    if change in CHANGES:
        CHANGES[change](a)
        CHANGES[change](g)
    elif change == "new_B":
        B = 3
    else:
        blocks_fused.BLOCK_FUSED_MAX_C = 512                 # every block on the fused path
    try:
        for s, want in enumerate(({"warmup": 1}, {"capture": 1}, {"replay": 1})):
            x = _input(B, 3072, 20 + s)
            before = _counts()
            got = _tensors(g, _call(worlds["graphed"], g, x))
            _delta(before, **want)
            eager = _tensors(a, _call(worlds["eager"], a, x))
            for k, v in eager.items():
                assert (v is None and got[k] is None) or torch.equal(got[k], v) or _close(got[k], v) < 1e-4, (change, s, k)
    finally:
        blocks_fused.BLOCK_FUSED_MAX_C = old_max_c
        graphs.release_graphs()


def test_calls_that_are_not_graphed_run_the_previous_forward(worlds):
    (g,) = _models(worlds, BOUNDARY, True, copies=("graphed",))
    x = _input(1, 4096, 3)
    before = _counts()
    with worlds["graphed"]:
        out = g([x])                                          # autograd on: the parameters need gradients
    assert out[0].requires_grad
    _delta(before, eager=1)
    calls = []

    def previous(model, inputs):
        calls.append(len(inputs))
        return "previous"

    before = _counts()
    target = torch.zeros(1, 1, 4096, device="cuda")
    with torch.no_grad():
        assert graphs.forward(g, previous, [x, target]) == "previous"           # targets: the loss needs them
    _delta(before, eager=1)
    assert calls == [2]
    no_decoder = _world(decoder=False)
    (h,) = _models({"graphed": no_decoder, "eager": worlds["eager"]}, BOUNDARY, True, copies=("graphed",))
    before = _counts()
    for s in range(3):
        _call(no_decoder, h, _input(1, 4096, s))             # TransitionUp and the heads on the reference's code
    _delta(before, eager=3)
    assert all(not e.eligible and e.graph is None for e in graphs.graph_entries(h).values())
    graphs.release_graphs()
