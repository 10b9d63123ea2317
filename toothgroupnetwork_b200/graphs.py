"""CUDA-graph replay of the point-transformer network's no-grad forward (``PointTransformerSeg.forward``,
models/modules/cbl_point_transformer/cbl_point_transformer_module.py:93-216).

With the fused layers, TransitionDowns, TransitionUps, heads and blocks of ``blocks_fused`` installed, a forward of tgnet's networks
is a few hundred launches whose Python, ctypes and launch overhead is about half its wall clock (DESIGN §3.7).
``accelerate(module)`` wraps the class's forward: an eligible call replays one CUDA graph of the whole forward, every other call
runs the class's previous forward.  Per module and per key (``graph_key``):

* the first call runs the forward eagerly (the warm-up: modules load, shared-memory attributes are set, weights are packed);
* the second captures it, then replays the graph once -- capture executes nothing, so every call advances the BatchNorm running
  statistics and ``num_batches_tracked`` exactly once, as an eager call does;
* later calls copy the input into the graph's static input, replay, and return clones of the outputs.

The key holds what the captured launches depend on: the input's shape, dtype and device, every module's training flag, each
BatchNorm's momentum and eps, the (data_ptr, _version) of every parameter, the data_ptr of every buffer, the forwards installed on
the model's classes and the library switches that select kernels.  A graph is only replayed under its own key; a small LRU per
module keeps the graphs of the last few keys (the crop batch's B varies with the tooth count), ``release_graphs()`` frees them.

Eligibility is decided before the warm-up, from the module tree and ``blocks_fused``'s predicates: no gradient is needed, there
are no targets, the input is CUDA float32, and every TransitionDown with stride != 1, every TransitionUp and the heads take their
fused paths, so no reference code that reads the offsets on the host runs.  The forward is restated here
(``_forward``) with the same submodule calls in the same order; it builds o0 on the device and runs under
``blocks_fused.equal_clouds()``, where the fused paths take their host sizes from the tensor shapes.  ``counters`` records
what each call did.
"""
from __future__ import annotations

import collections
import contextlib
import sys
import time
import weakref

import torch

from . import _lib as L
from . import blocks_fused as bf
from . import pointnet2_utils as pn2
from . import pointops

MAX_GRAPHS_PER_MODULE = 4
counters = collections.Counter()        # "eager" (not eligible), "warmup", "capture", "replay"
_graphs = weakref.WeakKeyDictionary()  # module -> OrderedDict(key -> _Entry)


class _Entry:
    """One key of one module: whether it is eligible and, once captured, the graph and every tensor its launches read or write
    that the graph's private pool does not own (the static input, the parameters and buffers)."""

    def __init__(self, eligible: bool):
        self.eligible = eligible
        self.graph = None
        self.static_in = None
        self.static_out = None
        self.keep = None
        self.capture_s = self.instantiate_s = 0.0


def _switches() -> tuple:
    return (bf._enabled, bf.BLOCK_FUSED_MAX_C, pn2._pw_enabled, pointops._knn_grid_enabled, pointops.KNN_GRID_MIN_POINTS,
            int(L.load().tgn_pt_layer_cta_threshold()), torch.get_float32_matmul_precision(), torch.backends.cudnn.enabled)


def graph_key(model, x: torch.Tensor):
    """-> (key, tensors): the key of a call of ``model`` on the (B, C, N) input x, and the parameters and buffers it covers."""
    parts = [tuple(x.shape), x.dtype, x.device]
    tensors = []
    classes = {}
    for m in model.modules():
        classes[type(m)] = type(m).forward
        parts.append(m.training)
        if isinstance(m, torch.nn.modules.batchnorm._BatchNorm):
            parts.append((m.momentum, m.eps, m.track_running_stats))
        for t in m._parameters.values():
            parts.append(None if t is None else (t.data_ptr(), t._version))
            if t is not None:
                tensors.append(t)
        for t in m._buffers.values():
            parts.append(None if t is None else t.data_ptr())
            if t is not None:
                tensors.append(t)
    parts.append(tuple((c.__module__, c.__qualname__, f) for c, f in classes.items()))
    parts.append(_switches())
    return tuple(parts), tensors


def _placeholder(c: int, dev, dtype=torch.float32) -> torch.Tensor:
    return torch.empty((0, c), dtype=dtype, device=dev)


def _fused(cls) -> bool:
    return bool(getattr(cls, "_tgn_fused", False))


def eligible(model, B: int, dev) -> bool:
    """The module-tree half of eligibility: ``blocks_fused``'s predicates on empty stand-ins of the widths each module reads
    (within ``equal_clouds``, as the graphed forward runs them), for every TransitionDown with stride != 1, every TransitionUp and
    the heads the forward calls.  The call-level half (no gradient, no targets, CUDA float32 input) is checked per call."""
    mod = sys.modules.get(type(model).__module__)
    tdc, tuc, mhc = (getattr(mod, n, None) for n in ("TransitionDown", "TransitionUp", "MultiHead"))
    if None in (tdc, tuc, mhc) or getattr(model, "block_num", None) not in (2, 3, 5):
        return False
    if not (isinstance(model.cls_head, mhc) and (B != 1 or isinstance(model.offset_head, mhc))):
        return False
    o = torch.empty((B,), dtype=torch.int32, device=dev)
    p = _placeholder(3, dev)
    with bf.equal_clouds():
        for m in model.modules():
            if isinstance(m, tdc) and m.stride != 1:
                if not (_fused(type(m)) and bf.transition_down_fusable(m, p, _placeholder(m.linear.in_features - 3, dev), o)):
                    return False
            elif isinstance(m, tuc):
                if not _fused(type(m)):
                    return False
                if len(m.linear2) == 2:                                  # head form (blocks.py:84-86)
                    ok = bf.transition_up_fusable(m, [p, _placeholder(m.linear1[0].out_features, dev), o])
                else:
                    ok = bf.transition_up_fusable(m, [p, _placeholder(m.linear1[0].in_features, dev), o],
                                                  [p, _placeholder(m.linear2[0].in_features, dev), o])
                if not ok:
                    return False
        for mh in (model.cls_head, model.offset_head) if B == 1 else (model.cls_head,):
            if not (_fused(type(mh)) and bf.multi_head_structure_ok(mh)):
                return False
            stages = {}
            for (n, i), func in zip(mh.ni_list, mh.infer_list):
                stages.setdefault(n, {})[i] = {"p_out": p, "f_out": _placeholder(func.infer[0].in_features, dev), "offset": o}
            stages.setdefault("up", {}).setdefault(0, {"p_out": p, "f_out": _placeholder(0, dev), "offset": o})
            if not bf.multi_head_fusable(mh, stages):
                return False
    return True


def _forward(model, x_in: torch.Tensor) -> list:
    """PointTransformerSeg.forward (:93-216) without targets, for block_num 5, 3 and 2: the same submodule calls in the same
    order, o0 made on the device, the same return list."""
    inputs = [x_in]
    B, C, N = x_in.shape
    pxo = x_in.permute(0, 2, 1)
    x0 = pxo.reshape(-1, C)
    p0 = pxo[:, :, :3].reshape(-1, 3).contiguous()
    o0 = torch.arange(1, B + 1, dtype=torch.int, device=x_in.device)
    o0 *= N
    stage_list = {"inputs": inputs}
    levels = model.block_num
    pxo = [[p0, x0, o0]]
    with bf.equal_clouds():
        for lvl in range(1, levels + 1):
            pxo.append(getattr(model, f"enc{lvl}")(pxo[-1]))
        stage_list["down"] = [{"p_out": p, "f_out": x, "offset": o} for p, x, o in pxo[1:]]
        dec = getattr(model, f"dec{levels}")
        p, x, o = pxo[levels]
        x = dec[1:]([p, dec[0]([p, x, o]), o])[1]                              # the head form: no upsampling
        pxo[levels] = [p, x, o]
        for lvl in range(levels - 1, 0, -1):
            dec = getattr(model, f"dec{lvl}")
            p, x, o = pxo[lvl]
            x = dec[1:]([p, dec[0]([p, x, o], pxo[lvl + 1]), o])[1]
            pxo[lvl] = [p, x, o]
        stage_list["up"] = [{"p_out": p, "f_out": x, "offset": o} for p, x, o in pxo[1:]]
        cls_results, stage_list = model.cls_head(stage_list)
        offset_results = model.offset_head(stage_list)[0] if B == 1 else None
    cls_results = cls_results.view(B, N, model.k).permute(0, 2, 1)
    if B == 1:
        offset_results = offset_results.view(B, N, 3).permute(0, 2, 1)
    return [cls_results, offset_results, None, pxo[1][1]]


@contextlib.contextmanager
def _capture_caches():
    """Run the capture against empty kNN / grid caches and chain maps and restore the previous ones afterwards; yields the maps
    the capture filled.  An entry made during capture holds graph-pool memory that only a replay writes, and an event recorded
    during capture, so eager code must never see it; a pre-capture entry would be read across the capture boundary (its event
    recorded outside the capture cannot be waited on inside it), so the capture does not see those either."""
    saved = (pointops._knn_cache, pointops._grid_cache, bf._td_chains, bf._tu_state, bf._mh_chains, bf._blk_chains)
    made = (pointops._Lru(saved[0].size), pointops._Lru(saved[1].size)) + tuple(weakref.WeakKeyDictionary() for _ in range(4))
    pointops._knn_cache, pointops._grid_cache, bf._td_chains, bf._tu_state, bf._mh_chains, bf._blk_chains = made
    try:
        yield made
    finally:
        pointops._knn_cache, pointops._grid_cache, bf._td_chains, bf._tu_state, bf._mh_chains, bf._blk_chains = saved


def _capture(e: _Entry, model, x: torch.Tensor, tensors: list) -> None:
    e.static_in = x.clone()
    g = torch.cuda.CUDAGraph(keep_graph=True)
    t0 = time.perf_counter()
    with _capture_caches() as made, torch.no_grad(), torch.cuda.graph(g):
        out = _forward(model, e.static_in)
    t1 = time.perf_counter()
    g.instantiate()
    e.capture_s, e.instantiate_s = t1 - t0, time.perf_counter() - t1
    # the parameters and buffers the launches read and update, and what the capture cached (graph-pool memory, kept with it)
    e.graph, e.static_out, e.keep = g, out, (tensors, made)


def _drop(lru, key) -> None:
    torch.cuda.synchronize()                 # no replay of the graph is still running when its pool and tensors go
    del lru[key]


def release_graphs(model=None) -> None:
    """Free the graphs of ``model`` (every module's when None)."""
    models = [model] if model is not None else list(_graphs.keys())
    for m in models:
        lru = _graphs.pop(m, None)
        if lru:
            torch.cuda.synchronize()
            lru.clear()


def graph_entries(model) -> dict:
    """key -> entry of ``model``'s graphs (for measurements and tests)"""
    return dict(_graphs.get(model, {}))


def forward(model, orig, inputs):
    x = inputs[0] if isinstance(inputs, (list, tuple)) and len(inputs) == 1 else None
    if not (isinstance(x, torch.Tensor) and x.is_cuda and x.dtype == torch.float32 and x.dim() == 3):
        counters["eager"] += 1
        return orig(model, inputs)
    key, tensors = graph_key(model, x)
    if torch.is_grad_enabled() and (x.requires_grad or any(t.requires_grad for t in tensors)):
        counters["eager"] += 1
        return orig(model, inputs)
    lru = _graphs.get(model)
    if lru is None:
        lru = _graphs[model] = collections.OrderedDict()
    e = lru.get(key)
    if e is None:
        e = lru[key] = _Entry(eligible(model, x.shape[0], x.device))
        while len(lru) > MAX_GRAPHS_PER_MODULE:
            _drop(lru, next(iter(lru)))
        if e.eligible:
            counters["warmup"] += 1
            with torch.no_grad():
                return _forward(model, x)
    lru.move_to_end(key)
    if not e.eligible:
        counters["eager"] += 1
        return orig(model, inputs)
    if e.graph is None:
        _capture(e, model, x, tensors)
        counters["capture"] += 1
    else:
        e.static_in.copy_(x)
        counters["replay"] += 1
    e.graph.replay()
    return [None if t is None else t.clone() for t in e.static_out]


def accelerate(cpm_module) -> None:
    """Wrap PointTransformerSeg.forward of an imported reference ``cbl_point_transformer_module``.  Idempotent."""
    cls = cpm_module.PointTransformerSeg
    if getattr(cls, "_tgn_graphs", False):
        return
    orig = cls.forward

    def seg_forward(self, inputs):
        return forward(self, orig, inputs)

    cls.forward, cls._tgn_graphs = seg_forward, True
