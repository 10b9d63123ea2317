"""CPU-side checks (no GPU): the C-ABI library loads and exports every symbol the header
declares, the host logic (BN folding, drop-in shim, sharding) is right, and the product path
refuses to run without CUDA instead of falling back."""
import ctypes
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def built_lib():
    from toothgroupnetwork_b200 import build
    return build.build()


def test_library_exports_every_symbol_of_the_header(built_lib):
    header = open(os.path.join(ROOT, "include", "tgn_b200.h")).read()
    declared = set(re.findall(r"\b(tgn_\w+|\w+_cuda_launcher)\s*\(", header))
    assert len(declared) >= 29
    lib = ctypes.CDLL(built_lib)
    missing = [s for s in sorted(declared) if not hasattr(lib, s)]
    assert not missing, missing
    from toothgroupnetwork_b200 import _lib
    assert set(_lib.EXPORTS) <= declared | {"tgn_version", "tgn_last_error", "tgn_launch_count"}
    assert _lib.load().tgn_version() >= 100


def test_reference_launcher_names_are_exactly_the_references(built_lib):
    """The ten extern "C" names of pointops/src/*/*_cuda_kernel.h."""
    from toothgroupnetwork_b200 import _lib
    want = {"furthestsampling", "knnquery", "grouping_forward", "grouping_backward", "interpolation_forward",
            "interpolation_backward", "subtraction_forward", "subtraction_backward", "aggregation_forward", "aggregation_backward"}
    assert {n.replace("_cuda_launcher", "") for n in _lib.REFERENCE_LAUNCHERS} == want


def test_library_contains_hopper_instructions(built_lib):
    """SASS evidence: warpgroup MMA (HGMMA), the bulk (TMA) copy of the layer kernel's weights (UBLKCP), mbarrier
    (SYNCS), and an sm_90a image."""
    try:
        sass = subprocess.run(["cuobjdump", "-sass", built_lib], capture_output=True, text=True, timeout=300).stdout
    except (FileNotFoundError, subprocess.TimeoutExpired):
        pytest.skip("cuobjdump unavailable")
    for mnemonic in ("HGMMA", "UBLKCP", "SYNCS"):
        assert mnemonic in sass, mnemonic
    assert "arch = sm_90a" in sass


def test_no_cpu_fallback():
    from toothgroupnetwork_b200 import _lib, pointops
    from toothgroupnetwork_b200 import pointnet2_utils as pn2
    with pytest.raises(_lib.TgnError):
        pointops.fps_packed(torch.rand(10, 3), torch.tensor([10], dtype=torch.int32), torch.tensor([2], dtype=torch.int32), 10, 2)
    with pytest.raises(_lib.TgnError):
        pn2.query_ball_point(0.1, 4, torch.rand(1, 10, 3), torch.rand(1, 2, 3))
    sa = pn2.PointNetSetAbstraction(4, 0.1, 4, 9, [8], False).eval()
    with pytest.raises(_lib.TgnError):
        sa(torch.rand(1, 3, 16), torch.rand(1, 6, 16))


def test_product_never_imports_the_oracle():
    pkg = os.path.join(ROOT, "toothgroupnetwork_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                text = open(os.path.join(dirpath, f)).read()
                assert "import oracle" not in text and "from oracle" not in text and "liboracle" not in text, f


def test_bn_folding_equals_conv_bn_eval():
    from toothgroupnetwork_b200.pointnet2_utils import _FoldedMlp
    torch.manual_seed(0)
    convs = nn.ModuleList([nn.Conv2d(9, 16, 1), nn.Conv2d(16, 24, 1)])
    bns = nn.ModuleList([nn.BatchNorm2d(16), nn.BatchNorm2d(24)])
    for b in bns:
        b.running_mean.normal_(0, 0.3)
        b.running_var.uniform_(0.5, 1.5)
        b.weight.data.uniform_(0.5, 1.5)
        b.bias.data.normal_(0, 0.2)
    f = _FoldedMlp().update(convs, bns)
    assert f.channels == [9, 16, 24]
    x = torch.randn(2, 9, 5, 7)
    h = x
    convs.eval(); bns.eval()
    for c, b in zip(convs, bns):
        h = torch.relu(b(c(h)))
    g = x
    for w, bias in zip(f.weights, f.biases):
        g = torch.relu(torch.einsum("oc,bckn->bokn", w, g) + bias.view(1, -1, 1, 1))
    assert torch.allclose(g, h, rtol=1e-5, atol=1e-5)
    key = f.key
    assert f.update(convs, bns).key == key                # cached
    bns[0].running_mean.add_(1.0)
    assert f.update(convs, bns).key != key                # invalidated by the version counter


def test_dropin_shim_resolves_reference_import_paths():
    import toothgroupnetwork_b200.dropin as dropin
    dropin.install()
    try:
        from external_libs.pointops.functions import pointops as p1
        from external_libs.pointnet2_utils.pointnet2_utils import (PointNetFeaturePropagation, PointNetSetAbstraction,  # noqa: F401
                                                                   PointNetSetAbstractionMsg, farthest_point_sample,
                                                                   index_points, query_ball_point, sample_and_group,
                                                                   sample_and_group_all, square_distance)
        import pointops_cuda
        for name in ("FurthestSampling", "furthestsampling", "KNNQuery", "knnquery", "Grouping", "grouping", "queryandgroup",
                     "Subtraction", "subtraction", "Aggregation", "aggregation", "interpolation", "Interpolation", "interpolation2"):
            assert hasattr(p1, name), name
        for name in ("knnquery_cuda", "furthestsampling_cuda", "grouping_forward_cuda", "grouping_backward_cuda",
                     "interpolation_forward_cuda", "interpolation_backward_cuda", "subtraction_forward_cuda",
                     "subtraction_backward_cuda", "aggregation_forward_cuda", "aggregation_backward_cuda"):
            assert hasattr(pointops_cuda, name), name
    finally:
        dropin.uninstall()


def test_dropin_serves_the_reference_real_model_files():
    """The reference's unmodified models/modules/*.py import and CONSTRUCT on this package through dropin.install()
    (parameter counts of SURVEY.md 8c), with this package's classes inside; needs the reference checkout or its staged archive."""
    import pytest
    import torch
    from oracle import ref_models
    if not ref_models.available():
        pytest.skip("reference snapshot not staged")
    w = ref_models.World("b200")
    count = lambda m: sum(q.numel() for q in m.parameters())
    with w:
        pp = w.mod("models.modules.pointnet_pp").get_model()
        assert count(pp) == 8957689 and type(pp.sa1).__module__ == "toothgroupnetwork_b200.pointnet2_utils"
        assert type(pp.fp1).__module__ == "toothgroupnetwork_b200.pointnet2_utils"
        assert count(w.mod("models.modules.tsg_centroid_module").get_model()) == 832660
        seg = w.mod("models.modules.tsg_seg_module").get_model()
        assert count(seg) == 1542325 and seg.flatten_sa.group_all
        blocks = w.mod("models.modules.cbl_point_transformer.blocks")
        assert blocks.pointops.__name__ == "toothgroupnetwork_b200.pointops"
        saved = torch.nn.Module.cuda
        torch.nn.Module.cuda = lambda self, *a, **k: self           # grouping_network_module.py:15 calls .cuda() in __init__
        try:
            g = w.mod("models.modules.grouping_network_module").GroupingNetworkModule(
                {"model_parameter": {"input_feat": 6, "stride": [1, 4, 4, 4, 4], "nsample": [36, 24, 24, 24, 24], "blocks": [2, 3, 4, 6, 3],
                                     "block_num": 5, "planes": [32, 64, 128, 256, 512], "crop_sample_size": 3072}})
        finally:
            torch.nn.Module.cuda = saved
        assert count(g) == 15729246
        # the crop search of ops_utils is served by the GPU version too
        assert w.mod("ops_utils").get_nearest_neighbor_idx.__module__ == "toothgroupnetwork_b200.crops"
        # ... and so are the clustering between the stages and the no-grad forwards of the transformer blocks
        assert w.mod("ops_utils").get_clustering_labels.__module__ == "toothgroupnetwork_b200.clustering"
        assert blocks.PointTransformerLayer._tgn_fused and blocks.PointTransformerLayer.forward.__name__ == "ptl_forward"
        assert blocks.TransitionDown.forward.__name__ == "td_forward"
    # state_dict keys are the reference's (checkpoints load unchanged)
    ref = ref_models.World("reference", cpu_dry_run=True)
    with ref:
        want = set(ref.mod("models.modules.pointnet_pp").get_model().state_dict().keys())
    assert set(pp.state_dict().keys()) == want


def test_fused_blocks_step_aside_without_a_gpu_or_under_autograd():
    """blocks_fused only takes CUDA fp32 inputs of supported shapes when no gradient is needed; everything else is the reference's code."""
    import torch
    import torch.nn as nn
    from toothgroupnetwork_b200 import blocks_fused

    class Layer(nn.Module):                                           # attribute layout of blocks.PointTransformerLayer (:15-29)
        def __init__(self, c, share=8):
            super().__init__()
            self.mid_planes = self.out_planes = c
            self.share_planes, self.nsample = share, 16
            self.linear_q = nn.Linear(c, c)
            self.linear_p = nn.Sequential(nn.Linear(3, 3), nn.BatchNorm1d(3), nn.ReLU(), nn.Linear(3, c))
            self.linear_w = nn.Sequential(nn.BatchNorm1d(c), nn.ReLU(), nn.Linear(c, c // share), nn.BatchNorm1d(c // share), nn.ReLU(),
                                          nn.Linear(c // share, c // share))

    p, x, o = torch.randn(50, 3), torch.randn(50, 32), torch.tensor([50], dtype=torch.int32)
    with torch.no_grad():
        assert not blocks_fused.pt_layer_fusable(Layer(32), p, x, o)                      # CPU tensors
    td = nn.Module()
    td.stride, td.nsample, td.linear, td.bn = 4, 16, nn.Linear(35, 64, bias=False), nn.BatchNorm1d(64)
    with torch.no_grad():
        assert not blocks_fused.transition_down_fusable(td, p, x, o)
    assert blocks_fused._needs_grad(Layer(32), p, x) and not blocks_fused._needs_grad(Layer(32).requires_grad_(False), p, x)
    bn = nn.BatchNorm1d(4, momentum=None)                              # cumulative moving average: not a shape the kernels update
    assert not blocks_fused._bn_ok(bn) and blocks_fused._bn_ok(nn.BatchNorm1d(4)) and blocks_fused._bn_mode(nn.BatchNorm1d(4).eval()) == 2


def test_square_distance_matches_oracle_bitwise_on_cpu():
    from oracle import oracle
    from toothgroupnetwork_b200 import clouds
    from toothgroupnetwork_b200.pointnet2_utils import square_distance
    a, b = clouds.cube(64, 1)[None], clouds.cube(200, 2)[None]
    assert np.array_equal(square_distance(a, b).numpy().view(np.uint32), oracle.square_distance(a.numpy(), b.numpy()).view(np.uint32))


def test_cloud_generators_are_deterministic():
    from toothgroupnetwork_b200 import clouds
    a, b = clouds.dental_arch(1000, 5), clouds.dental_arch(1000, 5)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]) and torch.equal(a[2], b[2])
    assert not torch.equal(a[0], clouds.dental_arch(1000, 6)[0])
    assert clouds.arch_features(100, 1).shape == (1, 6, 100)
    assert set(a[2].unique().tolist()) <= set(range(-1, 16))
    assert clouds.cloud_seed(3, 7) == 3007


def test_sharding_single_process_helpers():
    from toothgroupnetwork_b200 import sharding
    assert sharding.owned(10, 1, 4) == [1, 5, 9]
    assert sorted(sum((sharding.owned(11, r, 3) for r in range(3)), [])) == list(range(11))
    recs = sharding.gather_metrics({"sampled_points": 5, "clouds": 1, "seconds": 2.0, "parity_ok": 1, "launches": 3}, torch.device("cpu"))
    agg = sharding.reduce_metrics(recs)
    assert agg["sampled_points"] == 5 and agg["seconds"] == 2.0 and agg["parity_ok"] == 1.0


_WORKER = r"""
import os, sys, json
sys.path.insert(0, {root!r})
import torch
from toothgroupnetwork_b200 import sharding
rank, world, local = sharding.init("gloo")
mine = sharding.owned(7, rank, world)
sharding.barrier()
t = sharding.max_over_ranks(1.0 + rank, torch.device("cpu"))
recs = sharding.gather_metrics({{"sampled_points": 1024 * len(mine), "clouds": len(mine), "seconds": 1.0 + rank,
                                 "parity_ok": 1.0, "launches": 3 * len(mine)}}, torch.device("cpu"))
agg = sharding.reduce_metrics(recs)
if rank == 0:
    print(json.dumps({{"t": t, "agg": agg, "n": len(recs)}}))
"""


def test_sharding_world_size_2_gloo(tmp_path):
    script = tmp_path / "worker.py"
    script.write_text(_WORKER.format(root=ROOT))
    env = dict(os.environ, MASTER_ADDR="127.0.0.1")
    res = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr",
                          "127.0.0.1", "--master-port", "29577", str(script)], capture_output=True, text=True, env=env, timeout=240)
    assert res.returncode == 0, res.stderr[-2000:]
    import json
    line = [l for l in res.stdout.splitlines() if l.startswith("{")][-1]
    out = json.loads(line)
    assert out["n"] == 2 and out["t"] == 2.0
    assert out["agg"]["clouds"] == 7 and out["agg"]["sampled_points"] == 7 * 1024 and out["agg"]["seconds"] == 2.0


def test_bench_reference_arm_prints_contract_line():
    import json
    res = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--steps", "1", "--warmup", "0",
                          "--cpu-clouds", "2"], capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stderr[-2000:]
    line = json.loads(res.stdout.strip().splitlines()[-1])
    for key in ("impl", "metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "config",
                "cpu_baseline", "e2e"):
        assert key in line, key
    assert line["impl"] == "reference" and line["cpu_baseline"]["kind"] == "port" and line["value"] > 0


def test_host_pipeline_plan_covers_every_cloud_once():
    """Chunk spans and compute groups of HostPipeline (pure host logic): contiguous, complete, ordered."""
    from toothgroupnetwork_b200.pipeline import HostPipeline

    class Shape:
        pass

    for chunk, groups, B in [(148, (1,), 1184), (148, (2, 3, 2, 1), 1184), (148, (2, 3, 2, 1), 148 * 11 + 5),
                             (64, (2, 5, 1), 100), (296, (1,), 10), (148, (2, 2), 1)]:
        f = Shape()
        f.chunk, f.groups = chunk, groups
        spans, plan = HostPipeline._plan(f, B)
        assert spans[0][0] == 0 and spans[-1][1] == B
        assert all(a[1] == b[0] for a, b in zip(spans, spans[1:]))
        assert all(0 < hi - lo <= chunk for lo, hi in spans)
        assert plan[0][0] == 0 and plan[-1][1] == len(spans) - 1
        assert all(a[1] + 1 == b[0] for a, b in zip(plan, plan[1:]))
        assert all(k0 <= k1 for k0, k1 in plan)
