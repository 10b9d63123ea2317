#!/usr/bin/env python
"""Operator-level timings on one GPU: this library beside the REFERENCE's own GPU path
(verbatim ``pointops`` kernels from ``oracle/_ref`` + the reference's torch ``pointnet2_utils.py``),
CUDA events on the launching stream, warm-up, median of ``reps``  (BASELINE.md 3: C1(a)/C2 "GPU
reference"; VERDICT r1 items 3, 5(ii), 7).

    python scripts/op_bench.py [--out gpurun_out/op_bench.json] [--sections fps,knn,ball,sa,fp]

Also importable: ``bench.py`` calls ``fps_latency_table`` / ``ref_gpu_step`` for its ``latency_ms`` and
``ref_gpu`` entries.  Test infrastructure side: the reference legs import ``oracle/``.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import warnings

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
warnings.filterwarnings("ignore")


def time_ms(fn, warm=2, reps=5):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return float(np.median(ts))


def arch_batch(B, N, distinct=8):
    from toothgroupnetwork_b200 import clouds
    base = [clouds.arch_features(N, s)[0] for s in range(min(B, distinct))]
    return torch.stack([base[j % len(base)] for j in range(B)]).contiguous().cuda()      # (B,6,N)


def ref_available():
    from oracle import ref_cuda
    return ref_cuda.available()


def ref_models_available():
    from oracle import ref_models
    return ref_models.available()


def c1_parity():
    """BASELINE configs[0]: FPS 24000->4096 on one synthetic random (cube) cloud: indices against the CPU oracle and,
    when present, the verbatim reference kernel (bitwise)."""
    from oracle import oracle
    from toothgroupnetwork_b200 import clouds, pointops
    xyz = clouds.cube(24000, 0)
    off, noff = np.array([24000], np.int32), np.array([4096], np.int32)
    want = oracle.furthestsampling(xyz.numpy(), off, noff)
    x = xyz.cuda()
    o, no = torch.from_numpy(off).cuda(), torch.from_numpy(noff).cuda()
    got = pointops.fps_packed(x, o, no, 24000, 4096)
    res = {"cube_idx_bitwise_vs_oracle": bool(np.array_equal(got.cpu().numpy(), want)), "cube_ours_ms": time_ms(lambda: pointops.fps_packed(x, o, no, 24000, 4096))}
    if ref_available():
        from oracle import ref_cuda
        ridx, _ = ref_cuda.furthestsampling(x, o, no, 24000, 4096)
        res["cube_idx_bitwise_vs_reference_kernel"] = bool(torch.equal(ridx, got))
        res["cube_ref_kernel_ms"] = time_ms(lambda: ref_cuda.furthestsampling(x, o, no, 24000, 4096), warm=1, reps=3)
    return res


# ------------------------------------------------------------------------------------------ FPS
def fps_latency_table(batches=(1, 16, 132, 1056), npoints=(1024, 4096), N=24000, with_ref=True, ref_max_batch=132):
    """ms per call of FPS N->M over a batch of B clouds: ours (auto shape) and the verbatim reference kernel."""
    from toothgroupnetwork_b200 import pointops
    rows = []
    for B in batches:
        feats = arch_batch(B, N)
        xyz = feats[:, :3].permute(0, 2, 1).contiguous().view(-1, 3)
        off = (torch.arange(1, B + 1, dtype=torch.int32) * N).cuda()
        for M in npoints:
            noff = (torch.arange(1, B + 1, dtype=torch.int32) * M).cuda()
            ours = time_ms(lambda: pointops.fps_packed(xyz, off, noff, N, B * M))
            row = {"clouds": B, "n": N, "m": M, "ours_ms": ours, "ours_us_per_iteration": ours * 1e3 / (M - 1)}
            if with_ref and ref_available() and B <= ref_max_batch:
                from oracle import ref_cuda
                ref = time_ms(lambda: ref_cuda.furthestsampling(xyz, off, noff, N, B * M), warm=1, reps=3)
                row.update({"ref_kernel_ms": ref, "speedup": ref / ours})
            rows.append(row)
        del feats, xyz
    return rows


# ------------------------------------------------------------------------------------------ kNN
KNN_MIX = [  # (label, n_src, m_query, k)   tgnet_fps net 1 launch mix (blocks.py:34-35,69-71, heads.py:44-51)
    ("enc1 self 24k x 24k k=36", 24000, 24000, 36),
    ("down 6000 <- 24000 k=24", 24000, 6000, 24),
    ("enc2 self 6000 k=24", 6000, 6000, 24),
    ("enc3 self 1500 k=24", 1500, 1500, 24),
    ("up 24000 <- 6000 k=3", 6000, 24000, 3),
    ("head 24000 <- 6000 k=1", 6000, 24000, 1),
    ("head 24000 <- 93 k=1", 93, 24000, 1),
]


def knn_table(with_ref=True):
    from toothgroupnetwork_b200 import clouds, pointops
    xyz_full = clouds.dental_arch(24000, 0)[0].cuda()
    rows = []
    for label, n, m, k in KNN_MIX:
        src = xyz_full[torch.linspace(0, 23999, n).long()].contiguous()
        qry = xyz_full[torch.linspace(0, 23999, m).long()].contiguous()
        o = torch.tensor([n], dtype=torch.int32).cuda()
        no = torch.tensor([m], dtype=torch.int32).cuda()
        def cold():                       # grid build (4 kernels) + query: what the first search against a point set costs
            pointops.clear_knn_caches()
            return pointops.knn_packed(k, src, qry, o, no)

        def warm():                       # grid cached (every later search against the same points), answer NOT cached
            pointops._knn_cache.clear()
            return pointops.knn_packed(k, src, qry, o, no)

        def brute():
            pointops.set_knn_grid(False)
            try:
                return pointops.knn_packed(k, src, qry, o, no)
            finally:
                pointops.set_knn_grid(True)

        ours = time_ms(cold)
        row = {"case": label, "n": n, "m": m, "k": k, "ours_ms": ours, "ours_grid_cached_ms": time_ms(warm), "ours_bruteforce_kernel_ms": time_ms(brute),
               "ours_repeated_identical_query_ms": time_ms(lambda: pointops.knn_packed(k, src, qry, o, no)), "pair_evals": n * m,
               "path": "grid" if n >= pointops.KNN_GRID_MIN_POINTS else "brute force"}
        if with_ref and ref_available():
            from oracle import ref_cuda
            ref = time_ms(lambda: ref_cuda.knnquery(k, src, qry, o, no), warm=1, reps=3)
            a = cold()
            b = ref_cuda.knnquery(k, src, qry, o, no)
            row.update({"ref_kernel_ms": ref, "speedup": ref / ours,
                        "bitwise_idx": bool(torch.equal(a[0], b[0])), "bitwise_d2": bool(torch.equal(a[1], b[1]))})
        rows.append(row)
    return rows


# ------------------------------------------------------------------------------------------ reference torch path
_ref_world = None


def ref_world():
    global _ref_world
    if _ref_world is None:
        from oracle import ref_models
        _ref_world = ref_models.World("reference")
    return _ref_world


def ball_table(with_ref=True):
    from toothgroupnetwork_b200 import pointnet2_utils as pn2
    rows = []
    for B in (1, 16):
        feats = arch_batch(B, 24000)
        xyz_t = feats[:, :3].permute(0, 2, 1).contiguous()
        new_xyz = pn2._take_rows(xyz_t.view(-1, 3), pn2._fps_batched(xyz_t, 1024)).view(B, 1024, 3)
        for r, K in ((0.025, 32), (0.05, 64), (0.1, 32), (0.2, 64)):
            ours = time_ms(lambda: pn2._ball_query(r, K, xyz_t, new_xyz, True))
            row = {"clouds": B, "radius": r, "K": K, "ours_ms": ours}
            if with_ref:
                w = ref_world()
                with w:
                    refpn = w.mod("external_libs.pointnet2_utils.pointnet2_utils")
                    ref = time_ms(lambda: refpn.query_ball_point(r, K, xyz_t, new_xyz), warm=1, reps=3)
                    same = bool(torch.equal(refpn.query_ball_point(r, K, xyz_t, new_xyz), pn2.query_ball_point(r, K, xyz_t, new_xyz)))
                row.update({"ref_torch_ms": ref, "speedup": ref / ours, "bitwise": same})
            rows.append(row)
    return rows


def _copy_sa(src, dst):
    dst.load_state_dict(src.state_dict())
    return dst


def ref_gpu_step(B=16, train_bn=False, reps=5):
    """The BASELINE C2(i) step, ``PointNetSetAbstraction(1024, 0.1, 32, 9, [32,32,64])`` forward on B 24k clouds,
    through the REFERENCE's own GPU path: verbatim FPS kernel + torch query_ball_point / index_points /
    Conv2d+BN+ReLU / max (``pointnet2_utils.py:213-239``), IEEE fp32 convolutions.  Returns ms and sampled points/s."""
    from toothgroupnetwork_b200 import pointnet2_utils as pn2
    feats = arch_batch(B, 24000)
    xyz = feats[:, :3].contiguous()
    torch.manual_seed(0)
    ours = pn2.PointNetSetAbstraction(1024, 0.1, 32, 9, [32, 32, 64], False).cuda().train(train_bn)
    w = ref_world()
    with w, torch.no_grad():
        refpn = w.mod("external_libs.pointnet2_utils.pointnet2_utils")
        ref = _copy_sa(ours, refpn.PointNetSetAbstraction(1024, 0.1, 32, 9, [32, 32, 64], False).cuda()).train(train_bn)
        saved = torch.backends.cudnn.allow_tf32
        torch.backends.cudnn.allow_tf32 = False
        try:
            ref_ms = time_ms(lambda: ref(xyz, feats), warm=1, reps=reps)
            want = ref(xyz, feats)
        finally:
            torch.backends.cudnn.allow_tf32 = saved
    with torch.no_grad():
        ours_ms = time_ms(lambda: ours(xyz, feats), warm=2, reps=reps)
        got = ours(xyz, feats)
    rel = float(((got[1] - want[1]).abs() / want[1].abs().clamp(min=0.05 * float(want[1].abs().max()))).max())
    return {"clouds": B, "bn": "train" if train_bn else "eval", "ref_gpu_ms": ref_ms, "ours_ms": ours_ms,
            "ref_gpu_sampled_points_per_s": B * 1024 / ref_ms * 1e3, "ours_sampled_points_per_s": B * 1024 / ours_ms * 1e3,
            "speedup": ref_ms / ours_ms, "new_xyz_bitwise": bool(torch.equal(got[0], want[0])), "max_rel_elementwise": rel}


def fp_table(with_ref=True):
    """PointNetFeaturePropagation fp1 of tsg_centroid_module (24000 <- 1024, 134 -> 64 -> 32), train and eval BN."""
    from toothgroupnetwork_b200 import pointnet2_utils as pn2
    rows = []
    feats = arch_batch(1, 24000)
    xyz1 = feats[:, :3].contiguous()
    xyz_t = xyz1.permute(0, 2, 1).contiguous()
    sel = pn2.farthest_point_sample(xyz_t, 1024)
    xyz2 = pn2.index_points(xyz_t, sel).permute(0, 2, 1).contiguous()
    g = torch.Generator(device="cuda").manual_seed(5)
    p2 = torch.randn(1, 128, 1024, device="cuda", generator=g)
    for train_bn in (True, False):
        torch.manual_seed(0)
        ours = pn2.PointNetFeaturePropagation(134, [64, 32]).cuda().train(train_bn)
        with torch.no_grad():
            ours_ms = time_ms(lambda: ours(xyz1, xyz2, feats, p2))
            got = ours(xyz1, xyz2, feats, p2)
        row = {"bn": "train" if train_bn else "eval", "ours_ms": ours_ms}
        if with_ref:
            w = ref_world()
            with w, torch.no_grad():
                refpn = w.mod("external_libs.pointnet2_utils.pointnet2_utils")
                ref = _copy_sa(ours, refpn.PointNetFeaturePropagation(134, [64, 32]).cuda()).train(train_bn)
                saved = torch.backends.cudnn.allow_tf32
                torch.backends.cudnn.allow_tf32 = False
                try:
                    ref_ms = time_ms(lambda: ref(xyz1, xyz2, feats, p2), warm=1, reps=3)
                    want = ref(xyz1, xyz2, feats, p2)
                finally:
                    torch.backends.cudnn.allow_tf32 = saved
            rel = float(((got - want).abs() / want.abs().clamp(min=0.05 * float(want.abs().max()))).max())
            row.update({"ref_torch_ms": ref_ms, "speedup": ref_ms / ours_ms, "max_rel_elementwise": rel})
        rows.append(row)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "gpurun_out", "op_bench.json"))
    ap.add_argument("--sections", default="fps,knn,ball,sa,fp")
    ap.add_argument("--no-ref", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available()
    with_ref = not args.no_ref
    rep = {"device": torch.cuda.get_device_name(0), "timing": "CUDA events, median, warm-up 1-2"}
    sec = args.sections.split(",")
    if "fps" in sec:
        rep["fps_latency"] = fps_latency_table(with_ref=with_ref)
    if "knn" in sec:
        rep["knn"] = knn_table(with_ref=with_ref)
    if "ball" in sec:
        rep["ball_query"] = ball_table(with_ref=with_ref)
    if "sa" in sec:
        rep["sa1_c2i_step"] = [ref_gpu_step(B, bn) for B in (1, 16) for bn in (False, True)]
    if "fp" in sec:
        rep["feature_propagation_fp1"] = fp_table(with_ref=with_ref)
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(rep, f, indent=1)
    print(json.dumps(rep, indent=1))


if __name__ == "__main__":
    main()


# ------------------------------------------------------------------------------------------ SURVEY 8(f) rows
def raw_mesh_fps(n=100000, m=24000):
    """8(f)-2: one raw mesh of n vertices -> m samples (gen_utils.py:135-140), beside the verbatim reference kernel, bitwise."""
    from toothgroupnetwork_b200 import clouds, pointops
    xyz = clouds.dental_arch(n, 7)[0].cuda().contiguous()
    off, noff = torch.tensor([n], dtype=torch.int32).cuda(), torch.tensor([m], dtype=torch.int32).cuda()
    got = pointops.fps_packed(xyz, off, noff, n, m)
    row = {"n": n, "m": m, "ours_ms": time_ms(lambda: pointops.fps_packed(xyz, off, noff, n, m), warm=1, reps=3)}
    if ref_available():
        from oracle import ref_cuda
        ridx, _ = ref_cuda.furthestsampling(xyz, off, noff, n, m)
        row["idx_bitwise_vs_reference_kernel"] = bool(torch.equal(ridx, got))
        row["ref_kernel_ms"] = time_ms(lambda: ref_cuda.furthestsampling(xyz, off, noff, n, m), warm=0, reps=2)
        row["speedup"] = row["ref_kernel_ms"] / row["ours_ms"]
    return row


def dbscan_row(pull=0.9, jitter=0.004, n=24000):
    """8(f)-4: DBSCAN(eps=0.03, min_samples=30) of ops_utils.get_clustering_labels (:98) on offset-moved foreground points:
    scikit-learn on the host (what the reference runs) beside csrc/dbscan.cu; labels and core samples compared."""
    import time
    from toothgroupnetwork_b200 import clouds, clustering
    xyz, _, label = clouds.dental_arch(n, 0)
    xyz, label = xyz.numpy(), np.where(label.numpy() < 0, 0, label.numpy()).astype(np.int64)
    cent = np.stack([xyz[label == c].mean(0) if (label == c).any() else np.zeros(3, np.float32) for c in range(int(label.max()) + 1)])
    fg = (xyz + pull * (cent[label] - xyz) + np.random.default_rng(0).normal(0, jitter, xyz.shape)).astype(np.float32)[label != 0]
    dev = torch.as_tensor(fg).cuda()
    lab, core = clustering.dbscan(fg)
    row = {"points": int(len(fg)), "pull": pull, "device_ms_resident": time_ms(lambda: clustering.dbscan_device(dev)),
           "device_ms_numpy_in_out": time_ms(lambda: clustering.dbscan(fg))}
    try:
        from sklearn.cluster import DBSCAN
        t = time.perf_counter()
        ref = DBSCAN(eps=0.03, min_samples=30).fit(fg)
        row["sklearn_host_ms"] = (time.perf_counter() - t) * 1e3
        row["labels_equal"] = bool(np.array_equal(lab, ref.labels_) and np.array_equal(core, ref.core_sample_indices_))
        row["speedup"] = row["sklearn_host_ms"] / row["device_ms_numpy_in_out"]
    except ImportError:
        row["sklearn_host_ms"] = None
    return row


def tgnet_nograd_row(points=24000):
    """8(f)-3 in context: GroupingNetworkModule (tgnet_fps) forward under no_grad on the reference's unmodified model files: reference
    operators / this package with the reference's block code / this package with the fused blocks, train-mode BatchNorm."""
    import model_parity as mp
    from oracle import ref_models
    from toothgroupnetwork_b200 import blocks_fused
    feats, labels = mp.make_inputs(points)
    ms, outs, state = {}, {}, None
    for ops in ("reference", "b200"):
        w = ref_models.World(ops)
        with w, torch.no_grad():
            torch.manual_seed(0)
            module = w.mod("models.modules.grouping_network_module").GroupingNetworkModule({"model_parameter": dict(mp.TGN_PARAMS)}).cuda().train()
            if state is None:
                state = {k: v.clone() for k, v in module.state_dict().items()}

            def fwd():
                module.load_state_dict(state)
                return module([feats, labels])

            outs[ops] = fwd()["sem_1"].clone()
            ms[ops] = time_ms(fwd, warm=1, reps=3)
            if ops == "b200":
                blocks_fused.set_enabled(False)
                try:
                    ms["b200_unfused_blocks"] = time_ms(fwd, warm=1, reps=3)
                finally:
                    blocks_fused.set_enabled(True)
    a, b = outs["b200"].double(), outs["reference"].double()
    err = float(((a - b).abs() / b.abs().clamp(min=0.05 * float(b.abs().max()))).max())
    return {"points": points, "ms": ms, "speedup_vs_reference_ops": ms["reference"] / ms["b200"], "sem_1_elementwise_vs_reference": err,
            "note": "train-mode BatchNorm amplifies fp32 rounding for both sides; scripts/model_parity.py --cases tgni gives the float64 verdict"}
