#!/usr/bin/env python
"""Model-level parity + timing of the reference's REAL model files on the two operator sets
(VERDICT r1 item 1; SURVEY.md 8d configs C2-model, C3, C4).

    python scripts/model_parity.py [--out PATH.json] [--points 24000] [--cases pp,tseg,tgn,tgni,tgnb] [--fused-decoder-blocks]

For each case the reference's unmodified ``models/modules/*.py`` is built twice in this process
(``oracle/ref_models.World``): once on the reference's own operators (verbatim ``pointops`` kernels
from ``oracle/_ref`` + the reference's torch ``pointnet2_utils.py``) and once on
``toothgroupnetwork_b200`` via ``dropin.install()``; same weights (state_dict copy), same inputs,
BatchNorm mode recorded, cuDNN/cuBLAS TF32 off (SURVEY.md 7.1).  Compared: every output tensor
ELEMENT-WISE, |a-b| / max(|b|, FLOOR * max|b|) with FLOOR = 0.05, i.e. rtol 1e-4 with atol 5e-6 * max|b| (an fp32
chain of this depth carries ~1e-6 * max|b| of rounding noise on every element; the strict 1e-3 floor and the norm-wise figure
are reported beside it), every sampled coordinate set bitwise (=> FPS indices identical), crop indices bitwise,
and for C3 every parameter gradient.

Noise floor.  With batch-statistics BatchNorm and random-init weights these networks amplify fp32 rounding
differences by 1e3-1e5 (a channel with small variance is scaled by 1/sqrt(var)); the reference does not reproduce
ITSELF to 1e-4 when only its summation order changes.  Each case therefore also runs the reference a second time
with an arithmetic-equivalent change (cuDNN disabled -> native convolution kernels for the pointnet++ models; a
second run of the atomics-based backward for tgnet) and reports that deviation as ``reference_self_noise``.
For the pointnet++ models a float64 run of the REFERENCE model (same indices: FPS / ball query evaluated on the
float32 coordinates) gives the exact answer of the network; both fp32 implementations are measured against it.
The verdict is  worst <= max(1e-4, 3 x self-noise)  OR  (ours vs fp64 truth) <= max(1e-4, 2 x (reference vs fp64 truth)):
i.e. within 1e-4 of the reference, or -- where the reference itself is further than that from the exact result -- at
least as close to the exact result as the reference is.

Cases
  pp    ``PointPpFirstModule`` forward (``models/modules/pointnet_pp.py:80-92``), train-mode BN (what the
        reference's inference runs, SURVEY 3c) and eval-mode BN.
  tseg  tsegnet centroid + seg pipeline (``models/modules/tsegnet.py:35-88``): ``cent_module`` on the
        24k cloud, 3072-NN crops (``ops_utils.py:146-161,198-218``), distance field (``tsegnet.py:24-33``),
        ``seg_module`` on (8, 36, 3072).  The DBSCAN step (``tsegnet.py:57-71``) needs trained offsets
        to find clusters; with random-init weights the 8 crop centres are the GT tooth centroids instead.
  tgn   ``GroupingNetworkModule`` forward + backward, ``train_configs/tgnet_fps.py:27-36`` parameters.
  tgni  the same module under no_grad (validation form, labels given), train- and eval-mode BN; fused and unfused blocks timed.
  tgnb  the boundary network (``train_configs/tgnet_bdl.py``: planes [16, 32], stride [1, 1], nsample [36, 24]) under no_grad
        in the form the tgnet inference pipeline calls it (``test=True``, inference_pipeline_tgn.py:229), train-mode BN; its
        c = 16 transformer layers run on the fused kernel's half-warp schedule.  Fused and unfused blocks timed.

This is test infrastructure: it imports ``oracle/``.  ``--cpu-dry-run`` exercises the harness on the
reference world only (oracle FPS/kNN on CPU, small cloud) in a GPU-less container.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time
import warnings

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
warnings.filterwarnings("ignore")

from oracle import ref_models  # noqa: E402
from toothgroupnetwork_b200 import clouds  # noqa: E402

REL_TOL = 1e-4
FLOOR = 0.05
TRUTH_FACTOR = 2.0
NOISE_FACTOR = 3.0
TGN_PARAMS = {"input_feat": 6, "stride": [1, 4, 4, 4, 4], "nsample": [36, 24, 24, 24, 24], "blocks": [2, 3, 4, 6, 3],
              "block_num": 5, "planes": [32, 64, 128, 256, 512], "crop_sample_size": 3072}
TGNB_PARAMS = {"input_feat": 6, "stride": [1, 1], "nsample": [36, 24], "blocks": [2, 3], "block_num": 2, "planes": [16, 32],
               "crop_sample_size": 3072}


def dev(t):
    return t.cuda() if torch.cuda.is_available() else t


def make_inputs(n, seed=0):
    xyz, normal, label = clouds.dental_arch(n, seed)
    feats = torch.cat([xyz, normal], 1).t().contiguous().unsqueeze(0)
    return dev(feats), dev(label.view(1, 1, n).float())


def compare(a: torch.Tensor, b: torch.Tensor, abs_floor: float = 0.0):
    """element-wise relative error of a (ours) against b (reference): |a-b| / max(|b|, FLOOR * max|b|, abs_floor)."""
    a, b = a.detach().double().flatten(), b.detach().double().flatten()
    if not b.numel():
        return {"max_rel": 0.0, "max_rel_floor1e-3": 0.0, "normwise": 0.0, "p999_rel": 0.0, "max_abs": 0.0, "ref_max_abs": 0.0,
                "bitwise": True, "numel": 0}
    scale = float(b.abs().max())
    d = (a - b).abs()
    rel = d / torch.clamp(b.abs(), min=max(FLOOR * scale, abs_floor, 1e-300))
    strict = d / torch.clamp(b.abs(), min=max(1e-3 * scale, abs_floor, 1e-300))
    return {"max_rel": float(rel.max()), "max_rel_floor1e-3": float(strict.max()), "normwise": float(d.max() / max(scale, 1e-300)),
            "p999_rel": float(torch.quantile(rel[: 4_000_000], 0.999)), "max_abs": float(d.max()), "ref_max_abs": scale,
            "bitwise": bool(torch.equal(a, b)), "numel": int(a.numel())}


class cudnn_disabled:
    """Arithmetic-equivalent perturbation of the reference: native convolution kernels instead of cuDNN's."""

    def __enter__(self):
        self.saved = torch.backends.cudnn.enabled
        torch.backends.cudnn.enabled = False

    def __exit__(self, *exc):
        torch.backends.cudnn.enabled = self.saved


def verdict(worst: float, noise, truth=None):
    bar = max(REL_TOL, NOISE_FACTOR * noise) if noise is not None else REL_TOL
    ok = worst <= bar
    out = {"worst_max_rel": worst, "reference_self_noise": noise, "bar": bar,
           "rule": f"worst <= max({REL_TOL}, {NOISE_FACTOR} x reference_self_noise), element-wise with floor {FLOOR} * max|ref|"}
    if truth is not None:
        ours_t, ref_t = truth
        ok_t = ours_t <= max(REL_TOL, TRUTH_FACTOR * ref_t)
        out.update({"ours_vs_fp64_truth": ours_t, "reference_vs_fp64_truth": ref_t, "pass_vs_truth": bool(ok_t),
                    "rule_truth": f"ours_vs_fp64_truth <= max({REL_TOL}, {TRUTH_FACTOR} x reference_vs_fp64_truth)"})
        ok = ok or ok_t
    out["pass"] = bool(ok)
    return out


class float64_reference:
    """Run the reference's pointnet2 modules in float64 while its index-producing steps keep seeing the float32
    coordinates (so that FPS / ball-query indices are the ones of the fp32 runs): the exact answer of the network."""

    def __init__(self, world):
        self.pn = world.mod("external_libs.pointnet2_utils.pointnet2_utils")

    def __enter__(self):
        pn = self.pn
        self.saved = (pn.farthest_point_sample, pn.query_ball_point)
        fps, qbp = self.saved
        pn.farthest_point_sample = lambda xyz, npoint: fps(xyz.float(), npoint)
        pn.query_ball_point = lambda radius, nsample, xyz, new_xyz: qbp(radius, nsample, xyz.float(), new_xyz.float())

    def __exit__(self, *exc):
        self.pn.farthest_point_sample, self.pn.query_ball_point = self.saved


class float64_point_transformer:
    """The same for the packed-layout operators of the point-transformer models: FPS and kNN see the float32 coordinates, the
    3-NN interpolation of the decoder keeps float64 (the reference's own accumulates into a FloatTensor, pointops.py:160-180)."""

    def __init__(self, world):
        self.po = world.mod("external_libs.pointops.functions.pointops")

    def __enter__(self):
        po = self.po
        self.saved = (po.furthestsampling, po.knnquery, po.interpolation)
        fps, knn, _ = self.saved
        po.furthestsampling = lambda xyz, off, noff: fps(xyz.float().contiguous(), off, noff)

        def knn64(k, xyz, new_xyz, off, noff):
            idx, _ = knn(k, xyz.float().contiguous(), (xyz if new_xyz is None else new_xyz).float().contiguous(), off, noff)
            q = xyz if new_xyz is None else new_xyz
            d = (xyz[idx.long().view(-1)].view(idx.shape[0], idx.shape[1], 3) - q.unsqueeze(1)).pow(2).sum(-1).sqrt()
            return idx, d

        def interp64(xyz, new_xyz, feat, off, noff, k=3):
            idx, dist = knn64(k, xyz, new_xyz, off, noff)
            w = 1.0 / (dist + 1e-8)
            w = w / w.sum(1, keepdim=True)
            return (feat[idx.long().view(-1)].view(idx.shape[0], k, -1) * w.unsqueeze(-1)).sum(1)

        po.knnquery, po.interpolation = knn64, interp64

    def __exit__(self, *exc):
        self.po.furthestsampling, self.po.knnquery, self.po.interpolation = self.saved


class Timer:
    def __init__(self):
        self.gpu = torch.cuda.is_available()

    def __call__(self, fn, warm=1, reps=3):
        out = None
        for _ in range(warm):
            out = fn()
        if self.gpu:
            torch.cuda.synchronize()
            ts = []
            for _ in range(reps):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                out = fn()
                e1.record()
                torch.cuda.synchronize()
                ts.append(e0.elapsed_time(e1))
            return out, float(np.median(ts))
        t0 = time.perf_counter()
        out = fn()
        return out, (time.perf_counter() - t0) * 1e3


def hook_sampled_coords(model, store):
    """Record the coordinates every sampling stage hands on (bitwise equality <=> identical FPS indices)."""
    hs = []
    for name, m in model.named_modules():
        cls = type(m).__name__
        if cls in ("PointNetSetAbstractionMsg", "PointNetSetAbstraction", "TransitionDown"):
            def hook(mod, inp, out, name=name):
                store.setdefault(name, out[0].detach().clone())      # a hook's return value would replace the output
            hs.append(m.register_forward_hook(hook))
    return hs


def summarize(pairs, tol=REL_TOL):
    worst = max((v["max_rel"] for v in pairs.values()), default=0.0)
    return {"worst_max_rel": worst, "pass": bool(worst <= tol), "tensors": pairs}


# ------------------------------------------------------------------------------------------ cases
def case_pp(worlds, feats, train_bn, timer):
    outs, coords, times, launches = {}, {}, {}, {}
    state = None
    for w in worlds:
        with w:
            torch.manual_seed(0)
            model = dev(w.mod("models.modules.pointnet_pp").PointPpFirstModule({}))
            if state is None:
                state = {k: v.clone() for k, v in model.state_dict().items()}
            else:
                model.load_state_dict(state)
            model.train(train_bn)
            coords[w.ops] = {}
            hs = hook_sampled_coords(model, coords[w.ops])
            with torch.no_grad():
                (o, ms) = timer(lambda: model([feats]))
            for h in hs:
                h.remove()
            outs[w.ops], times[w.ops] = {"cls_pred": o["cls_pred"]}, ms
            if w.ops == "reference" and torch.cuda.is_available():
                model.load_state_dict(state)                      # training-mode BN moved the running statistics
                with torch.no_grad(), cudnn_disabled():
                    outs["reference_noise"] = {"cls_pred": model([feats])["cls_pred"]}
                model.load_state_dict(state)
                model.double()
                with torch.no_grad(), float64_reference(w):
                    outs["fp64_truth"] = {"cls_pred": model([feats.double()])["cls_pred"]}
                model.float()
    return finish(outs, coords, times)


def gt_centroids(feats, labels, take=None, seed=0):
    lab = labels.view(-1).cpu().numpy()
    xyz = feats[0, :3].t().cpu().numpy()
    cents = [xyz[lab == t].mean(0) for t in np.unique(lab) if t != -1]
    cents = np.stack(cents)
    if take is not None:
        cents = cents[np.random.RandomState(seed).permutation(len(cents))[:take]]
    return cents


def case_tseg(worlds, feats, labels, train_bn, timer):
    outs, coords, times = {}, {}, {}
    cstate = sstate = None
    for w in worlds:
        with w:
            torch.manual_seed(0)
            tseg = w.mod("models.modules.tsegnet")
            ou = w.mod("ops_utils")
            module = dev(tseg.TSegNetModule({"run_tooth_segmentation_module": True}))
            if cstate is None:
                cstate = {k: v.clone() for k, v in module.state_dict().items()}
            else:
                module.load_state_dict(cstate)
            module.train(train_bn)
            coords[w.ops] = {}
            hs = hook_sampled_coords(module, coords[w.ops])
            centres = gt_centroids(feats, labels, take=8)[None].astype(np.float32)          # (1, 8, 3)

            def pipeline(feats=feats, centres=centres):
                l0_points, l3_points, l0_xyz, l3_xyz, offset_result, dist_result = module.cent_module(feats)
                nn_idx = ou.get_nearest_neighbor_idx(l0_xyz.permute(0, 2, 1).detach().float().cpu().numpy(), centres.astype(np.float32), 3072)   # tsegnet.py:73
                cropped_input = ou.get_indexed_features(feats, nn_idx)
                cropped_feat = ou.get_indexed_features(l0_points, nn_idx)
                ddf = module.get_ddf(cropped_input[:, :3, :].permute(0, 2, 1), centres) if torch.cuda.is_available() else \
                    torch.zeros(cropped_input.shape[0], 1, 3072)
                x = torch.cat([cropped_input[:, :3, :], cropped_feat, ddf], axis=1)
                pd_1, weight_1, pd_2, id_pred = module.seg_module(x)
                return {"l0_points": l0_points, "l3_points": l3_points, "offset_result": offset_result, "dist_result": dist_result,
                        "seg_input": x, "pd_1": pd_1, "weight_1": weight_1, "pd_2": pd_2, "id_pred": id_pred}

            with torch.no_grad():
                o, ms = timer(pipeline)
            for h in hs:
                h.remove()
            outs[w.ops], times[w.ops] = o, ms
            if w.ops == "reference" and torch.cuda.is_available():
                module.load_state_dict(cstate)
                with torch.no_grad(), cudnn_disabled():
                    outs["reference_noise"] = pipeline()
                module.load_state_dict(cstate)
                module.double()
                with torch.no_grad(), float64_reference(w):
                    outs["fp64_truth"] = pipeline(feats.double(), centres.astype(np.float64))
                module.float()
    return finish(outs, coords, times)


def case_tgn(worlds, feats, labels, timer):
    outs, coords, times, grads = {}, {}, {}, {}
    state = None
    for w in worlds:
        with w:
            torch.manual_seed(0)
            gm = w.mod("models.modules.grouping_network_module")
            module = dev(gm.GroupingNetworkModule({"model_parameter": dict(TGN_PARAMS)}))
            if state is None:
                state = {k: v.clone() for k, v in module.state_dict().items()}
            else:
                module.load_state_dict(state)
            module.train()
            coords[w.ops] = {}
            hs = hook_sampled_coords(module, coords[w.ops])
            keys = ("cbl_loss_1", "sem_1", "offset_1", "first_features", "cbl_loss_2", "sem_2", "cropped_feature_ls")

            def fwd_bwd():
                module.zero_grad(set_to_none=True)
                coords[w.ops].clear()
                out = module([feats, labels])
                loss = out["cbl_loss_1"].sum() + out["cbl_loss_2"].sum()
                for k in ("sem_1", "offset_1", "sem_2"):
                    loss = loss + (out[k] ** 2).mean()
                loss.backward()
                return out, loss

            (o, loss), ms = timer(fwd_bwd, warm=1, reps=2)
            for h in hs:
                h.remove()
            outs[w.ops] = {k: o[k] for k in keys if o.get(k) is not None}
            outs[w.ops]["loss"] = loss.detach().view(1)
            outs[w.ops]["nn_crop_indexes"] = torch.from_numpy(np.stack([np.asarray(x) for x in o["nn_crop_indexes"]]).astype(np.int64))
            grads[w.ops] = {n: p.grad.detach().clone() for n, p in module.named_parameters() if p.grad is not None}
            times[w.ops] = ms
            if w.ops == "reference" and torch.cuda.is_available():
                module.load_state_dict(state)
                o2, loss2 = fwd_bwd()                             # same code again: the atomics-based backward is order-dependent
                outs["reference_noise"] = {k: o2[k] for k in keys if o2.get(k) is not None}
                outs["reference_noise"]["loss"] = loss2.detach().view(1)
                outs["reference_noise"]["nn_crop_indexes"] = outs[w.ops]["nn_crop_indexes"]
                grads["reference_noise"] = {n: p.grad.detach().clone() for n, p in module.named_parameters() if p.grad is not None}
    res = finish(outs, coords, times)
    if "b200" in grads and "reference" in grads:
        g_ref = grads["reference"]
        gmax = max(float(g.abs().max()) for g in g_ref.values())
        # parameters whose true gradient is zero (a bias in front of a BatchNorm) hold pure rounding noise ~1e-9 of the
        # largest gradient in both runs: every tensor is compared above an absolute floor of 1e-6 * max|any gradient|

        def sweep(g_other):
            worst, worst_name, over = 0.0, None, {}
            for n in g_ref:
                c = compare(g_other[n], g_ref[n], abs_floor=1e-6 * gmax)
                if c["max_rel"] > worst:
                    worst, worst_name = c["max_rel"], n
                if c["max_rel"] > REL_TOL:
                    over[n] = c["max_rel"]
            return worst, worst_name, over

        worst, worst_name, over = sweep(grads["b200"])
        noise = sweep(grads["reference_noise"])[0] if "reference_noise" in grads else None
        res["grads"] = dict(verdict(worst, noise), n_tensors=len(g_ref), worst_tensor=worst_name, max_abs_gradient=gmax,
                            n_over_tol=len(over), abs_floor="1e-6 * max|any gradient|")
    return res


def case_tgn_infer(worlds, feats, labels, train_bn, timer, params=TGN_PARAMS, test=False):
    """GroupingNetworkModule forward under torch.no_grad() with labels given (the reference's validation step,
    grouping_network_module.py:25-35,46-57: crops around the ground-truth centroids; the label-free inference branch :58-69 clusters
    the predicted offsets instead, which needs trained weights -- tests/test_gpu_clustering.py covers that function): in the b200 world the
    PointTransformerLayer and TransitionDown forwards run on the fused kernels (toothgroupnetwork_b200.blocks_fused).
    ``params`` is the model_parameter dict (TGN_PARAMS: the first network; TGNB_PARAMS: the boundary network); ``test=True`` is the
    forward's test flag, as the inference pipeline passes it (the first model then runs without labels; crops still follow them)."""
    outs, coords, times = {}, {}, {}
    state = None
    keys = ("sem_1", "offset_1", "first_features", "sem_2", "cropped_feature_ls")
    for w in worlds:
        with w, torch.no_grad():
            torch.manual_seed(0)
            gm = w.mod("models.modules.grouping_network_module")
            if w.ops == "b200" and FUSED_DECODER_BLOCKS:
                from toothgroupnetwork_b200 import blocks_fused
                blk = w.mod("models.modules.cbl_point_transformer.blocks")
                blocks_fused.accelerate_decoder(blk, w.mod("models.modules.cbl_point_transformer.heads"))
                blocks_fused.accelerate_blocks(blk)
            module = dev(gm.GroupingNetworkModule({"model_parameter": dict(params)}))
            if state is None:
                state = {k: v.clone() for k, v in module.state_dict().items()}
            module.train(train_bn)
            coords[w.ops] = {}
            hs = hook_sampled_coords(module, coords[w.ops])

            def fwd():
                module.load_state_dict(state)                      # same running statistics every repetition
                coords[w.ops].clear()
                return module([feats, labels], test=test)

            o, ms = timer(fwd, warm=1, reps=3)
            outs[w.ops] = {k: o[k] for k in keys if o.get(k) is not None}
            outs[w.ops]["nn_crop_indexes"] = torch.from_numpy(np.stack([np.asarray(x) for x in o["nn_crop_indexes"]]).astype(np.int64))
            times[w.ops] = ms
            raw_crops = o["nn_crop_indexes"]
            if w.ops == "b200" and torch.cuda.is_available():
                from toothgroupnetwork_b200 import blocks_fused
                blocks_fused.set_enabled(False)
                try:
                    _, times["b200_unfused_blocks"] = timer(fwd, warm=1, reps=3)
                finally:
                    blocks_fused.set_enabled(True)
            for h in hs:
                h.remove()
            if w.ops == "reference" and torch.cuda.is_available():
                ou = w.mod("ops_utils")
                saved_crop = ou.get_nearest_neighbor_idx
                # the float64 run clusters slightly different offsets: it is handed the float32 run's crops, so that the second
                # module's outputs are the exact answer for the same crops
                ou.get_nearest_neighbor_idx = lambda *a, **k: raw_crops
                try:
                    with float64_point_transformer(w):
                        module.load_state_dict(state)
                        module.double()
                        o = module([feats.double(), labels], test=test)
                        outs["fp64_truth"] = {k: o[k] for k in keys if o.get(k) is not None}
                        outs["fp64_truth"]["nn_crop_indexes"] = torch.from_numpy(np.stack([np.asarray(x) for x in o["nn_crop_indexes"]]).astype(np.int64))
                except Exception as e:                             # the truth leg is an aid, not the gate
                    print("fp64 truth unavailable:", repr(e)[:300])
                    outs.pop("fp64_truth", None)
                finally:
                    ou.get_nearest_neighbor_idx = saved_crop
    return finish(outs, coords, times)


def finish(outs, coords, times):
    res = {"ms": times}
    if "b200" in outs and "reference" in outs:
        new, ref = outs["b200"], outs["reference"]
        res.update(summarize({k: compare(new[k].float(), ref[k].float()) for k in ref}))
        noise = None
        if "reference_noise" in outs:
            pert = outs["reference_noise"]
            per = {k: compare(pert[k].float(), ref[k].float())["max_rel"] for k in ref}
            noise = max(per.values())
            res["reference_self_noise_per_tensor"] = per
        truth = None
        if "fp64_truth" in outs:
            t = outs["fp64_truth"]
            per_o = {k: compare(new[k].double(), t[k].double())["max_rel"] for k in ref}
            per_r = {k: compare(ref[k].double(), t[k].double())["max_rel"] for k in ref}
            res["vs_fp64_truth_per_tensor"] = {k: {"ours": per_o[k], "reference": per_r[k]} for k in ref}
            # the verdict compares tensor by tensor: the worst ratio decides
            worst_k = max(ref, key=lambda k: per_o[k] / max(REL_TOL / TRUTH_FACTOR, per_r[k]))
            truth = (per_o[worst_k], per_r[worst_k])
        res["verdict"] = verdict(res["worst_max_rel"], noise, truth)
        c_new, c_ref = coords["b200"], coords["reference"]
        res["sampled_coords_bitwise"] = {k: bool(torch.equal(c_new[k], c_ref[k])) for k in c_ref}
        res["indices_identical"] = bool(all(res["sampled_coords_bitwise"].values()))
        if "nn_crop_indexes" in ref:
            res["crop_indexes_identical"] = bool(torch.equal(new["nn_crop_indexes"], ref["nn_crop_indexes"]))
        res["speedup_vs_reference_ops"] = times["reference"] / times["b200"] if times["b200"] > 0 else None
    return res


FUSED_DECODER_BLOCKS = False


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "gpurun_out", "model_parity.json"))
    ap.add_argument("--points", type=int, default=24000)
    ap.add_argument("--cases", default="pp,tseg,tgn,tgni")
    ap.add_argument("--cpu-dry-run", action="store_true")
    ap.add_argument("--fused-decoder-blocks", action="store_true",
                    help="tgni / tgnb: also run TransitionUp, MultiHead and PointTransformerBlock on the fused kernels "
                         "(blocks_fused.accelerate_decoder and accelerate_blocks)")
    args = ap.parse_args()
    global FUSED_DECODER_BLOCKS
    FUSED_DECODER_BLOCKS = args.fused_decoder_blocks

    if args.cpu_dry_run:
        torch.Tensor.cuda = lambda self, *a, **k: self
        torch.nn.Module.cuda = lambda self, *a, **k: self
        mk = lambda dt: (lambda *a: torch.tensor(a[0], dtype=dt) if len(a) == 1 and isinstance(a[0], (list, tuple))
                         else torch.zeros(*[int(x) for x in a], dtype=dt))
        torch.cuda.IntTensor, torch.cuda.FloatTensor = mk(torch.int32), mk(torch.float32)
        worlds = [ref_models.World("reference", cpu_dry_run=True)]
    else:
        assert torch.cuda.is_available(), "model parity needs the GPU (or --cpu-dry-run)"
        torch.backends.cudnn.allow_tf32 = False
        torch.backends.cuda.matmul.allow_tf32 = False
        worlds = [ref_models.World("reference"), ref_models.World("b200")]

    feats, labels = make_inputs(args.points)
    timer = Timer()
    report = {"points": args.points, "fused_decoder_blocks": FUSED_DECODER_BLOCKS, "rel_tol": REL_TOL, "floor": "1e-3 * max|reference tensor|",
              "precision": "cudnn.allow_tf32=False, cuda.matmul.allow_tf32=False", "device": torch.cuda.get_device_name(0) if torch.cuda.is_available() else "cpu"}
    cases = args.cases.split(",")
    if "pp" in cases:
        report["pointnet_pp_trainBN"] = case_pp(worlds, feats, True, timer)
        report["pointnet_pp_evalBN"] = case_pp(worlds, feats, False, timer)
    if "tseg" in cases:
        report["tsegnet_trainBN"] = case_tseg(worlds, feats, labels, True, timer)
        report["tsegnet_evalBN"] = case_tseg(worlds, feats, labels, False, timer)
    if "tgn" in cases:
        report["tgnet_fps_fwd_bwd"] = case_tgn(worlds, feats, labels, timer)
    if "tgni" in cases:
        report["tgnet_fps_nograd_trainBN"] = case_tgn_infer(worlds, feats, labels, True, timer)
        report["tgnet_fps_nograd_evalBN"] = case_tgn_infer(worlds, feats, labels, False, timer)
    if "tgnb" in cases:
        report["tgnet_bdl_nograd_test_trainBN"] = case_tgn_infer(worlds, feats, labels, True, timer, params=TGNB_PARAMS, test=True)
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(report, f, indent=1)
    brief = {k: {kk: v[kk] for kk in ("verdict", "indices_identical", "crop_indexes_identical", "ms", "speedup_vs_reference_ops", "grads")
                 if kk in v}
             for k, v in report.items() if isinstance(v, dict)}
    print(json.dumps(brief, indent=1))


if __name__ == "__main__":
    main()
