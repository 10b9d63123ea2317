"""Bucket-FPS traffic: bytes the main kernel reads per iteration, and the rate it reads them at.

    python scripts/fps_traffic.py [--layout 16|20] [--no-gpu] [--out fps_traffic.json]

CPU model (no GPU needed): the bench clouds (24 000-point dental arches, seeds 0..7) -> 1024 samples, sorted and
bucketed as fps_bucket_sort_kernel does (17-bit Morton codes, 64-point buckets, boxes inflated by 4e-6*max|coord|),
pruned with the main kernel's test dist2(o, box) > max_t*1.00002.  Per iteration it counts
  * bucket_points: 64 points per surviving bucket, what fps_bucket_kernel reads (16 B per point: x,y | z,t, the tie keys
    kept apart; the earlier record was 20 B: x,y | z,key | t);
  * subbox_points: what a variant with 16-point sub-boxes, quantised to 4 bits inside the bucket box, would read: the whole
    bucket when the sub-box of the bucket's current candidate survives (the candidate must be refreshed), otherwise the
    surviving sub-boxes only;
  * subbox_exact_points: the same with unquantised sub-boxes.
On a GPU it also times the sort kernel and the main kernel apart (torch.profiler) at B in {132, 264, 528, 1056} in auto mode
and with mode -14 (4 warps per cloud) at B = 1056, and prints counted bytes over main-kernel time against the HBM peak.
--layout names the point record of the library being timed, in bytes (counted traffic = bucket_points * layout).
"""
from __future__ import annotations

import argparse
import json
import os
import re
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

N, M, BP, HBM_GBS = 24000, 1024, 64, 3350.0


def _spread3(x):
    x = x.astype(np.uint32)
    x = (x | (x << 16)) & np.uint32(0x030000FF)
    x = (x | (x << 8)) & np.uint32(0x0300F00F)
    x = (x | (x << 4)) & np.uint32(0x030C30C3)
    x = (x | (x << 2)) & np.uint32(0x09249249)
    return x


def _box_dist2(lo, hi, o):
    e = np.maximum(np.maximum(lo - o, o - hi), np.float32(0))
    return (e[..., 0] * e[..., 0] + e[..., 1] * e[..., 1]) + e[..., 2] * e[..., 2]


def _quantised_subboxes(lo_b, hi_b, lo_t, hi_t):
    """Decoded 4-bit sub-box bounds inside the bucket box [lo_b, hi_b] (the scheme of fps_bucket_sort_kernel: lower bound
    L + q*s, upper bound H - q*s with s = (H - L)/15, the tightest q that still encloses [lo_t, hi_t])."""
    s = ((hi_b - lo_b) * np.float32(1.0 / 15.0)).astype(np.float32)[:, None, :]
    L, H = lo_b[:, None, :], hi_b[:, None, :]
    q = np.arange(16, dtype=np.float32)[:, None, None, None]
    dec_lo = (q * s.astype(np.float64) + L).astype(np.float32)          # (16, nb, 4, 3)
    dec_hi = (-q * s.astype(np.float64) + H).astype(np.float32)
    ok_lo = dec_lo <= lo_t[None]
    ok_hi = dec_hi >= hi_t[None]
    qlo = 15 - np.argmax(ok_lo[::-1], axis=0)                            # largest q with dec_lo(q) <= lo_t (q = 0 always holds)
    qhi = 15 - np.argmax(ok_hi[::-1], axis=0)
    take = lambda d, qq: np.take_along_axis(d, qq[None], axis=0)[0]
    return take(dec_lo, qlo), take(dec_hi, qhi)


def model_cloud(xyz: np.ndarray, m: int = M) -> dict:
    xyz = np.ascontiguousarray(xyz, np.float32)
    n = xyz.shape[0]
    lo, hi = xyz.min(0), xyz.max(0)
    code = np.zeros(n, np.uint32)
    for a, bits in enumerate((6, 6, 5)):
        ext = np.float32(hi[a] - lo[a])
        inv = np.float32((np.float32(1 << bits) - np.float32(0.001)) / ext) if ext > 0 else np.float32(0)
        q = np.minimum(np.uint32((1 << bits) - 1), np.maximum((xyz[:, a] - lo[a]) * inv, np.float32(0)).astype(np.uint32))
        code |= _spread3(q) << np.uint32(a)
    order = np.argsort(code, kind="stable")
    slack = np.float32(4e-6) * np.float32(max(np.abs(lo).max(), np.abs(hi).max()))
    nb = (n + BP - 1) // BP
    P = np.zeros((nb * BP, 3), np.float32)
    P[:n] = xyz[order]
    valid = np.zeros(nb * BP, bool)
    valid[:n] = True
    Pb, Vb = P.reshape(nb, BP, 3), valid.reshape(nb, BP)
    inf = np.float32(np.inf)
    blo = np.where(Vb[..., None], Pb, inf).min(1) - slack
    bhi = np.where(Vb[..., None], Pb, -inf).max(1) + slack
    Ps, Vs = Pb.reshape(nb, 4, 16, 3), Vb.reshape(nb, 4, 16)
    slo = np.where(Vs[..., None], Ps, inf).min(2) - slack
    shi = np.where(Vs[..., None], Ps, -inf).max(2) + slack
    qlo, qhi = _quantised_subboxes(blo, bhi, slo, shi)
    t = np.where(valid, np.float32(1e10), np.float32(-1)).astype(np.float32)
    o = xyz[0]
    bucket_pts = sub_pts = exact_pts = 0
    for _ in range(1, m):
        tb = t.reshape(nb, BP)
        maxt, cand = tb.max(1), tb.argmax(1)
        thr = maxt * np.float32(1.00002)
        act = ~(_box_dist2(blo, bhi, o) > thr)
        sub_act = ~(_box_dist2(qlo, qhi, o[None, None]) > thr[:, None]) & act[:, None]
        full = sub_act[np.arange(nb), cand // 16]
        bucket_pts += BP * int(act.sum())
        sub_pts += int(np.where(full, BP, 16 * sub_act.sum(1)).sum())
        exact_sub = ~(_box_dist2(slo, shi, o[None, None]) > thr[:, None]) & act[:, None]
        exact_pts += int(np.where(exact_sub[np.arange(nb), cand // 16], BP, 16 * exact_sub.sum(1)).sum())
        d = P - o
        d2 = (d[:, 1] * d[:, 1] + d[:, 0] * d[:, 0]) + d[:, 2] * d[:, 2]
        t = np.where(valid, np.minimum(t, d2), t)
        o = P[int(np.argmax(t))]
    it = m - 1
    return {"buckets": nb, "bucket_points_per_it": bucket_pts / it, "subbox_points_per_it": sub_pts / it,
            "subbox_exact_points_per_it": exact_pts / it}


def model(seeds=range(8)) -> dict:
    from toothgroupnetwork_b200 import clouds
    rows = [model_cloud(clouds.arch_features(N, clouds.cloud_seed(0, s))[0][:3].T.contiguous().numpy()) for s in seeds]
    avg = {k: float(np.mean([r[k] for r in rows])) for k in rows[0] if k != "buckets"}
    return {"per_cloud": rows, "mean": avg,
            "bytes_per_it_20B_buckets": 20.0 * avg["bucket_points_per_it"],
            "bytes_per_it_16B_buckets": 16.0 * avg["bucket_points_per_it"],
            "bytes_per_it_16B_subboxes": 16.0 * avg["subbox_points_per_it"]}


def gpu_times(layout_bytes_per_it: float) -> list:
    import torch
    from torch.profiler import ProfilerActivity, profile
    from toothgroupnetwork_b200 import clouds, pointops
    base = [clouds.arch_features(N, clouds.cloud_seed(0, s))[0][:3].T.contiguous() for s in range(8)]
    rows = []
    for B, mode in ((132, 0), (264, 0), (528, 0), (1056, 0), (1056, -14)):
        xyz = torch.cat([base[j % 8] for j in range(B)]).cuda()
        off = (torch.arange(1, B + 1, dtype=torch.int32) * N).cuda()
        noff = (torch.arange(1, B + 1, dtype=torch.int32) * M).cuda()
        run = lambda: pointops.fps_packed(xyz, off, noff, N, B * M, mode)
        for _ in range(2):
            run()
        torch.cuda.synchronize()
        reps = 5
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(reps):
                run()
            torch.cuda.synchronize()
        sort_us = main_us = 0.0
        main_names = set()
        for e in prof.key_averages():
            us = getattr(e, "device_time_total", None)
            if us is None:
                us = e.cuda_time_total
            if "fps_bucket_sort_kernel" in e.key:
                sort_us += us
            elif "fps_bucket_kernel" in e.key:
                main_us += us
                main_names.add(re.search(r"fps_bucket_kernel\w*(<[^>]*>)?", e.key).group(0))
        sort_ms, main_ms = sort_us / reps / 1e3, main_us / reps / 1e3
        counted = layout_bytes_per_it * (M - 1) * B
        gbs = counted / (main_ms * 1e-3) / 1e9 if main_ms > 0 else float("nan")
        row = {"clouds": B, "mode": mode, "main_kernel": sorted(main_names), "sort_ms": round(sort_ms, 3),
               "main_ms": round(main_ms, 3), "counted_GB": round(counted / 1e9, 3), "main_GBs": round(gbs, 1),
               "frac_hbm_peak": round(gbs / HBM_GBS, 3)}
        rows.append(row)
        print(json.dumps(row), flush=True)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layout", type=int, choices=(16, 20), default=16, help="point record of the library being timed")
    ap.add_argument("--no-gpu", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    rep = {"model": model()}
    print(json.dumps(rep["model"]["mean"]), flush=True)
    print(json.dumps({k: v for k, v in rep["model"].items() if k.startswith("bytes")}), flush=True)
    if not args.no_gpu:
        import torch
        assert torch.cuda.is_available(), "timing needs a CUDA device (use --no-gpu for the model alone)"
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True)
        rep["gpu"] = q.stdout.strip()
        print(rep["gpu"], flush=True)
        per_it = args.layout * rep["model"]["mean"]["bucket_points_per_it"]
        rep["layout_bytes_per_point"] = args.layout
        rep["timing"] = gpu_times(per_it)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(rep, f, indent=1)


if __name__ == "__main__":
    main()
