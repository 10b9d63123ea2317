"""Device k-means fits (csrc/kmeans.cu through clustering.KMeans and one-launch batches) against scikit-learn on the host.

    python scripts/kmeans_bench.py [--reps 10] [--agree 12] [--out FILE]

At n in {5 000, 15 000, 24 000} and k in {8, 16, 17}, medians of --reps: the whole class call and scikit-learn's fit with its
default threads (host clock, same seeds); with CUDA events, the kernel on the class's prepared values of one of those fits, the
same fit stopped after one Lloyd step (to split seeding from Lloyd), and 16 such fits in one launch.  Then counts, per input family
and seed, how often live scikit-learn with 1 thread and with the default threads gives the class's labels_, and its own.  Prints
one JSON object with the card's name and power limit.
"""
import argparse
import json
import os
import subprocess
import sys
import time
import warnings

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from toothgroupnetwork_b200 import clouds, clustering  # noqa: E402


def family(name, n, seed):
    rng = np.random.default_rng(seed)
    if name == "arch":
        return clouds.dental_arch(n, seed)[0].numpy().astype(np.float32)
    c = rng.uniform(-0.6, 0.6, (16, 3))
    sigma = 0.015 if name == "tight" else 0.05
    return (c[rng.integers(0, 16, n)] + rng.normal(0, sigma, (n, 3))).astype(np.float32)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--agree", type=int, default=12)
    ap.add_argument("--out")
    a = ap.parse_args()
    from sklearn.cluster import KMeans
    from threadpoolctl import threadpool_limits
    warnings.simplefilter("ignore")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    res = {"card": card, "timing_ms": [], "agreement": {}}
    def events(fn, reps):
        """median CUDA-event time of fn() over reps calls, after one warm-up call"""
        fn()
        out = []
        for _ in range(reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            out.append(e0.elapsed_time(e1))
        return float(np.median(out))

    for n in (5000, 15000, 24000):
        X = family("tight", n, 1)
        for k in (8, 16, 17):
            # the class's own fit (host preparation, launch, copies back), and scikit-learn's, on the same seeds
            clustering.KMeans(k, random_state=0).fit(X)                   # warm-up
            ms_class, ms_sk = [], []
            for r in range(a.reps):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                clustering.KMeans(k, random_state=r).fit(X)
                ms_class.append((time.perf_counter() - t0) * 1e3)
                t0 = time.perf_counter()
                KMeans(k, random_state=r).fit(X)
                ms_sk.append((time.perf_counter() - t0) * 1e3)
            # the device part of the same fit as the class's random_state=0 call: the kernel on its prepared values
            Xc, _, tol, first, u = clustering.kmeans_prepare(X, k, 1e-4, np.random.RandomState(0))
            T = u.shape[1]
            args = dict(X=torch.from_numpy(Xc).cuda(), offsets=torch.tensor([0, n], dtype=torch.int32).cuda(), k=k,
                        first=torch.tensor([first], dtype=torch.int32).cuda(), uniforms=torch.from_numpy(u.reshape(1, k - 1, T)).cuda(),
                        tol=torch.tensor([tol], dtype=torch.float32).cuda())
            n_iter = int(clustering.kmeans_device(**args)[3][0])
            full = events(lambda: clustering.kmeans_device(**args), a.reps)
            one = events(lambda: clustering.kmeans_device(**args, max_iter=1), a.reps)
            # phases: max_iter = 1 is the seeding, one Lloyd step and the final E-step; the other n_iter - 1 steps make up the rest
            lloyd_step = (full - one) / max(n_iter - 1, 1)
            B = 16
            bargs = dict(args, X=args["X"].repeat(B, 1), offsets=torch.arange(B + 1, dtype=torch.int32).cuda() * n,
                         first=args["first"].repeat(B), uniforms=args["uniforms"].repeat(B, 1, 1), tol=args["tol"].repeat(B))
            batch = events(lambda: clustering.kmeans_device(**bargs), a.reps) / B
            res["timing_ms"].append({"n": n, "k": k, "n_iter": n_iter, "device_fit": full, "seeding": one - 2 * lloyd_step,
                                     "lloyd_step": lloyd_step, "class_fit": float(np.median(ms_class)), "batch16_per_fit": batch,
                                     "sklearn_default_threads": float(np.median(ms_sk))})
            print(json.dumps(res["timing_ms"][-1]), file=sys.stderr)
    for fam in ("tight", "loose", "arch"):
        counts = {"class_vs_sk1": 0, "class_vs_skdefault": 0, "sk1_vs_skdefault": 0, "fits": 0}
        for s in range(a.agree):
            X = family(fam, 14400, 50 + s)
            got = clustering.KMeans(16, random_state=s).fit(X).labels_
            with threadpool_limits(1):
                one = KMeans(16, random_state=s).fit(X).labels_
            many = KMeans(16, random_state=s).fit(X).labels_
            counts["class_vs_sk1"] += int(np.array_equal(got, one))
            counts["class_vs_skdefault"] += int(np.array_equal(got, many))
            counts["sk1_vs_skdefault"] += int(np.array_equal(one, many))
            counts["fits"] += 1
        res["agreement"][fam] = counts
    res["host_fits"] = clustering.KMeans.host_fits
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
