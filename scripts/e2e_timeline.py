"""Timeline of one pipelined end-to-end step: when each chunk's H2D, kernels and D2H finish (ms)."""
import sys, torch
sys.path.insert(0, ".")
from toothgroupnetwork_b200 import clouds, pointnet2_utils as pn2
import bench

B = int(sys.argv[1]) if len(sys.argv) > 1 else 1056
chunk = int(sys.argv[2]) if len(sys.argv) > 2 else 132
ns = int(sys.argv[3]) if len(sys.argv) > 3 else 2
mode = sys.argv[4] if len(sys.argv) > 4 else "all"      # all | h2d | compute
host = bench.make_clouds(0, B).pin_memory()
sa = pn2.PointNetSetAbstraction(bench.NPOINT, bench.RADIUS, bench.NSAMPLE, 9, bench.MLP, False).cuda().eval()
ox = torch.empty((B, 3, bench.NPOINT)).pin_memory(); op = torch.empty((B, bench.MLP[-1], bench.NPOINT)).pin_memory()
cin, cout = torch.cuda.Stream(), torch.cuda.Stream()
comp = [torch.cuda.Stream() for _ in range(ns)]
spans = [(lo, min(B, lo + chunk)) for lo in range(0, B, chunk)]
dev_cache = [host[lo:hi].cuda() for lo, hi in spans] if mode == "compute" else None

def step(record):
    main = torch.cuda.current_stream()
    t0 = torch.cuda.Event(enable_timing=True); t0.record(main)
    for s in [cin, cout] + comp: s.wait_stream(main)
    ev = []
    landed = []
    with torch.no_grad():
        with torch.cuda.stream(cin):
            for k, (lo, hi) in enumerate(spans):
                d = dev_cache[k] if mode == "compute" else host[lo:hi].to("cuda", non_blocking=True)
                e = torch.cuda.Event(enable_timing=True); e.record(cin); landed.append((d, e))
        for k, (lo, hi) in enumerate(spans):
            d, e = landed[k]
            s = comp[k % ns]; s.wait_event(e); d.record_stream(s)
            e2 = torch.cuda.Event(enable_timing=True); e3 = torch.cuda.Event(enable_timing=True)
            if mode != "h2d":
                with torch.cuda.stream(s):
                    nx, npts = sa(d[:, :3].contiguous(), d)
                    e2.record(s)
                cout.wait_event(e2); nx.record_stream(cout); npts.record_stream(cout)
                with torch.cuda.stream(cout):
                    if mode == "all":
                        ox[lo:hi].copy_(nx, non_blocking=True); op[lo:hi].copy_(npts, non_blocking=True)
                    e3.record(cout)
            else:
                e2.record(s); e3.record(s)
            ev.append((e, e2, e3))
    main.wait_stream(cout)
    for s in comp: main.wait_stream(s)
    t1 = torch.cuda.Event(enable_timing=True); t1.record(main)
    torch.cuda.synchronize()
    if record:
        print(f"mode {mode} B={B} chunk={chunk} streams={ns}: total {t0.elapsed_time(t1):.2f} ms")
        for k, (a, b, c) in enumerate(ev):
            print(f"  chunk {k}: h2d {t0.elapsed_time(a):6.2f}  kernels {t0.elapsed_time(b):6.2f}  d2h {t0.elapsed_time(c):6.2f}")

for _ in range(3): step(False)
step(True)
