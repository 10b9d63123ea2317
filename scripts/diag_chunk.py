"""How long does one chunk of the host pipeline take?  Times the module forward on one 132-cloud chunk alone, with a
concurrent H2D copy stream, and stage by stage."""
import sys, torch
sys.path.insert(0, ".")
import bench
from toothgroupnetwork_b200 import pointnet2_utils as pn2
B = 132
sa = bench.build_module("cuda")
host = bench.make_clouds(0, 1056).pin_memory()
feats = host[:B].cuda()
xyz = feats[:, :3].contiguous()
ev = lambda: torch.cuda.Event(enable_timing=True)

def timed(fn, reps=5):
    for _ in range(2): fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = ev(), ev(); a.record(); fn(); b.record(); torch.cuda.synchronize(); ts.append(a.elapsed_time(b))
    return sorted(ts)[len(ts) // 2]

with torch.no_grad():
    print("module forward B=148 alone: %.3f ms" % timed(lambda: sa(xyz, feats)))
    for mode in (0, -14, -18, -26):
        pn2.set_fps_mode(mode)
        print("  fps mode %d: %.3f ms" % (mode, timed(lambda: sa(xyz, feats))))
    pn2.set_fps_mode(0)
    xyz_t = pn2.transpose_last2(xyz); feats_t = pn2.transpose_last2(feats)
    print("transposes %.3f" % timed(lambda: (pn2.transpose_last2(xyz), pn2.transpose_last2(feats))))
    print("slice+contiguous %.3f" % timed(lambda: feats[:, :3].contiguous()))
    fps = pn2._fps_batched(xyz_t, 1024)
    print("fps %.3f" % timed(lambda: pn2._fps_batched(xyz_t, 1024)))
    new_xyz_t = pn2._take_rows(xyz_t.view(-1, 3), fps).view(B, 1024, 3)
    print("ball %.3f" % timed(lambda: pn2._ball_query(0.1, 32, xyz_t, new_xyz_t, False, None, 1)))
    gidx = pn2._ball_query(0.1, 32, xyz_t, new_xyz_t, False, None, 1)
    folded = sa._folded.update(sa.mlp_convs, sa.mlp_bns)
    out = torch.empty((B, 64, 1024), device="cuda")
    print("mlp %.3f" % timed(lambda: pn2.sa_group_mlp_max(xyz_t, feats_t, new_xyz_t, gidx, True, folded, out, 0)))
    # with a concurrent H2D stream
    cs = torch.cuda.Stream()
    dev = torch.empty_like(host, device="cuda")
    def with_copy():
        cs.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(cs):
            dev.copy_(host, non_blocking=True)
        sa(xyz, feats)
    print("module forward with a concurrent 682 MB H2D: %.3f ms (includes nothing of the copy)" % timed(with_copy))
    def fwd_only_during_copy():
        with torch.cuda.stream(cs):
            dev.copy_(host, non_blocking=True)
        a, b = ev(), ev(); a.record(); sa(xyz, feats); b.record(); torch.cuda.synchronize(); return a.elapsed_time(b)
    print("forward while the copy runs: %s" % [round(fwd_only_during_copy(), 3) for _ in range(4)])
    def fps_during_copy():
        with torch.cuda.stream(cs):
            dev.copy_(host, non_blocking=True)
        a, b = ev(), ev(); a.record(); pn2._fps_batched(xyz_t, 1024); b.record(); torch.cuda.synchronize(); return a.elapsed_time(b)
    print("fps while the copy runs: %s" % [round(fps_during_copy(), 3) for _ in range(4)])
