"""FPS 24000->1024 (and ->4096 at B=1): old three-barrier bucket schedule against the single-barrier one, per batch size and warps per cloud."""
import sys, json, torch
sys.path.insert(0, "."); sys.path.insert(0, "scripts")
import op_bench
from toothgroupnetwork_b200 import pointops
rows = []
for B in (1, 16, 132, 264, 528, 1056):
    feats = op_bench.arch_batch(B, 24000)
    xyz = feats[:, :3].permute(0, 2, 1).contiguous().view(-1, 3)
    off = (torch.arange(1, B + 1, dtype=torch.int32) * 24000).cuda()
    for M in ((1024, 4096) if B == 1 else (1024,)):
        noff = (torch.arange(1, B + 1, dtype=torch.int32) * M).cuda()
        ref = pointops.fps_packed(xyz, off, noff, 24000, B * M, -2)
        row = {"clouds": B, "m": M}
        for mode in (-2, -14, -18, -26, -44, -48, -56, -72, -84, -88, -96, -112):
            try:
                t = op_bench.time_ms(lambda: pointops.fps_packed(xyz, off, noff, 24000, B * M, mode), warm=1, reps=3)
                same = bool(torch.equal(pointops.fps_packed(xyz, off, noff, 24000, B * M, mode), ref))
                row[str(mode)] = round(t, 3) if same else "MISMATCH"
            except Exception as e:
                row[str(mode)] = "err"
        rows.append(row)
        print(row, flush=True)
json.dump(rows, open("gpurun_out/fps_modes.json", "w"), indent=1)
