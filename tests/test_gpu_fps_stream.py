"""The three-barrier bucket FPS kernel (fps_bucket_kernel, the large-batch path the benchmark runs) on every FPS case at every
CTA width, and one auto-mode launch large enough to select it: idx AND the final running minima bitwise those of the oracle."""
import numpy as np
import pytest
import torch

from oracle import oracle
from toothgroupnetwork_b200 import _lib as L
from toothgroupnetwork_b200 import clouds, pointops

from test_gpu_pointops import FPS_CASES, _pack, i32

pytestmark = pytest.mark.gpu


def _fps_with_tmp(xyz, offset, new_offset, n_max, mode):
    x, o, no = xyz.cuda().contiguous(), i32(offset), i32(new_offset)
    idx = torch.zeros(int(new_offset[-1]), dtype=torch.int32, device="cuda")
    tmp = torch.full((xyz.shape[0],), 1e10, dtype=torch.float32, device="cuda")
    L.call("tgn_furthestsampling", len(offset), int(n_max), L.ptr(x), L.ptr(o), L.ptr(no), L.ptr(tmp), L.ptr(idx), int(mode),
           L.stream_ptr())
    torch.cuda.synchronize()
    return idx.cpu().numpy(), tmp.cpu().numpy()


@pytest.mark.parametrize("name,build,ms", FPS_CASES, ids=[c[0] for c in FPS_CASES])
@pytest.mark.parametrize("mode", [-11, -12, -14, -18, -26])   # -(10 + W): W warps per cloud
def test_three_barrier_kernel_idx_and_tmp(name, build, ms, mode):
    cl = build()
    xyz, offset, new_offset = _pack(cl, ms)
    n_max = max(c.shape[0] for c in cl)
    want_idx, want_tmp = oracle.furthestsampling(xyz.numpy(), offset, new_offset, return_tmp=True)
    got_idx, got_tmp = _fps_with_tmp(xyz, offset, new_offset, n_max, mode)
    assert np.array_equal(got_idx, want_idx)
    assert np.array_equal(got_tmp.view(np.uint32), want_tmp.view(np.uint32))


def test_auto_large_batch_selects_three_barrier_kernel():
    """More than 4 clouds per SM: auto takes fps_bucket_kernel<128>.  Every cloud against the single-barrier register kernel
    (mode -84), a seeded sample against the oracle; duplicated-vertex clouds in the mix take the tie path all the time."""
    n, m = 24000, 1024
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    b = 4 * sms + 8
    base = [clouds.dental_arch(n, s)[0] for s in range(6)]
    base += [clouds.with_duplicates(clouds.dental_arch(n // 2, 20 + s)[0], 20 + s) for s in range(2)]
    cl = [base[j % len(base)] for j in range(b)]
    xyz = torch.cat(cl, 0).cuda().contiguous()
    off = i32(np.arange(1, b + 1) * n)
    noff = i32(np.arange(1, b + 1) * m)
    got = pointops.fps_packed(xyz, off, noff, n, b * m, 0)
    ref = pointops.fps_packed(xyz, off, noff, n, b * m, -84)
    torch.cuda.synchronize()
    assert torch.equal(got, ref)
    got = got.cpu().numpy()
    rng = np.random.default_rng(0)
    for j in sorted(rng.choice(b, 4, replace=False).tolist()) + [6, 7]:
        want = oracle.furthestsampling(cl[j].numpy(), np.array([n], np.int32), np.array([m], np.int32))
        assert np.array_equal(got[j * m:(j + 1) * m] - j * n, want), f"cloud {j}"
