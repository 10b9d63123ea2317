#!/usr/bin/env python
"""Pin the arithmetic of DGCNN's feature-space kNN (models/modules/dgcnn.py:4-10) on this GPU (DESIGN §3.11).

    inner = -2*torch.matmul(x.transpose(2, 1), x); xx = torch.sum(x**2, dim=1, keepdim=True)
    pairwise_distance = -xx - inner - xx.transpose(2, 1); idx = pairwise_distance.topk(k=k, dim=-1)[1]

1. The two subtractions: v_ij = fl(fl(-xx_j + 2 dot_ij) - xx_i), checked against torch's own pairwise_distance over all N^2 pairs
   (and -2 * matmul against matmul, to show the scaling is exact).
2. dot_ij of cuBLAS (FP32, matmul precision "highest") against candidate orders over all N^2 pairs: the sequential FFMA chain from
   a product, the same from +0, 2-/4-/8-way sliced-K partial sums (contiguous slices, chains summed in slice order), and unfused
   multiply-then-add.  C in {6, 64}, N in {4096, 24000}, B in {1, 2}, on both layouts the model passes: a permute(0, 2, 1) view of
   a (B, N, C) tensor and a contiguous (B, C, N) tensor.  The candidates run in a small CUDA helper compiled here with nvcc.
3. topk's selection and order against the rule the kernel implements (topk_rule), on tie-heavy inputs: the k largest by torch's
   radix key (-0 < +0, NaN largest), lower index first among equal keys; then the selection in gather order (the values above
   the k-th key in index order, then those equal to it) through torch's bitonic sort of 32 entries.  For comparison, the rows
   where a stable order (equal values by index) would differ, and the rows whose index *sets* differ.

Prints one JSON object with the card's name and power limit, and also writes it to the file given by --out.
"""
import argparse
import ctypes
import json
import os
import shutil
import subprocess
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from toothgroupnetwork_b200 import clouds  # noqa: E402

CANDIDATES = ["seq_from_product", "seq_from_zero", "sliced2", "sliced4", "sliced8", "unfused"]
HELPER = r"""
#include <cstdint>
__device__ float chain(const float* a, long long sa, const float* b, long long sb, int c0, int c1, bool from_zero, bool fused) {
    float acc = from_zero ? 0.0f : __fmul_rn(a[c0 * sa], b[c0 * sb]);
    for (int c = from_zero ? c0 : c0 + 1; c < c1; ++c)
        acc = fused ? __fmaf_rn(a[c * sa], b[c * sb], acc) : __fadd_rn(acc, __fmul_rn(a[c * sa], b[c * sb]));
    return acc;
}
__device__ float sliced(const float* a, long long sa, const float* b, long long sb, int C, int S) {
    const int w = (C + S - 1) / S;
    float tot = 0.0f;
    bool first = true;
    for (int s = 0; s < S; ++s) {
        const int c0 = s * w, c1 = min(C, c0 + w);
        if (c0 >= c1) continue;
        const float p = chain(a, sa, b, sb, c0, c1, false, true);
        tot = first ? p : __fadd_rn(tot, p);
        first = false;
    }
    return tot;
}
// x: element (b, c, n) at b*sb_ + c*sc + n*sn; ref: (B, N, N) contiguous cuBLAS dot products; counts[6] mismatches
extern "C" __global__ void diag_kernel(int B, int N, int C, const float* x, long long sb_, long long sc, long long sn,
                                       const float* ref, unsigned long long* counts) {
    const long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (t >= (long long)B * N * N) return;
    const int b = (int)(t / ((long long)N * N)), i = (int)(t / N % N), j = (int)(t % N);
    const float* a = x + b * sb_ + i * sn;
    const float* q = x + b * sb_ + j * sn;
    const uint32_t r = __float_as_uint(ref[t]);
    float v[6];
    v[0] = chain(a, sc, q, sc, 0, C, false, true);
    v[1] = chain(a, sc, q, sc, 0, C, true, true);
    v[2] = sliced(a, sc, q, sc, C, 2);
    v[3] = sliced(a, sc, q, sc, C, 4);
    v[4] = sliced(a, sc, q, sc, C, 8);
    v[5] = chain(a, sc, q, sc, 0, C, false, false);
    for (int m = 0; m < 6; ++m)
        if (__float_as_uint(v[m]) != r) atomicAdd(counts + m, 1ull);
}
extern "C" int diag_launch(int B, int N, int C, const float* x, long long sb, long long sc, long long sn, const float* ref,
                           unsigned long long* counts) {
    const long long total = (long long)B * N * N;
    diag_kernel<<<(unsigned)((total + 255) / 256), 256>>>(B, N, C, x, sb, sc, sn, ref, counts);
    return (int)cudaDeviceSynchronize();
}
"""


def _helper() -> ctypes.CDLL:
    d = tempfile.mkdtemp(prefix="diag_dgcnn_knn_")
    src, so = os.path.join(d, "h.cu"), os.path.join(d, "h.so")
    with open(src, "w") as f:
        f.write(HELPER)
    subprocess.check_call([shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc", "-O3", "-gencode", "arch=compute_90a,code=sm_90a", "-Xcompiler", "-fPIC", "-shared", src,
                           "-o", so])
    lib = ctypes.CDLL(so)
    ll = ctypes.c_longlong
    lib.diag_launch.argtypes = [ctypes.c_int] * 3 + [ctypes.c_void_p, ll, ll, ll, ctypes.c_void_p, ctypes.c_void_p]
    return lib


def features(B: int, N: int, C: int, layout: str, seed: int = 0) -> torch.Tensor:
    """(B, C, N) cuda float32 in one of the model's two layouts.  C = 6: [xyz; normal] of an arch; C = 64: a seeded LeakyReLU
    projection of it, the kind of features DGCNN's later layers search in."""
    f6 = torch.cat([clouds.arch_features(N, seed + b) for b in range(B)])                   # (B, 6, N)
    if C == 6:
        x = f6
    else:
        g = torch.Generator().manual_seed(seed + 17)
        w = torch.randn(C, 6, generator=g) * 2.0
        x = torch.nn.functional.leaky_relu(torch.einsum("oc,bcn->bon", w, f6) + 0.1 * torch.randn(B, C, N, generator=g), 0.2)
    x = x.cuda()
    return x.transpose(1, 2).contiguous().permute(0, 2, 1) if layout == "permuted" else x.contiguous()


def reference(x: torch.Tensor, k: int):
    inner = -2 * torch.matmul(x.transpose(2, 1), x)
    xx = torch.sum(x ** 2, dim=1, keepdim=True)
    pd = -xx - inner - xx.transpose(2, 1)
    return pd, pd.topk(k=k, dim=-1)


def main(out_path=None) -> None:
    torch.backends.cuda.matmul.allow_tf32 = False
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    out = {"gpu": q.stdout.strip(), "torch": torch.__version__, "dot": {}, "subtractions": {}, "topk": {}}
    lib = _helper()
    counts = torch.zeros(len(CANDIDATES), dtype=torch.int64, device="cuda")
    for C in (6, 64):
        for N in (4096, 24000):
            for B in (1, 2):
                for layout in ("permuted", "contiguous"):
                    x = features(B, N, C, layout)
                    dot = torch.matmul(x.transpose(2, 1), x)
                    counts.zero_()
                    rc = lib.diag_launch(B, N, C, x.data_ptr(), x.stride(0), x.stride(1), x.stride(2), dot.data_ptr(),
                                         counts.data_ptr())
                    assert rc == 0, rc
                    key = f"C{C}_N{N}_B{B}_{layout}"
                    out["dot"][key] = dict(zip(CANDIDATES, counts.tolist()), pairs=B * N * N)
                    # the two subtractions on torch's own inner, and the exactness of the -2 scaling
                    inner = -2 * dot
                    xx = torch.sum(x ** 2, dim=1, keepdim=True)
                    pd = -xx - inner - xx.transpose(2, 1)
                    t = -xx + 2.0 * dot                                                   # fl(-xx_j + 2 dot_ij)
                    v = t - xx.transpose(2, 1)                                            # fl(t - xx_i)
                    out["subtractions"][key] = {
                        "v_mismatch": int((v.view(torch.int32) != pd.view(torch.int32)).sum()),
                        "scaling_mismatch": int(((inner / -2).view(torch.int32) != dot.view(torch.int32)).sum())}
                    del dot, inner, pd, t, v
                    torch.cuda.empty_cache()
    # selection and order on tie-heavy inputs
    g = torch.Generator().manual_seed(3)
    xyz = clouds.dental_arch(2048, 3)[0]
    dup = clouds.with_duplicates(xyz, 3)                                                           # (4096, 3)
    lattice = torch.randint(-3, 4, (1, 64, 4096), generator=g).float()
    zeros = torch.randn(1, 6, 4096, generator=g)
    zeros[:, :, torch.randperm(4096, generator=g)[:1500]] = 0.0
    negz = zeros.clone()
    negz[:, :, :64] = -0.0
    tie_inputs = {
        "duplicates_C3": dup.t().unsqueeze(0).contiguous().cuda(),
        "duplicates_C6_permuted": torch.cat([dup, dup], 1).unsqueeze(0).cuda().permute(0, 2, 1),
        "lattice_C64": lattice.cuda(),
        "lattice_C6": lattice[:, :6].contiguous().cuda(),
        "zero_vectors_C6": zeros.cuda(),
        "negative_zero_C6": negz.cuda(),
    }
    for name, x in tie_inputs.items():
        dot = torch.matmul(x.transpose(2, 1), x)
        counts.zero_()
        assert lib.diag_launch(1, x.shape[2], x.shape[1], x.data_ptr(), x.stride(0), x.stride(1), x.stride(2), dot.data_ptr(),
                               counts.data_ptr()) == 0
        out["dot"][name] = dict(zip(CANDIDATES, counts.tolist()), pairs=x.shape[2] ** 2)
        for k in (1, 20, 32):
            pd, (vals, idx) = reference(x, k)
            rule_v, rule_i = topk_rule(pd, k)
            out["topk"][f"{name}_k{k}"] = {
                "rows": int(pd.shape[0] * pd.shape[1]),
                "rows_with_kth_tie": int((pd == vals[..., -1:]).sum(-1).gt((vals == vals[..., -1:]).sum(-1)).sum()),
                "value_mismatch_rows": int((rule_v.view(torch.int32) != vals.view(torch.int32)).any(-1).sum()),
                "index_mismatch_rows": int((rule_i != idx).any(-1).sum()),
                "index_ascending_among_equal_values_mismatch_rows": int((_index_order(pd, k)[1] != idx).any(-1).sum()),
                "index_set_mismatch_rows": int((rule_i.sort(-1)[0] != idx.sort(-1)[0]).any(-1).sum()),
            }
    if out_path:
        with open(out_path, "w") as f:
            json.dump(out, f, indent=1)
    print(json.dumps(out, indent=1))


def radix_key(v: torch.Tensor) -> torch.Tensor:
    """torch's topk key of a float32 (TopKTypeConfig<float>::convert) as int64: order-preserving, -0 < +0, every NaN largest"""
    bits = v.view(torch.int32).long() & 0xFFFFFFFF
    key = torch.where(bits >= 0x80000000, bits ^ 0xFFFFFFFF, bits ^ 0x80000000)
    return torch.where(v != v, torch.full_like(key, 0xFFFFFFFF), key)


def topk_rule(pd: torch.Tensor, k: int):
    """The kernel's rule on a full (B, N, N) matrix: select by (key descending, index ascending); put the selection in gather
    order (above the k-th key in index order, then equal to it in index order); sort it by a bitonic network of 32 with the
    comparator a > b (NaN largest), as at::native::bitonicSortKVInPlace does."""
    n = pd.shape[-1]
    assert n <= 1 << 16
    cols = torch.arange(n, device=pd.device)
    key = radix_key(pd)
    sel = torch.topk(key * 65536 + (65535 - cols), k, dim=-1)[0]
    idx = 65535 - sel % 65536
    skey = sel // 65536
    above = (skey > skey[..., -1:]).long()
    order = torch.sort(idx, dim=-1, stable=True)[1]
    order = torch.gather(order, -1, torch.sort(torch.gather(above, -1, order), dim=-1, descending=True, stable=True)[1])
    idx = torch.gather(idx, -1, order)
    val = torch.gather(pd, -1, idx)
    if k == 1:
        return val, idx
    pad = 32 - k
    v = torch.cat([val, val.new_zeros(val.shape[:-1] + (pad,))], -1)
    i = torch.cat([idx, idx.new_zeros(idx.shape[:-1] + (pad,))], -1)
    ok = torch.cat([torch.ones_like(idx, dtype=torch.bool), torch.zeros(idx.shape[:-1] + (pad,), dtype=torch.bool,
                                                                                 device=idx.device)], -1)
    lanes = torch.arange(32, device=pd.device)
    steps = [(size, stride) for size in (2, 4, 8, 16) for stride in (size // 2, size // 4, size // 8, size // 16) if stride] + \
        [(32, s) for s in (16, 8, 4, 2, 1)]
    for size, stride in steps:
        a = lanes[(lanes & stride) == 0]
        bb = a + stride
        direction = ((a & size) != 0) if size < 32 else torch.zeros_like(a, dtype=torch.bool)
        va, vb, oka, okb = v[..., a], v[..., bb], ok[..., a], ok[..., bb]
        gt = (va.isnan() & ~vb.isnan()) | (va > vb)
        swap = ((gt & oka) | ~okb) == direction
        for t in (v, i, ok):
            ta, tb = t[..., a].clone(), t[..., bb].clone()
            t[..., a] = torch.where(swap, tb, ta)
            t[..., bb] = torch.where(swap, ta, tb)
    return v[..., :k], i[..., :k]


def _index_order(pd: torch.Tensor, k: int):
    """(value descending with +0 == -0, index ascending): the order a stable sort of an index-ordered slice gives"""
    order = torch.sort(pd, dim=-1, descending=True, stable=True)[1][..., :k]
    return torch.gather(pd, -1, order), order


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    main(ap.parse_args().out)
