"""Generate tests/golden/ref_torch_blocks16.npz: the REAL ``PointTransformerLayer(16, 16, 8, 36)`` of the reference
(models/modules/cbl_point_transformer/blocks.py:14-44) -- the boundary network's first level (train_configs/tgnet_bdl.py:
planes [16, 32], nsample [36, 24]) -- run on CPU as make_ref_blocks_golden.py runs the c = 32 / 64 layers: two packed arches,
randomised BatchNorm affine and running statistics, train() and eval() outputs, the state_dict, and the running statistics the
train() call leaves.

    python tests/golden/make_ref_blocks16_golden.py
"""
import os
import sys
import warnings

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
from make_ref_blocks_golden import cpu_cuda_shims, randomize_bn  # noqa: E402
from oracle import ref_models  # noqa: E402
from toothgroupnetwork_b200 import clouds  # noqa: E402

C, K = 16, 36


def blocks16_fixture():
    warnings.filterwarnings("ignore")
    cpu_cuda_shims()
    w = ref_models.World("reference", cpu_dry_run=True)
    fix = {}
    gen = torch.Generator().manual_seed(16)
    p = torch.cat([clouds.dental_arch(420, 13)[0], clouds.dental_arch(280, 14)[0]]).contiguous()
    o = torch.tensor([420, 700], dtype=torch.int32)
    fix["p"], fix["o"] = p.numpy(), o.numpy()
    with w, torch.no_grad():
        B = w.mod("models.modules.cbl_point_transformer.blocks")
        torch.manual_seed(C)
        layer = B.PointTransformerLayer(C, C, 8, K)
        randomize_bn(layer, gen)
        x = torch.randn(700, C, generator=gen)
        tag = f"ptl{C}"
        fix[tag + "_x"] = x.numpy()
        fix[tag + "_K"] = np.int64(K)
        for k, v in layer.state_dict().items():
            fix[f"{tag}_state_{k}"] = v.clone().numpy()
        state = {k: v.clone() for k, v in layer.state_dict().items()}
        fix[tag + "_out_train"] = layer.train()([p, x, o]).numpy()
        for k, v in layer.state_dict().items():
            if "running" in k:
                fix[f"{tag}_after_{k}"] = v.clone().numpy()      # .numpy() alone would alias the live buffer
        layer.load_state_dict(state)
        fix[tag + "_out_eval"] = layer.eval()([p, x, o]).numpy()
    out = os.path.join(HERE, "ref_torch_blocks16.npz")
    np.savez_compressed(out, **fix)
    print(out, os.path.getsize(out), "bytes")


if __name__ == "__main__":
    blocks16_fixture()
