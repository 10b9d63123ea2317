"""Generate tests/golden/ref_torch_decoder.npz: the REAL ``TransitionUp`` (both forms) and ``MultiHead`` of the reference
(models/modules/cbl_point_transformer/blocks.py:82-111, heads.py:13-61), imported from the reference checkout and run on CPU
with pointops served by the oracle's C restatement, in train() and eval() BatchNorm mode, with each module's full
``state_dict``, the running statistics after the train() step, and the neighbour indices / weights pointops.interpolation used.

    python tests/golden/make_ref_decoder_golden.py
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
from oracle import oracle as O  # noqa: E402
from oracle import ref_models  # noqa: E402
from toothgroupnetwork_b200 import clouds  # noqa: E402


class Cfg(dict):
    """the attribute-and-membership access of the reference's CfgNode"""
    __getattr__ = dict.get


def _run(fix, tag, module, call):
    for k, v in module.state_dict().items():
        fix[f"{tag}_state_{k}"] = v.clone().numpy()
    state = {k: v.clone() for k, v in module.state_dict().items()}
    out = call(module.train())
    fix[tag + "_out_train"] = out[0].numpy()
    for i, extra in enumerate(out[1:]):
        fix[f"{tag}_extra{i}_train"] = extra.numpy()
    for k, v in module.state_dict().items():
        if "running" in k or "num_batches" in k:
            fix[f"{tag}_after_{k}"] = v.clone().numpy()
    module.load_state_dict(state)
    out = call(module.eval())
    fix[tag + "_out_eval"] = out[0].numpy()
    for i, extra in enumerate(out[1:]):
        fix[f"{tag}_extra{i}_eval"] = extra.numpy()


def main():
    warnings.filterwarnings("ignore")
    cpu_cuda_shims()
    w = ref_models.World("reference", cpu_dry_run=True)
    gen = torch.Generator().manual_seed(3)
    fix = {}
    # two clouds of different sizes at the fine level, every 4th point at the coarse one
    p1 = torch.cat([clouds.dental_arch(400, 1)[0], clouds.dental_arch(400, 2)[0]]).contiguous()
    o1 = torch.tensor([400, 800], dtype=torch.int32)
    p2 = torch.cat([p1[:400:4], p1[400::4]]).contiguous()
    o2 = torch.tensor([100, 200], dtype=torch.int32)
    fix["p1"], fix["o1"], fix["p2"], fix["o2"] = p1.numpy(), o1.numpy(), p2.numpy(), o2.numpy()
    idx, dist, _ = O.knnquery(3, p2.numpy(), p1.numpy(), o2.numpy(), o1.numpy())
    rec = 1.0 / (torch.from_numpy(dist) + 1e-8)
    fix["interp_idx"], fix["interp_w"] = idx, (rec / rec.sum(1, keepdim=True)).numpy()
    nn1, _, _ = O.knnquery(1, p2.numpy(), p1.numpy(), o2.numpy(), o1.numpy())
    fix["nn1"] = nn1
    with w, torch.no_grad():
        B = w.mod("models.modules.cbl_point_transformer.blocks")
        H = w.mod("models.modules.cbl_point_transformer.heads")
        torch.manual_seed(11)
        tu = B.TransitionUp(64, 32)
        randomize_bn(tu, gen)
        x1, x2 = torch.randn(800, 32, generator=gen), torch.randn(200, 64, generator=gen)
        fix["tu_x1"], fix["tu_x2"] = x1.numpy(), x2.numpy()
        _run(fix, "tu", tu, lambda m: (m([p1, x1, o1], [p2, x2, o2]),))
        torch.manual_seed(12)
        th = B.TransitionUp(32, None)
        randomize_bn(th, gen)
        xh = torch.randn(800, 32, generator=gen) + 0.5
        fix["th_x"] = xh.numpy()
        _run(fix, "th", th, lambda m: (m([p1, xh, o1]),))
        torch.manual_seed(13)
        config = Cfg(num_layers=2, base_fdim=32, num_classes=5)
        mh = H.MultiHead([32, 64], Cfg(stage="Ua", ftype="latent", combine="concat"), config, k=5)
        randomize_bn(mh, gen)
        f0, f1 = torch.randn(800, 32, generator=gen), torch.randn(200, 64, generator=gen)
        fix["mh_f0"], fix["mh_f1"] = f0.numpy(), f1.numpy()

        def head(m):
            stages = {"up": [{"p_out": p1, "f_out": f0, "offset": o1}, {"p_out": p2, "f_out": f1, "offset": o2}]}
            out, stages = m(stages)
            return out, stages["up"][0]["latent"], stages["up"][1]["latent"]

        _run(fix, "mh", mh, head)
    out = os.path.join(HERE, "ref_torch_decoder.npz")
    np.savez_compressed(out, **fix)
    print(out, os.path.getsize(out), "bytes")


if __name__ == "__main__":
    main()
