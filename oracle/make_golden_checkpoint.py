"""Golden checkpoint written by the REAL reference (needs the reference tree): a tiny HiFi-GAN generator after one
reference RAdam step (bin/train.py checkpoint layout), plus the state-dict key / shape layout of the reference
generator and HiFi-GAN MSD/MPD discriminator.  tests/test_checkpoint_cpu.py rebuilds the checkpoint from this file
(the discriminator weights are the seeded synthetic fill, regenerated from the layout).

    python -m oracle.make_golden_checkpoint REFERENCE_ROOT
"""
import json
import os
import sys

import numpy as np
import torch

from oracle import synth
from oracle.make_golden import import_reference

# a tiny generator keeps the stored weights and optimizer state small; the layout rules are the same at every size
HIFI_TINY = dict(in_channels=8, out_channels=1, channels=8, kernel_size=7, upsample_scales=[4, 2],
                 upsample_kernel_sizes=[8, 4], resblock_kernel_sizes=[3, 5], resblock_dilations=[[1, 3], [1, 3]])
OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "checkpoint_ref.npz")


def main(ref_root):
    import_reference(ref_root)
    import parallel_wavegan.models as rm
    from parallel_wavegan.optimizers import RAdam

    rg, rd = rm.HiFiGANGenerator(**HIFI_TINY), rm.HiFiGANMultiScaleMultiPeriodDiscriminator()
    for m, seed in ((rg, 11), (rd, 12)):
        m.load_state_dict(synth.synth_state_dict([(k, tuple(v.shape)) for k, v in m.state_dict().items()], seed, 1.0))
    ro = RAdam(rg.parameters(), lr=1e-3)
    gen = torch.Generator().manual_seed(13)
    for p in rg.parameters():
        p.grad = torch.randn(p.shape, generator=gen) * 0.01
    ro.step()
    osd = ro.state_dict()
    arrays = {f"g/{k}": v.numpy() for k, v in rg.state_dict().items()}
    for i, st in osd["state"].items():
        arrays[f"exp_avg/{i}"] = st["exp_avg"].numpy()
        arrays[f"exp_avg_sq/{i}"] = st["exp_avg_sq"].numpy()
        arrays[f"step/{i}"] = np.asarray(float(st["step"]))
    groups = [{k: v for k, v in g.items() if k != "params"} | {"params": list(g["params"])} for g in osd["param_groups"]]
    meta = {"generator_params": HIFI_TINY,
            "g_spec": [(k, list(v.shape)) for k, v in rg.state_dict().items()],
            "d_spec": [(k, list(v.shape)) for k, v in rd.state_dict().items()],
            "param_groups": groups}
    arrays["meta"] = np.asarray(json.dumps(meta))
    np.savez_compressed(OUT, **arrays)
    print(OUT, os.path.getsize(OUT))


if __name__ == "__main__":
    main(*sys.argv[1:])
