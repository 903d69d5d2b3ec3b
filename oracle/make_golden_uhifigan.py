#!/usr/bin/env python
"""Golden vectors of the reference's UHiFiGANGenerator (TEST INFRASTRUCTURE), run against the REAL reference in the
build container (needs ``/root/reference``); writes ``tests/golden/uhifigan_*.npz``.

    python oracle/make_golden_uhifigan.py

Each fixture stores the constructor kwargs, the state-dict spec (with weight norm), the (seed, gain) of the
synthetic weights and their checksum, the seeded inputs' (shape, seed), and the eval-mode outputs of ``forward``
(``y``) and of ``inference`` on utterance 0 (``y_inf``)."""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import synth  # noqa: E402
from oracle.make_golden import import_reference, load_synth, save  # noqa: E402

# egs/opencpop/voc1/conf/uhifigan.v1.yaml generator_params
OPENCPOP = dict(in_channels=80, out_channels=1, channels=32, kernel_size=7, downsample_scales=[5, 5, 4, 3],
                downsample_kernel_sizes=[10, 10, 8, 6], upsample_scales=[3, 4, 5, 5], upsample_kernel_sizes=[6, 8, 10, 10],
                resblock_kernel_sizes=[3, 7, 11], resblock_dilations=[[1, 3, 5], [1, 3, 5], [1, 3, 5]], dropout=0.1,
                use_additional_convs=True, bias=True, nonlinear_activation="LeakyReLU",
                nonlinear_activation_params={"negative_slope": 0.1}, use_weight_norm=True)


def gen_uhifigan(name, kwargs, B, frames, seed, gain):
    from parallel_wavegan.models import UHiFiGANGenerator

    torch.manual_seed(0)
    m = UHiFiGANGenerator(**kwargs).eval()
    spec, sd = load_synth(m, seed, gain)
    hop = 1
    for s in kwargs["upsample_scales"]:
        hop *= s
    c = synth.randn((B, kwargs.get("in_channels", 80), frames), seed + 1)
    f0 = synth.randn((B, 1, frames), seed + 2)
    e = synth.randn((B, 1, frames * hop), seed + 3, 0.3)
    with torch.no_grad():
        y = m(c, f0, e)
        y_inf = m.inference(excitation=e[0].reshape(frames, hop), f0=f0[0, 0], c=c[0].t())
    meta = dict(kind="uhifigan_generator", kwargs=kwargs, spec=spec, seed=seed, gain=gain, checksum=synth.checksum(sd),
                c_shape=list(c.shape), c_seed=seed + 1, f0_shape=list(f0.shape), f0_seed=seed + 2, e_shape=list(e.shape),
                e_seed=seed + 3, e_scale=0.3, hop=hop)
    print("   out std %.3f absmax %.3f" % (y.std(), y.abs().max()))
    save(name, meta, y=y, y_inf=y_inf)


def main():
    import_reference()
    small = dict(OPENCPOP, channels=32, downsample_scales=[2, 2, 2, 2], downsample_kernel_sizes=[4, 4, 4, 4],
                 upsample_scales=[2, 2, 2, 2], upsample_kernel_sizes=[4, 4, 4, 4])
    gen_uhifigan("uhifigan_small", small, B=2, frames=12, seed=81, gain=1.15)
    gen_uhifigan("uhifigan_opencpop", OPENCPOP, B=2, frames=40, seed=82, gain=1.15)
    # odd scales: output_padding = 1 on every decoder level; two MRF blocks, no additional convs, no bias
    odd = dict(OPENCPOP, channels=32, downsample_scales=[3, 5], downsample_kernel_sizes=[6, 10], upsample_scales=[5, 3],
               upsample_kernel_sizes=[10, 6], resblock_kernel_sizes=[3, 5], resblock_dilations=[[1, 3], [1, 2]],
               use_additional_convs=False, bias=False)
    gen_uhifigan("uhifigan_odd", odd, B=2, frames=9, seed=83, gain=1.3)


if __name__ == "__main__":
    main()
