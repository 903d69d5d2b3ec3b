#!/usr/bin/env python
"""Golden vectors of the reference's causal MelGANGenerator with the pads the reflect-padded ``melgan_causal`` fixture
does not cover, and of a causal multi-band MelGAN with its PQMF (TEST INFRASTRUCTURE), run against the REAL reference in
the build container (needs the reference checkout); writes ``tests/golden/melgan_causal_*.npz``.

    python oracle/make_golden_melgan_stream.py

Same fixture layout as ``oracle/make_golden.py`` (kwargs, state-dict spec with weight norm, (seed, gain) of the
synthetic weights and their checksum, the seeded inputs' (shape, seed)).  Each fixture stores eval-mode ``forward``
(``y``, the subbands for the multi-band model) and ``inference`` of utterance 0 (``y_inf``, after the PQMF synthesis
for the multi-band model)."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from oracle import synth  # noqa: E402
from oracle.make_golden import import_reference, load_synth, save  # noqa: E402

# the reference unit-test shapes of oracle/make_golden.py's melgan_causal, with the other two pads
SMALL = dict(in_channels=80, out_channels=1, kernel_size=7, channels=32, upsample_scales=[4, 4], stack_kernel_size=3, stacks=2,
             use_weight_norm=True, use_final_nonlinear_activation=True, use_causal_conv=True)
# a small causal multi-band MelGAN: 4 subbands, three levels, reflect padding (the default), PQMF defaults (62 taps)
MB = dict(in_channels=80, out_channels=4, kernel_size=7, channels=64, upsample_scales=[4, 4, 2], stack_kernel_size=3, stacks=3,
          use_weight_norm=True, use_causal_conv=True)


def gen(name, kwargs, B, T, seed, gain, subbands=None):
    from parallel_wavegan.layers import PQMF
    from parallel_wavegan.models import MelGANGenerator

    torch.manual_seed(0)
    m = MelGANGenerator(**kwargs).eval()
    spec, sd = load_synth(m, seed, gain)
    c = synth.randn((B, kwargs.get("in_channels", 80), T), seed + 1)
    with torch.no_grad():
        y = m(c)
        if subbands:
            m.pqmf = PQMF(subbands)
        y_inf = m.inference(c[0].t())
    meta = dict(kind="melgan_generator", kwargs=kwargs, spec=spec, seed=seed, gain=gain, checksum=synth.checksum(sd),
                c_shape=list(c.shape), c_seed=seed + 1, pqmf_subbands=subbands)
    print("   out std %.3f absmax %.3f" % (y_inf.std(), y_inf.abs().max()))
    save(name, meta, y=y, y_inf=y_inf)


def main():
    import_reference()
    gen("melgan_causal_replicate", dict(SMALL, pad="ReplicationPad1d"), B=2, T=20, seed=24, gain=1.2)
    gen("melgan_causal_zero", dict(SMALL, pad="ConstantPad1d", pad_params={"value": 0.0}), B=2, T=20, seed=25, gain=1.2)
    gen("melgan_causal_mb", MB, B=2, T=16, seed=26, gain=1.0, subbands=4)


if __name__ == "__main__":
    main()
