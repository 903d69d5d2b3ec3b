#!/usr/bin/env python
"""Golden vectors of the reference's centred MelGANGenerator for the lookahead stream (TEST INFRASTRUCTURE): the shapes
of ``melgan_small`` with the two pads that fixture does not cover, and a small centred multi-band MelGAN with its PQMF
and odd scales.  Run against the REAL reference in the build container (needs the reference checkout), with the
fixture layout and ``gen`` of ``oracle/make_golden_melgan_stream.py``; writes ``tests/golden/melgan_centred_*.npz``.

    python oracle/make_golden_melgan_lookahead_stream.py"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle.make_golden import import_reference  # noqa: E402
from oracle.make_golden_melgan_stream import MB, SMALL, gen  # noqa: E402

# melgan_small's shapes (oracle/make_golden.py) and a small multi-band model with an odd scale, both centred
SMALL_CENTRED = dict(SMALL, use_causal_conv=False, use_final_nonlinear_activation=False)
MB_CENTRED = dict(MB, upsample_scales=[3, 4, 2], use_causal_conv=False)


def main():
    import_reference()
    gen("melgan_centred_replicate", dict(SMALL_CENTRED, pad="ReplicationPad1d"), B=2, T=20, seed=27, gain=1.2)
    gen("melgan_centred_zero", dict(SMALL_CENTRED, pad="ConstantPad1d", pad_params={"value": 0.0}), B=2, T=20, seed=28, gain=1.2)
    gen("melgan_centred_mb", MB_CENTRED, B=2, T=16, seed=29, gain=1.0, subbands=4)


if __name__ == "__main__":
    main()
