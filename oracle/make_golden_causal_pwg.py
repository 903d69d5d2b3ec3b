#!/usr/bin/env python
"""Golden vectors of the reference's causal ParallelWaveGANGenerator and of ResidualParallelWaveGANDiscriminator
(TEST INFRASTRUCTURE), run against the REAL reference in the build container (needs the reference checkout); writes
``tests/golden/pwg_causal_*.npz`` and ``tests/golden/rpwgd_*.npz``.

    python oracle/make_golden_causal_pwg.py

Same fixture layout as ``oracle/make_golden.py`` (kwargs, state-dict spec with weight norm, (seed, gain) of the
synthetic weights and their checksum, the seeded inputs' (shape, seed)); all outputs are eval-mode: generators store
``forward`` (``y``), ``inference`` on utterance 0 (``y_inf``) and the upsampled conditioning, discriminators the
fingerprint of ``forward`` and its full output (``final0``)."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle.make_golden import gen_discriminator, gen_pwg, import_reference  # noqa: E402

# test/test_parallel_wavegan.py:31-52 generator shapes with the causal rows of its grids (:137-141, :304-358)
SMALL = dict(in_channels=1, out_channels=1, kernel_size=3, layers=6, stacks=3, residual_channels=8, gate_channels=16,
             skip_channels=8, aux_channels=10, aux_context_window=0, dropout=0.05, use_weight_norm=True, use_causal_conv=True,
             upsample_conditional_features=True, upsample_net="ConvInUpsampleNetwork", upsample_params={"upsample_scales": [4, 4]})
# egs/ljspeech/voc1/conf/parallel_wavegan.v1.yaml:28-46 with use_causal_conv
V1 = dict(SMALL, layers=30, stacks=3, residual_channels=64, gate_channels=128, skip_channels=64, aux_channels=80,
          aux_context_window=2, dropout=0.0, upsample_params={"upsample_scales": [4, 4, 4, 4]})


def main():
    import_reference()
    for acw in range(4):
        gen_pwg(f"pwg_causal_small_acw{acw}", dict(SMALL, aux_context_window=acw), B=2, frames=24, seed=70 + acw, gain=1.0)
    gen_pwg("pwg_causal_small_upnet", dict(SMALL, upsample_net="UpsampleNetwork"), B=2, frames=24, seed=74, gain=1.0)
    gen_pwg("pwg_causal_v1", V1, B=2, frames=40, seed=75, gain=1.0)
    # WaveNet's classic causal kernel size 2, one stack of 10 layers (dilations 1 .. 512)
    gen_pwg("pwg_causal_k2", dict(V1, kernel_size=2, layers=10, stacks=1, upsample_params={"upsample_scales": [4, 4, 4]}),
            B=2, frames=24, seed=76, gain=1.0)
    melup = dict(SMALL, aux_context_window=0, upsample_net="MelGANGenerator",
                 upsample_params=dict(upsample_scales=[4, 4], in_channels=10, out_channels=10, channels=32, kernel_size=7, stacks=2))
    gen_pwg("pwg_causal_melgan_up", melup, B=2, frames=24, seed=77, gain=1.0)
    # models/parallel_wavegan.py:374-513
    gen_discriminator("rpwgd_default", "ResidualParallelWaveGANDiscriminator", {}, B=2, T=3000, seed=78, gain=1.2)
    gen_discriminator("rpwgd_causal", "ResidualParallelWaveGANDiscriminator",
                      dict(layers=6, stacks=2, use_causal_conv=True, dropout=0.1), B=2, T=2000, seed=79, gain=1.2)
    gen_discriminator("rpwgd_small", "ResidualParallelWaveGANDiscriminator",
                      dict(kernel_size=5, layers=4, stacks=2, residual_channels=32, gate_channels=64, skip_channels=32, bias=False,
                           nonlinear_activation_params={"negative_slope": 0.1}), B=3, T=777, seed=80, gain=1.2)


if __name__ == "__main__":
    main()
