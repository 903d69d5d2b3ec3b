#!/usr/bin/env python
"""Golden vectors of the reference's DiscreteSymbolStyleMelGANGenerator (TEST INFRASTRUCTURE), run against the REAL
reference in the build container (needs ``/root/reference``); writes ``tests/golden/dsym_style_*.npz``.

    python oracle/make_golden_dsym_style.py

Each fixture stores the constructor kwargs, the state-dict spec (with weight norm), the (seed, gain) of the synthetic
weights and their checksum, and:

* ``c``, ``z``: symbol / speaker indices (B, 2, T) and noise (B, in_channels, T / noise_upsample_factor); ``y`` =
  forward(c, z), ``x0`` its noise path, ``x1`` / ``c1`` the first 96 samples of its first block's outputs;
* per inference case k (``T = noise_upsample_factor * j`` and a T that is not a multiple of it): ``inf{k}_c`` (T, 2),
  the noise ``inf{k}_noise`` that inference drew (recorded by replaying the seed it was drawn under), ``inf{k}_y`` =
  inference(c), and for the last case ``inf{k}_y_g`` = inference(c[:, :1], g).

It also asserts the reference's failures that the mirror reproduces: forward with a T other than the noise length, and
``concat_spk_emb=True``."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import synth  # noqa: E402
from oracle.make_golden import import_reference, load_synth, save  # noqa: E402
from oracle.make_golden_discrete import _symbols  # noqa: E402

# egs/vctk/hubert_voc1/conf/style_melgan_hubert.v1.yaml generator_params
VCTK = dict(in_channels=128, aux_channels=128, channels=64, out_channels=1, num_embs=100, num_spk_embs=128, spk_emb_dim=128,
            concat_spk_emb=False, kernel_size=9, dilation=2, bias=True, noise_upsample_scales=[7, 2, 2, 2],
            noise_upsample_activation="LeakyReLU", noise_upsample_activation_params={"negative_slope": 0.2},
            upsample_scales=[5, 2, 2, 2, 2, 2, 2, 1, 1], upsample_mode="nearest", gated_function="softmax", use_weight_norm=True)
# a short noise path (x6), an odd scale, a scale-1 block, the sigmoid gate and a dilation of 3
SMALL = dict(VCTK, in_channels=16, aux_channels=24, channels=32, num_embs=10, num_spk_embs=4, spk_emb_dim=24, kernel_size=5,
             dilation=3, noise_upsample_scales=[3, 2], upsample_scales=[3, 1, 2], gated_function="sigmoid")


def _raises(fn, text):
    try:
        fn()
    except RuntimeError as e:
        assert text in str(e), str(e)
        return
    raise AssertionError(f"the reference did not fail with {text!r}")


def gen_dsym_style(name, kwargs, B, z_len, inf_lengths, g, seed, gain):
    from parallel_wavegan.models import DiscreteSymbolStyleMelGANGenerator

    torch.manual_seed(0)
    m = DiscreteSymbolStyleMelGANGenerator(**kwargs).eval()
    spec, sd = load_synth(m, seed, gain)
    f = int(np.prod(kwargs["noise_upsample_scales"]))
    rng = np.random.RandomState(seed)
    c = _symbols(rng, B, f * z_len, kwargs["num_embs"], kwargs["num_spk_embs"])
    z = synth.randn((B, kwargs["in_channels"], z_len), seed + 1)
    arrays = dict(c=c, z=z)
    with torch.no_grad():
        arrays["y"] = m(c, z)
        x0 = m.noise_upsample(z)
        e = m.emb(c[:, 0].long()).transpose(1, 2) + m.spk_emb(c[:, 1, 0].long()).unsqueeze(2)
        arrays["x0"] = x0
        x1, c1 = m.blocks[0](x0, e)
        arrays["x1"], arrays["c1"] = x1[:, :, :96], c1[:, :, :96]  # the first 96 samples keep the fixture small
        for k, T in enumerate(inf_lengths):
            ci = _symbols(rng, 1, T, kwargs["num_embs"], kwargs["num_spk_embs"])[0].t().contiguous()
            torch.manual_seed(seed + 10 + k)
            noise = torch.randn(1, kwargs["in_channels"], (T - 1) // f + 1, dtype=torch.float)
            torch.manual_seed(seed + 10 + k)
            arrays[f"inf{k}_y"] = m.inference(ci)
            if k == len(inf_lengths) - 1:
                torch.manual_seed(seed + 10 + k)
                arrays[f"inf{k}_y_g"] = m.inference(ci[:, :1], g=g)
            arrays[f"inf{k}_c"], arrays[f"inf{k}_noise"] = ci, noise
        # forward does not crop: a T other than the noise path's length fails at the first TADE combine
        _raises(lambda: m(c[:, :, : f * z_len - 6], z), "size of tensor")
    cat = DiscreteSymbolStyleMelGANGenerator(**dict(kwargs, concat_spk_emb=True)).eval()
    with torch.no_grad():
        _raises(lambda: cat(c, z), "channels")
    meta = dict(kind="dsym_style_generator", kwargs=kwargs, spec=spec, seed=seed, gain=gain, checksum=synth.checksum(sd), g=g,
                inf_lengths=list(inf_lengths), n_params=sum(p.numel() for p in m.parameters()))
    print("   out std %.3f absmax %.3f, %d parameters" % (arrays["y"].std(), arrays["y"].abs().max(), meta["n_params"]))
    save(name, meta, **arrays)


def main():
    import_reference()
    gen_dsym_style("dsym_style_small", SMALL, B=2, z_len=2, inf_lengths=[12, 10], g=3, seed=95, gain=1.0)
    gen_dsym_style("dsym_style_vctk", VCTK, B=2, z_len=1, inf_lengths=[112, 100], g=7, seed=96, gain=1.0)


if __name__ == "__main__":
    main()
