#!/usr/bin/env python
"""Golden vectors of the reference's DiscreteSymbolHiFiGANGenerator / DiscreteSymbolDurationGenerator (TEST
INFRASTRUCTURE), run against the REAL reference in the build container (needs ``/root/reference``); writes
``tests/golden/dsym_*.npz``.

    python oracle/make_golden_discrete.py

Each fixture stores the constructor kwargs, the state-dict spec (with weight norm), the (seed, gain) of the synthetic
weights and their checksum, the symbol indices ``c`` themselves (and the teacher durations ``ds``), and the eval-mode
outputs.  The duration fixtures set ``duration_predictor.linear.bias`` and scale its weight (both recorded in meta) so that the predicted
durations spread over a few frames, and assert that every exp(x) - offset lies at least 1e-2 from a rounding boundary,
so the integer durations can be compared exactly on the GPU."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import synth  # noqa: E402
from oracle.make_golden import import_reference, load_synth, save  # noqa: E402

RES = dict(resblock_kernel_sizes=[3, 7, 11], resblock_dilations=[[1, 3, 5], [1, 3, 5], [1, 3, 5]], use_additional_convs=True, bias=True,
           nonlinear_activation="LeakyReLU", nonlinear_activation_params={"negative_slope": 0.1}, use_weight_norm=True)
# egs/vctk/hubert_voc1/conf/hifigan_hubert.v1.yaml generator_params
VCTK = dict(in_channels=512, out_channels=1, channels=512, num_embs=100, num_spk_embs=128, spk_emb_dim=512, concat_spk_emb=False,
            kernel_size=7, upsample_scales=[10, 8, 2, 2], upsample_kernel_sizes=[20, 16, 4, 4], **RES)
# egs/cvss_c/hubert_voc1/conf/hifigan_hubert_duration.v1.yaml generator_params
CVSS = dict(in_channels=512, out_channels=1, channels=512, num_embs=500, kernel_size=7, upsample_scales=[10, 8, 2, 2],
            upsample_kernel_sizes=[20, 16, 4, 4], duration_layers=2, duration_chans=384, duration_kernel_size=3, duration_offset=1.0,
            duration_dropout_rate=0.5, num_spk_embs=0, **RES)


def _symbols(rng, B, T, num_embs, num_spk=0, dtype=np.float32):
    c = rng.randint(0, num_embs, size=(B, 1, T))
    if num_spk:
        c = np.concatenate([c, np.repeat(rng.randint(0, num_spk, size=(B, 1, 1)), T, axis=2)], axis=1)
    return torch.from_numpy(c.astype(dtype))


def gen_dsym(name, kwargs, B, T, seed, gain, g=None):
    from parallel_wavegan.models import DiscreteSymbolHiFiGANGenerator

    torch.manual_seed(0)
    m = DiscreteSymbolHiFiGANGenerator(**kwargs).eval()
    spec, sd = load_synth(m, seed, gain)
    nspk = kwargs.get("num_spk_embs", 128)
    c = _symbols(np.random.RandomState(seed), B, T, kwargs["num_embs"], nspk)
    arrays = {}
    with torch.no_grad():
        arrays["y"] = m(c)
        arrays["y_inf"] = m.inference(c[0].t())
        if g is not None:
            arrays["y_inf_g"] = m.inference(c[0].t(), g=g)
    meta = dict(kind="dsym_generator", kwargs=kwargs, spec=spec, seed=seed, gain=gain, checksum=synth.checksum(sd), g=g)
    print("   out std %.3f absmax %.3f" % (arrays["y"].std(), arrays["y"].abs().max()))
    save(name, meta, c=c, **arrays)


def _margin(x, offset):
    v = (x.double().exp() - offset).reshape(-1)
    return float((v - (torch.floor(v) + 0.5)).abs().min())


def gen_dsym_duration(name, kwargs, B, S, seed, gain):
    """forward with teacher durations (one padded symbol: index num_embs, duration 0), synthesis and inference."""
    from parallel_wavegan.models import DiscreteSymbolDurationGenerator

    torch.manual_seed(0)
    m = DiscreteSymbolDurationGenerator(**kwargs).eval()
    spec, sd = load_synth(m, seed, gain)
    rng = np.random.RandomState(seed)
    c = _symbols(rng, B, S, kwargs["num_embs"], dtype=np.int64)
    ds = torch.from_numpy(rng.randint(0, 4, size=(B, S)).astype(np.int64))
    c[1, 0, -1] = kwargs["num_embs"]  # the collater's padding symbol (bin/train.py:1321-1323)
    ds[1, -1] = 0
    offset = kwargs.get("duration_offset", 1.0)
    # pick the predictor's output bias: predicted durations over 0..4 frames, every exp(x) - offset >= 1e-2 from a
    # rounding boundary
    lin = m.duration_predictor.linear
    scale = 0.25  # the synthetic LayerNorm gains make the log-durations spread over several octaves: narrow them
    with torch.no_grad():
        lin.weight.mul_(scale)
        base = lin.bias.clone()
        e = m.emb(c[:, 0]).transpose(1, 2)
        x0 = m.duration_predictor(e.transpose(1, 2)) - base
        bias = None
        for cand in np.linspace(-0.5, 2.0, 251):
            x = x0 + float(cand)
            d = torch.clamp(torch.round(x.exp() - offset), min=0)
            if _margin(x, offset) >= 1e-2 and int(d.min()) == 0 and 2 <= int(d.max()) <= 5 and float(d.sum(1).min()) > 0:
                bias = float(cand)
                break
        assert bias is not None, "no predictor bias with a 1e-2 rounding margin"
        lin.bias.fill_(bias)
        assert _margin(m.duration_predictor(e.transpose(1, 2)), offset) >= 1e-2
        y, ds_out = m(c, ds.clone())
        y_syn, ds_syn = m.synthesis(c)
        y_inf = m.inference(c[0].t())
        y_inf_ds = m.inference(c[0].t(), ds=ds[0].clone())
    meta = dict(kind="dsym_duration_generator", kwargs=kwargs, spec=spec, seed=seed, gain=gain, checksum=synth.checksum(sd),
                linear_bias=bias, linear_weight_scale=scale)
    print("   out std %.3f absmax %.3f, synthesis durations %s" % (y.std(), y.abs().max(), ds_syn.tolist()))
    save(name, meta, c=c, ds=ds, y=y, ds_out=ds_out, y_syn=y_syn, ds_syn=ds_syn, y_inf=y_inf, y_inf_ds=y_inf_ds)


def main():
    import_reference()
    small = dict(in_channels=64, out_channels=1, channels=64, num_embs=10, num_spk_embs=0, kernel_size=7, upsample_scales=[4, 2],
                 upsample_kernel_sizes=[8, 4], **RES)
    gen_dsym("dsym_small", small, B=2, T=12, seed=91, gain=1.15)
    gen_dsym("dsym_vctk", VCTK, B=2, T=20, seed=92, gain=1.15, g=7)
    gen_dsym_duration("dsym_dur_cvss", CVSS, B=2, S=10, seed=93, gain=1.15)
    # odd scale with k != 2s (padding (k - s) // 2 and no output_padding: lengths 3T + 1, then 6T + 2), two MRF blocks,
    # no additional convs, no bias
    odd = dict(CVSS, in_channels=32, channels=64, num_embs=20, upsample_scales=[3, 2], upsample_kernel_sizes=[6, 4], duration_chans=64,
               resblock_kernel_sizes=[3, 5], resblock_dilations=[[1, 3], [1, 2]], use_additional_convs=False, bias=False)
    gen_dsym_duration("dsym_dur_odd", odd, B=2, S=7, seed=94, gain=1.3)


if __name__ == "__main__":
    main()
