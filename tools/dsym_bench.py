#!/usr/bin/env python
"""Discrete-symbol HiFi-GAN measurements on one GPU; prints one JSON line.

* inference of the vctk HuBERT recipe's generator (egs/vctk/hubert_voc1/conf/hifigan_hubert.v1.yaml: 512 channels,
  scales 10 8 2 2, 100 units, 128 speakers; weight norm removed, eval mode) on a batch of 16 x 250 frames (5 s at
  16 kHz): ms per forward from device events with the L2 flushed before each step, libpwgb launches per forward, and
  the time of the embed kernel alone against the whole forward;
* one GanTrainStep of the cvss_c duration recipe (egs/cvss_c/hubert_voc1/conf/hifigan_hubert_duration.v1.yaml) at
  its batch (16 x 10240 samples) from the device duration collater: ms per step (host clock around synchronised steps);
* ``inference`` of the vctk HuBERT StyleMelGAN recipe's generator (egs/vctk/hubert_voc1/conf/style_melgan_hubert.v1.yaml:
  64 channels, noise scales 7 2 2 2, scales 5 2 2 2 2 2 2 1 1; weight norm removed, eval mode) on one utterance of 250
  frames (5 s at 16 kHz) with its noise on the device: ms per call from device events with the L2 flushed before each
  call, and libpwgb launches per call;
* the card's name and power limit, read in the same call.

    python tools/dsym_bench.py [--steps 10] [--warmup 3] [--cases inference,train,style]
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

from uhifigan_bench import card, timed  # noqa: E402

RES = dict(resblock_kernel_sizes=[3, 7, 11], resblock_dilations=[[1, 3, 5], [1, 3, 5], [1, 3, 5]], use_additional_convs=True, bias=True,
           nonlinear_activation="LeakyReLU", nonlinear_activation_params={"negative_slope": 0.1}, use_weight_norm=True)
VCTK = dict(in_channels=512, out_channels=1, channels=512, num_embs=100, num_spk_embs=128, spk_emb_dim=512, concat_spk_emb=False,
            kernel_size=7, upsample_scales=[10, 8, 2, 2], upsample_kernel_sizes=[20, 16, 4, 4], **RES)
CVSS = dict(in_channels=512, out_channels=1, channels=512, num_embs=500, kernel_size=7, upsample_scales=[10, 8, 2, 2],
            upsample_kernel_sizes=[20, 16, 4, 4], duration_layers=2, duration_chans=384, duration_kernel_size=3, duration_offset=1.0,
            duration_dropout_rate=0.5, num_spk_embs=0, **RES)
STYLE = dict(in_channels=128, aux_channels=128, channels=64, out_channels=1, num_embs=100, num_spk_embs=128, spk_emb_dim=128,
             concat_spk_emb=False, kernel_size=9, dilation=2, bias=True, noise_upsample_scales=[7, 2, 2, 2],
             noise_upsample_activation="LeakyReLU", noise_upsample_activation_params={"negative_slope": 0.2},
             upsample_scales=[5, 2, 2, 2, 2, 2, 2, 1, 1], upsample_mode="nearest", gated_function="softmax", use_weight_norm=True)
HOP = 320


def inference(args, dev, flush):
    from oracle import synth
    from parallelwavegan_b200 import capi, models, ops

    m = models.DiscreteSymbolHiFiGANGenerator(**VCTK)
    m.load_state_dict(synth.synth_state_dict([(k, tuple(v.shape)) for k, v in m.state_dict().items()], 61, 1.0))
    m.remove_weight_norm()
    m = m.to(dev).eval()
    rng = np.random.RandomState(0)
    B, F = 16, 250
    c = np.concatenate([rng.randint(0, 100, size=(B, 1, F)), np.repeat(rng.randint(0, 128, size=(B, 1, 1)), F, axis=2)], axis=1)
    c = torch.from_numpy(c.astype(np.float32)).to(dev)
    with torch.no_grad():
        m(c)
        torch.cuda.synchronize()
        capi.reset_launch_count()
        m(c)
        torch.cuda.synchronize()
        launches = capi.launch_count()
        ms, ms_embed = timed([lambda: m(c), lambda: ops.symbol_embed_raw(c, m.emb.weight, m.spk_emb.weight)], args.steps, args.warmup,
                             flush)
    return {"workload": f"vctk hubert inference, batch {B} x {F} frames (hop {HOP}), eval, weight norm removed",
            "ms_per_forward": round(ms, 3), "samples_per_s": round(B * F * HOP / (ms / 1e3)), "launches_per_forward": launches,
            "embed_ms": round(ms_embed, 4), "embed_share": round(ms_embed / ms, 5)}


def train_step(args, dev):
    from oracle import synth
    from parallelwavegan_b200 import datasets, losses, models, optimizers
    from parallelwavegan_b200.train_step import GanTrainStep

    g = models.DiscreteSymbolDurationGenerator(**CVSS)
    g.load_state_dict(synth.synth_state_dict([(k, tuple(v.shape)) for k, v in g.state_dict().items()], 62, 1.0))
    d = models.HiFiGANMultiScaleMultiPeriodDiscriminator()
    d.load_state_dict(synth.synth_state_dict([(k, tuple(v.shape)) for k, v in d.state_dict().items()], 63, 1.4))
    g, d = g.to(dev).train(), d.to(dev).train()
    crit = {
        "duration": losses.DurationPredictorLoss(offset=1.0),
        "mel": losses.MelSpectrogramLoss(fs=16000, fft_size=1024, hop_size=256, win_length=None, window="hann", num_mels=80, fmin=0,
                                         fmax=8000, log_base=None).to(dev),
        "gen_adv": losses.GeneratorAdversarialLoss(average_by_discriminators=False),
        "dis_adv": losses.DiscriminatorAdversarialLoss(average_by_discriminators=False),
        "feat_match": losses.FeatureMatchLoss(average_by_layers=False, average_by_discriminators=False, include_final_outputs=False),
    }
    opt_g = optimizers.FusedAdam(g.parameters(), lr=2e-4, betas=(0.5, 0.9), weight_decay=0.0)
    opt_d = optimizers.FusedAdam(d.parameters(), lr=2e-4, betas=(0.5, 0.9), weight_decay=0.0)
    step = GanTrainStep(g, d, crit, opt_g, opt_d, lambda_aux=45.0, lambda_adv=1.0, lambda_feat_match=2.0, steps=1)
    rng = np.random.RandomState(1)
    items = []
    for _ in range(32):  # HuBERT-like units: runs of 1-3 frames
        frames = int(rng.randint(60, 200))
        codes = np.repeat(rng.randint(0, 500, size=(frames, 1)), rng.randint(1, 4, size=frames), axis=0)[:frames]
        items.append(((0.3 * rng.randn(frames * HOP)).astype(np.float32), codes.astype(np.float32)))
    corpus = datasets.DeviceCorpus(items, dev, hop_size=HOP)
    col = datasets.Collater(batch_max_steps=10240, hop_size=HOP, aux_context_window=0, use_duration=True, pad_value=500)
    np.random.seed(0)
    torch.manual_seed(0)
    batches = [col(corpus, list(rng.choice(len(items), 16, replace=False))) for _ in range(args.steps + args.warmup)]
    for x, y, ds in batches[: args.warmup]:
        step(x, y, ds.clone())
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for x, y, ds in batches[args.warmup:]:
        stats = step(x, y, ds.clone())
    torch.cuda.synchronize()
    ms = (time.perf_counter() - t0) * 1e3 / args.steps
    return {"workload": "cvss_c duration recipe GanTrainStep, batch 16 x 10240 samples, Adam",
            "ms_per_step": round(ms, 2), "duration_loss": float(stats["duration_loss"]), "generator_loss": float(stats["generator_loss"])}


def style_inference(args, dev, flush):
    from oracle import synth
    from parallelwavegan_b200 import capi, models

    m = models.DiscreteSymbolStyleMelGANGenerator(**STYLE)
    m.load_state_dict(synth.synth_state_dict([(k, tuple(v.shape)) for k, v in m.state_dict().items()], 64, 1.0))
    m.remove_weight_norm()
    m = m.to(dev).eval()
    rng = np.random.RandomState(2)
    F = 250
    c = np.stack([rng.randint(0, 100, size=F), np.full(F, 7)], axis=1)
    c = torch.from_numpy(c).to(dev)
    noise = torch.randn(1, 128, (F - 1) // 56 + 1, generator=torch.Generator().manual_seed(3)).to(dev)
    with torch.no_grad():
        m.inference(c, noise=noise)
        torch.cuda.synchronize()
        capi.reset_launch_count()
        m.inference(c, noise=noise)
        torch.cuda.synchronize()
        launches = capi.launch_count()
        (ms,) = timed([lambda: m.inference(c, noise=noise)], args.steps, args.warmup, flush)
    return {"workload": f"vctk hubert StyleMelGAN inference, one utterance of {F} frames (hop {HOP}), eval, weight norm removed",
            "ms_per_inference": round(ms, 3), "samples_per_s": round(F * HOP / (ms / 1e3)), "launches_per_inference": launches}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--cases", default="inference,train,style")
    args = ap.parse_args()
    cases = args.cases.split(",")
    if not torch.cuda.is_available():
        raise SystemExit("dsym_bench: needs a CUDA device (no CPU measurement)")
    import __graft_entry__

    __graft_entry__.build()
    dev = torch.device("cuda:0")
    flush = torch.empty(256 * 1024 * 1024 // 4, device=dev)
    runs = {"inference": lambda: inference(args, dev, flush), "train": lambda: train_step(args, dev),
            "style": lambda: style_inference(args, dev, flush)}
    line = {k: runs[k]() for k in cases}
    line["timing"] = (f"inference, style: device events, mean of {args.steps} steps after {args.warmup} warm-up, L2 flushed (256 MiB "
                      f"write) before each; train: host clock over {args.steps} synchronised steps after {args.warmup} warm-up")
    line["gpu"] = card()
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
