#!/usr/bin/env python
"""VQ-VAE measurements on one GPU (egs/vctk/vq1/conf/local_conditioned_melgan_vae.v3.yaml: K = 512 codes of D = 256,
2 local features embedded to 32 channels, 128 speakers of 128 channels, hop 64); prints one JSON line.

* inference, encode + decode, weight norm removed, eval mode, at 16 utterances x 8192 samples and at one 10 s utterance
  (240000 samples at 24 kHz): ms per call from device events with the L2 flushed before each, libpwgb launches per
  forward, and the VQ kernels' (vq_forward) time and share of the forward;
* the VQ forward kernel (search, gather, assembly) against the torch composition it replaces
  (addmm + min + index_select + cat) on the same z_e, alternated in one run, L2 flushed before each;
* one GanTrainStep with the discriminator on at 16 x 8192 samples (host clock around synchronised steps);
* the card's name and power limit, read in the same call.

    python tools/vqvae_bench.py [--steps 10] [--warmup 3]
"""
import argparse
import copy
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

VCTK_LG = dict(in_channels=1, out_channels=1, num_embeds=512, embed_dim=256, num_local_embeds=2, local_embed_dim=32, num_global_embeds=128,
               global_embed_dim=128, encoder_type="MelGANDiscriminator", decoder_type="MelGANGenerator",
               encoder_conf={"out_channels": 256, "downsample_scales": [4, 4, 2, 2], "max_downsample_channels": 1024},
               decoder_conf={"in_channels": 416, "upsample_scales": [4, 4, 2, 2], "channels": 512, "stacks": 3})
HOP = 64


def _model(dev, seed):
    from parallelwavegan_b200 import models
    from parallelwavegan_b200.synth_weights import synth_state_dict

    m = models.VQVAE(**copy.deepcopy(VCTK_LG))
    m.load_state_dict(synth_state_dict([(k, tuple(v.shape)) for k, v in m.state_dict().items()], seed, 1.15))
    return m.to(dev)


def _inputs(dev, B, T, seed):
    g = torch.Generator().manual_seed(seed)
    x = (0.3 * torch.randn(B, 1, T, generator=g)).to(dev)
    l = torch.randn(B, 2, T // HOP, generator=g).to(dev)
    gid = torch.randint(0, 128, (B,), generator=g).to(dev)
    return x, l, gid


def inference(args, dev, flush):
    from parallelwavegan_b200 import capi, ops

    m = _model(dev, 71)
    m.remove_weight_norm()
    m.eval()
    out = []
    for B, T, what in ((16, 8192, "16 x 8192 samples"), (1, 240000, "one 10 s utterance (240000 samples at 24 kHz)")):
        x, l, gid = _inputs(dev, B, T, 72)
        with torch.no_grad():
            m.decode(m.encode(x), l, gid)
            torch.cuda.synchronize()
            capi.reset_launch_count()
            m(x, l, gid)
            torch.cuda.synchronize()
            launches = capi.launch_count()
            z_e = m.encoder(x)[-1]
            le = m._local(l)
            cb, gt = m.codebook.embedding.weight, m.global_embed.weight
            ms, ms_fwd, ms_vq = timed([lambda: m.decode(m.encode(x), l, gid), lambda: m(x, l, gid),
                                       lambda: ops.vq_raw(z_e, cb, l=le, global_table=gt, g=gid)], args.steps, args.warmup, flush)
        out.append({"workload": f"vctk local_conditioned encode + decode, {what}, eval, weight norm removed",
                    "ms_encode_decode": round(ms, 3), "ms_forward": round(ms_fwd, 3), "launches_per_forward": launches,
                    "vq_forward_ms": round(ms_vq, 4), "vq_share_of_forward": round(ms_vq / ms_fwd, 5)})
    return out


def vq_vs_torch(args, dev, flush):
    """The VQ forward kernel against addmm + min + index_select + cat at the training shape (2048 frames)."""
    from parallelwavegan_b200 import ops

    g = torch.Generator().manual_seed(5)
    B, T, D, K = 16, 8192 // HOP, 256, 512
    z_e = torch.randn(B, D, T, generator=g).to(dev)
    cb = (0.06 * torch.randn(K, D, generator=g)).to(dev)
    l = torch.randn(B, 32, T, generator=g).to(dev)
    gt = torch.randn(128, 128, generator=g).to(dev)
    gid = torch.randint(0, 128, (B,), generator=g).to(dev)

    def composed():
        flat = z_e.transpose(1, 2).reshape(-1, D)
        d = torch.addmm((cb * cb).sum(1)[None] + (flat * flat).sum(1, keepdim=True), flat, cb.t(), beta=1.0, alpha=-2.0)
        idx = d.min(1)[1]
        zq = torch.index_select(cb, 0, idx).view(B, T, D).transpose(1, 2)
        return torch.cat([zq, l, gt[gid].unsqueeze(2).expand(-1, -1, T)], 1), idx

    with torch.no_grad():
        ms_k, ms_t = timed([lambda: ops.vq_raw(z_e, cb, z_q=False, l=l, global_table=gt, g=gid), composed], args.steps * 5, args.warmup,
                           flush)
        idx_k, _, dec_k = ops.vq_raw(z_e, cb, z_q=False, l=l, global_table=gt, g=gid)
        dec_t, idx_t = composed()
    agree = float((idx_k.reshape(-1) == idx_t).float().mean())
    return {"shape": f"B {B} x T' {T} frames, K {K}, D {D}, Cl 32, Cg 128", "vq_kernel_ms": round(ms_k, 4), "torch_composed_ms": round(ms_t, 4),
            "fma": B * T * K * D, "index_agreement_with_torch": agree,
            "dec_bit_identical_where_indices_agree": bool(torch.equal(dec_k.transpose(1, 2).reshape(-1, dec_k.shape[1])[idx_k.reshape(-1) == idx_t],
                                                                      dec_t.transpose(1, 2).reshape(-1, dec_t.shape[1])[idx_k.reshape(-1) == idx_t]))}


def train_step(args, dev):
    from parallelwavegan_b200 import losses, models, optimizers
    from parallelwavegan_b200.synth_weights import synth_state_dict
    from parallelwavegan_b200.train_step import GanTrainStep

    g = _model(dev, 73).train()
    d = models.MelGANMultiScaleDiscriminator()
    d.load_state_dict(synth_state_dict([(k, tuple(v.shape)) for k, v in d.state_dict().items()], 74, 1.3))
    d = d.to(dev).train()
    crit = {"stft": losses.MultiResolutionSTFTLoss().to(dev), "mse": losses.MSELoss(), "gen_adv": losses.GeneratorAdversarialLoss(),
            "dis_adv": losses.DiscriminatorAdversarialLoss(), "feat_match": losses.FeatureMatchLoss()}
    opt_g = optimizers.FusedAdam(g.parameters(), lr=1e-4, eps=1e-6)
    opt_d = optimizers.FusedAdam(d.parameters(), lr=5e-5, eps=1e-6)
    step = GanTrainStep(g, d, crit, opt_g, opt_d, lambda_aux=1.0, lambda_adv=4.0, lambda_feat_match=25.0, lambda_commit=0.25,
                        grad_norm_g=10, grad_norm_d=1, steps=1)
    batches = [_inputs(dev, 16, 8192, 100 + i) for i in range(args.steps + args.warmup)]
    for x, l, gid in batches[: args.warmup]:
        step((l, gid), x)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for x, l, gid in batches[args.warmup:]:
        stats = step((l, gid), x)
    torch.cuda.synchronize()
    ms = (time.perf_counter() - t0) * 1e3 / args.steps
    return {"workload": "vctk local_conditioned GanTrainStep, discriminator on, batch 16 x 8192 samples, Adam",
            "ms_per_step": round(ms, 2), "generator_loss": float(stats["generator_loss"]),
            "quantization_loss": float(stats["quantization_loss"])}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("vqvae_bench: needs a CUDA device (no CPU measurement)")
    import __graft_entry__

    __graft_entry__.build()
    dev = torch.device("cuda:0")
    flush = torch.empty(256 * 1024 * 1024 // 4, device=dev)
    line = {"inference": inference(args, dev, flush), "vq_vs_torch": vq_vs_torch(args, dev, flush), "train": train_step(args, dev),
            "timing": f"inference and kernels: device events, mean over alternated calls after {args.warmup} warm-up, L2 flushed "
                      f"(256 MiB write) before each; train: host clock over {args.steps} synchronised steps after {args.warmup} warm-up",
            "gpu": card()}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
