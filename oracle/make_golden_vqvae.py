#!/usr/bin/env python
"""Golden vectors of the reference's VQVAE (TEST INFRASTRUCTURE), run against the REAL reference in the build
container (needs ``/root/reference``); writes ``tests/golden/vqvae_*.npz``.

    python oracle/make_golden_vqvae.py

Each model fixture stores the constructor kwargs, the state-dict spec (with weight norm), the (seed, gain) of the
synthetic weights and their checksum, the factor the codebook rows are scaled by (recorded in meta), the inputs x, l,
g and the eval-mode outputs x_bar, z_e, z_q, indices and decode(indices, l, g).  The synthetic codebook is scaled
until every frame's fp64 gap between its best and second-best code distance is at least MARGIN of the frame's
distance scale |x|^2 + max_k |c_k|^2, so the GPU's indices can be compared exactly.  ``vqvae_collate.npz`` holds
batches of the REAL reference Collater's VQ-wav2wav branch."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import synth  # noqa: E402
from oracle.make_golden import GOLD, import_reference, load_synth, save  # noqa: E402

MARGIN = 1e-3
# egs/yesno/vq1/conf/melgan_vae.v3.debug.yaml generator_params
YESNO = dict(in_channels=1, out_channels=1, num_embeds=16, embed_dim=8, encoder_type="MelGANDiscriminator", decoder_type="MelGANGenerator",
             encoder_conf={"out_channels": 8, "downsample_scales": [4, 4, 2, 2], "max_downsample_channels": 32},
             decoder_conf={"in_channels": 8, "upsample_scales": [4, 4, 2, 2], "channels": 64, "stacks": 2})
# egs/vctk/vq1/conf/conditioned_melgan_vae.v3.yaml generator_params
VCTK_G = dict(in_channels=1, out_channels=1, num_embeds=512, embed_dim=256, num_global_embeds=128, global_embed_dim=128,
              encoder_type="MelGANDiscriminator", decoder_type="MelGANGenerator",
              encoder_conf={"out_channels": 256, "downsample_scales": [4, 4, 2, 2], "max_downsample_channels": 1024},
              decoder_conf={"in_channels": 384, "upsample_scales": [4, 4, 2, 2], "channels": 512, "stacks": 3})
# egs/vctk/vq1/conf/local_conditioned_melgan_vae.v3.yaml generator_params
VCTK_LG = dict(VCTK_G, num_local_embeds=2, local_embed_dim=32,
               decoder_conf={"in_channels": 416, "upsample_scales": [4, 4, 2, 2], "channels": 512, "stacks": 3})


def gaps(z_e, cb):
    """fp64 (best-to-second gap / distance scale) of every frame."""
    x = z_e.double().transpose(1, 2).reshape(-1, cb.shape[1])
    c = cb.double()
    d = (c * c).sum(1)[None] + (x * x).sum(1)[:, None] - 2 * x @ c.t()
    s = d.sort(dim=1)[0]
    return (s[:, 1] - s[:, 0]) / ((x * x).sum(1) + (c * c).sum(1).max())


def gen_vqvae(name, kwargs, B, frames, seed, gain, local=False, glob=False):
    from parallel_wavegan.models import VQVAE

    import copy

    torch.manual_seed(0)
    m = VQVAE(**copy.deepcopy(kwargs)).eval()
    spec, sd = load_synth(m, seed, gain)
    T = frames * 64
    x = synth.randn((B, 1, T), seed + 1, 0.5)
    l = synth.randn((B, kwargs["num_local_embeds"], frames), seed + 2) if local else None
    g = torch.from_numpy(np.random.RandomState(seed).randint(0, kwargs["num_global_embeds"], size=B).astype(np.int64)) if glob else None
    cb0 = m.codebook.embedding.weight.detach().clone()
    with torch.no_grad():
        z_e = m.encoder(x)[-1]
        xn = float(z_e.double().pow(2).sum(1).sqrt().median())
        cn = float(cb0.double().pow(2).sum(1).sqrt().median())
        scale = None
        for f in np.linspace(0.5, 3.0, 26):  # codebook rows of about the frames' norm: the widest relative gaps
            cand = round(float(f * xn / cn), 4)
            if float(gaps(z_e, cb0 * cand).min()) >= MARGIN:
                scale = cand
                break
        assert scale is not None, f"{name}: no codebook scale gives a {MARGIN} margin"
        m.codebook.embedding.weight.mul_(scale)
        min_gap = float(gaps(z_e, m.codebook.embedding.weight).min())
        x_bar, z_e2, z_q = m(x, l, g)
        idx = m.encode(x)
        dec = m.decode(idx, l, g)
    assert torch.equal(z_e2, z_e)
    meta = dict(kind="vqvae", kwargs=kwargs, spec=spec, seed=seed, gain=gain, checksum=synth.checksum(sd), codebook_scale=scale,
                margin=MARGIN, min_gap=min_gap)
    print(f"   {name}: codebook scale {scale}, min relative gap {min_gap:.2e}, x_bar std {float(x_bar.std()):.3f}, "
          f"{len(set(idx.reshape(-1).tolist()))} distinct codes")
    arrays = dict(x=x, x_bar=x_bar, z_e=z_e, z_q=z_q, indices=idx, decode=dec)
    if l is not None:
        arrays["l"] = l
    if g is not None:
        arrays["g"] = g
    save(name, meta, **arrays)


def collate_items():
    """audio, 2-channel local features and a global id per item; one item too short, one 17 samples short of its
    features (edge-padded by _adjust_length)."""
    items = []
    for k, frames in enumerate([40, 9, 33, 52, 21]):
        x = synth.randn((frames * 64,), 8000 + k).numpy()
        if k == 3:
            x = x[:-17]
        items.append((x, synth.randn((frames, 2), 8100 + k).numpy(), np.array([k * 7 % 5], dtype=np.int64)))
    return items


def make_collate_golden():
    sys.modules["tensorboardX"].SummaryWriter = object
    sys.modules["matplotlib"].use = lambda *a, **k: None
    from parallel_wavegan.bin.train import Collater

    items = collate_items()
    out = {}
    np.random.seed(21)
    (l, g), y = Collater(batch_max_steps=1280, hop_size=64, aux_context_window=0, use_aux_input=False, use_global_condition=True,
                         use_local_condition=True)(items)
    out["lg_l"], out["lg_g"], out["lg_y"] = l.numpy(), g.numpy(), y.numpy()
    np.random.seed(22)
    (l, g), y = Collater(batch_max_steps=1280, hop_size=64, aux_context_window=0, use_aux_input=False,
                         use_global_condition=True)([(x, gid) for x, _, gid in items])
    assert l is None
    out["g_g"], out["g_y"] = g.numpy(), y.numpy()
    np.savez_compressed(os.path.join(GOLD, "vqvae_collate.npz"), **out)
    print("wrote vqvae_collate.npz", {k: v.shape for k, v in out.items()})


def main():
    import_reference()
    gen_vqvae("vqvae_yesno", YESNO, B=2, frames=24, seed=101, gain=1.15)
    gen_vqvae("vqvae_vctk_g", VCTK_G, B=2, frames=16, seed=102, gain=1.15, glob=True)
    gen_vqvae("vqvae_vctk_lg", VCTK_LG, B=2, frames=16, seed=103, gain=1.15, local=True, glob=True)
    make_collate_golden()


if __name__ == "__main__":
    main()
