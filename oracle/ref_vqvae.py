"""CPU restatement of the reference's VQ-VAE (TEST INFRASTRUCTURE): models/vqvae.py, layers/vector_quantize_codebook.py,
functions/vector_quantizer.py, the VQ losses of bin/train.py:204-219 and the VQ-wav2wav branch of its Collater
(bin/train.py:799-876).  Effective (weight-norm folded) weights keyed like the reference ``state_dict()`` after
``remove_weight_norm()``, plain fp32 ATen ops.  Differentiable with torch autograd (the straight-through estimator is a
small Function), so the GPU gradient tests use it as their reference.

Citations are relative to ``/root/reference/``.  Parity status: pinned (see ``tests/test_vqvae_cpu.py``).
"""
import numpy as np
import torch
import torch.nn.functional as F

from oracle.ref_ops import melgan_discriminator, melgan_generator


def _sub(w, prefix):
    n = len(prefix) + 1
    return {k[n:]: v for k, v in w.items() if k.startswith(prefix + ".")}


def encoder(w, x, cfg):
    """The MelGANDiscriminator encoder's last output z_e (B, embed_dim, T') (vqvae.py:96-97)."""
    ec = cfg.get("encoder_conf", {"downsample_scales": [4, 4, 2, 2], "max_downsample_channels": 1024})
    return melgan_discriminator(w, "encoder", x, downsample_scales=tuple(ec.get("downsample_scales", [4, 4, 4, 4])),
                                kernel_sizes=tuple(ec.get("kernel_sizes", [5, 3])), channels=ec.get("channels", 16),
                                max_ch=ec.get("max_downsample_channels", 1024))[-1]


def distances(z_e, codebook):
    """(B * T', K) fp32 distances of every frame to every code, the reference's formula (vector_quantizer.py:37-50):
    (|c|^2 + |x|^2) - 2 x.c as one addmm."""
    D = codebook.shape[1]
    flat = z_e.transpose(1, 2).reshape(-1, D)
    base = (codebook * codebook).sum(1)[None, :] + (flat * flat).sum(1)[:, None]
    return torch.addmm(base, flat, codebook.t(), beta=1.0, alpha=-2.0)


def quantize(z_e, codebook):
    """Nearest-code indices (B, T') (torch.min over the codes)."""
    with torch.no_grad():
        return distances(z_e, codebook).min(dim=1)[1].reshape(z_e.shape[0], z_e.shape[2])


class _StraightThrough(torch.autograd.Function):
    """codes in the forward, the gradient passed to z_e unchanged (vector_quantizer.py:107-108)."""

    @staticmethod
    def forward(ctx, z_e, codes):
        return codes.clone()

    @staticmethod
    def backward(ctx, g):
        return g, None


def gather(codebook, indices):
    """codebook rows of the indices, channel-major (B, D, T')."""
    return F.embedding(indices, codebook).transpose(1, 2)


def assemble(w, z, l, g):
    """decoder input: z, then local_embed(l) (or l), then the global embedding broadcast over time (vqvae.py:100-108)."""
    parts = [z]
    if l is not None:
        if "local_embed.weight" in w:
            l = F.conv1d(l, w["local_embed.weight"], w["local_embed.bias"])
        parts.append(l)
    if g is not None:
        parts.append(F.embedding(g, w["global_embed.weight"]).unsqueeze(2).expand(-1, -1, z.shape[2]))
    return torch.cat(parts, dim=1)


def decoder(w, dec, cfg):
    dc = dict(kernel_size=7, stack_kernel_size=3, negative_slope=0.2, **cfg.get("decoder_conf", {}))
    return melgan_generator(_sub(w, "decoder"), dec, dc)


def vqvae_forward(w, x, cfg, l=None, g=None):
    """VQVAE.forward (vqvae.py:80-110) -> (x_bar, z_e, z_q, indices)."""
    cb = w["codebook.embedding.weight"]
    z_e = encoder(w, x, cfg)
    idx = quantize(z_e, cb)
    z_q = gather(cb, idx)
    z_q_st = _StraightThrough.apply(z_e, gather(cb.detach(), idx))
    return decoder(w, assemble(w, z_q_st, l, g), cfg), z_e, z_q, idx


def vqvae_encode(w, x, cfg):
    return quantize(encoder(w, x, cfg), w["codebook.embedding.weight"])


def vqvae_decode(w, indices, cfg, l=None, g=None):
    """VQVAE.decode (vqvae.py:127-147)."""
    return decoder(w, assemble(w, gather(w["codebook.embedding.weight"], indices), l, g), cfg)


def vq_losses(z_e, z_q):
    """(quantization_loss, commitment_loss) of bin/train.py:210-211: MSE(z_q, sg(z_e)), MSE(z_e, sg(z_q))."""
    return F.mse_loss(z_q, z_e.detach()), F.mse_loss(z_e, z_q.detach())


def collate_vq(batch, batch_max_steps=8192, hop_size=64, aux_context_window=0, use_local_condition=False,
               use_global_condition=False):
    """The VQ-wav2wav branch of Collater.__call__ (bin/train.py:799-876).  batch items: audio, (audio, g),
    (audio, l (frames, C)) or (audio, l, g).  Returns ((l (B, C, frames) or None, g (B,) int64 or None), y (B, 1, T));
    consumes np.random exactly like the reference (one randint per kept item)."""
    if hop_size is not None and batch_max_steps % hop_size != 0:
        batch_max_steps -= batch_max_steps % hop_size
    frames = batch_max_steps // hop_size if hop_size else None
    l_out = g_out = None
    if use_local_condition:
        thr = frames + 2 * aux_context_window
        kept = []
        for item in batch:
            x, lc = item[0], item[1]
            if len(lc) >= thr:
                if len(x) < len(lc) * hop_size:
                    x = np.pad(x, (0, len(lc) * hop_size - len(x)), mode="edge")
                assert len(x) == len(lc) * hop_size
                kept.append((x, lc) + tuple(item[2:]))
        starts = np.array([np.random.randint(aux_context_window, len(it[1]) - frames - aux_context_window) for it in kept])
        y = [it[0][s * hop_size : s * hop_size + batch_max_steps] for it, s in zip(kept, starts)]
        l_out = np.array([it[1][s : s + frames] for it, s in zip(kept, starts)], dtype=np.float32).transpose(0, 2, 1)
        if use_global_condition:
            g_out = np.array([int(np.asarray(it[2]).reshape(-1)[0]) for it in kept], dtype=np.int64)
    else:
        items = [it if use_global_condition else (it,) for it in batch]
        kept = [it for it in items if len(it[0]) >= batch_max_steps]
        starts = np.array([np.random.randint(0, len(it[0]) - batch_max_steps) for it in kept])
        y = [it[0][s : s + batch_max_steps] for it, s in zip(kept, starts)]
        if use_global_condition:
            g_out = np.array([int(np.asarray(it[1]).reshape(-1)[0]) for it in kept], dtype=np.int64)
    y = np.array(y, dtype=np.float32)[:, None, :]
    return (l_out, g_out), y
