"""CPU restatement of the reference's DiscreteSymbolStyleMelGANGenerator (TEST INFRASTRUCTURE): the embedding of
``oracle.ref_discrete`` on ``oracle.ref_ops``' StyleMelGAN restatement.  Effective (weight-norm folded) weights keyed like
the reference ``state_dict()`` after ``remove_weight_norm()``, plain ATen ops in the dtype of the weights (float64
weights, noise and a float64 target give the float64 autograd the gradient checks compare against).

``forward`` is ``ref_ops.style_melgan_generator`` on the embedding.  ``inference`` crops the upsampled noise before the
first block, which that function's single pass cannot express, so the noise path is restated here for it and the blocks
run through ``ref_ops.tade_res_block``.

Citations are relative to ``/root/reference/``.  Parity status: pinned (see ``tests/test_dsym_style_cpu.py``).
"""
import torch.nn.functional as F

from oracle.ref_discrete import embed
from oracle.ref_ops import style_melgan_generator, tade_res_block


def _style_cfg(cfg):
    return dict(cfg, noise_upsample_negative_slope=cfg["noise_upsample_activation_params"]["negative_slope"])


def noise_path(w, z, cfg):
    """noise_upsample (style_melgan.py:430-455): per scale s ConvTranspose1d(2s, s, padding s // 2 + s % 2,
    output_padding s % 2) -> LeakyReLU; z (B, in_channels, T_z) -> (B, channels, T_z * prod(scales))."""
    slope = cfg["noise_upsample_activation_params"]["negative_slope"]
    x = z
    for i, s in enumerate(cfg["noise_upsample_scales"]):
        x = F.conv_transpose1d(x, w[f"noise_upsample.{2 * i}.weight"], w.get(f"noise_upsample.{2 * i}.bias"), stride=s,
                               padding=s // 2 + s % 2, output_padding=s % 2)
        x = F.leaky_relu(x, slope)
    return x


def dsym_style_generator(w, c, z, cfg):
    """forward(c, z) (style_melgan.py:474-508): c (B, 2, T) indices, z (B, in_channels, T / prod(noise scales))."""
    return style_melgan_generator(w, embed(w, c, cfg), z, _style_cfg(cfg))


def dsym_style_inference(w, c, noise, cfg):
    """inference (style_melgan.py:563-602) on c (T, 2) with its noise (1, in_channels, (T - 1) // prod(noise scales) + 1):
    the upsampled noise is cropped to T frames, nothing else is padded or cropped -> (T * prod(upsample_scales), 1)."""
    c = embed(w, c.t().unsqueeze(0), cfg)
    x = noise_path(w, noise, cfg)[:, :, : c.shape[2]]
    for i, s in enumerate(cfg["upsample_scales"]):
        x, c = tade_res_block(w, f"blocks.{i}", x, c, cfg["kernel_size"], cfg["dilation"], s, cfg.get("gated_function", "softmax"))
    pad = (cfg["kernel_size"] - 1) // 2
    return F.conv1d(x, w["output_conv.0.weight"], w.get("output_conv.0.bias"), padding=pad).tanh()[0].t()
