"""CPU restatement of the reference's UHiFiGAN generator (TEST INFRASTRUCTURE), in the style of
``oracle.ref_ops.hifigan_generator``: effective (weight-norm folded) weights keyed like the reference
``state_dict()`` after ``remove_weight_norm()``, plain fp32 ATen ops, eval mode (dropout is the identity).

Citations are relative to ``/root/reference/``.  Parity status: pinned (see ``tests/test_uhifigan_cpu.py``).
"""
import torch
import torch.nn.functional as F

from oracle.ref_ops import hifigan_resblock


def _mrf(w, prefix, first, x, cfg, slope):
    nb = len(cfg["resblock_kernel_sizes"])
    cs = 0.0
    for j in range(nb):
        cs = cs + hifigan_resblock(w, f"{prefix}.{first + j}", x, cfg["resblock_kernel_sizes"][j], cfg["resblock_dilations"][j],
                                   cfg.get("use_additional_convs", True), slope)
    return cs / nb


def uhifigan_generator(w, excitation, c, cfg):
    """UHiFiGANGenerator.forward (models/uhifigan.py:262-301) in eval mode; ``cfg`` holds the constructor kwargs.
    excitation (B, 1, T' * hop), c (B, in_channels, T') -> (B, out_channels, T' * hop)."""
    ks = cfg.get("kernel_size", 7)
    slope = cfg.get("nonlinear_activation_params", {"negative_slope": 0.1}).get("negative_slope", 0.1)
    nb = len(cfg["resblock_kernel_sizes"])
    # input conv -> LeakyReLU -> Dropout (uhifigan.py:79-90)
    h = F.leaky_relu(F.conv1d(excitation, w["input_conv.0.weight"], w.get("input_conv.0.bias"), padding=(ks - 1) // 2), slope)
    skips = []
    for i, s in enumerate(cfg["downsample_scales"]):
        h = _mrf(w, "downsamples_mrf", i * nb, h, cfg, slope)
        # Conv1d(k, stride s, padding s//2 + s%2) -> LeakyReLU -> Dropout (uhifigan.py:118-134)
        h = F.leaky_relu(F.conv1d(h, w[f"downsamples.{i}.0.weight"], w.get(f"downsamples.{i}.0.bias"), stride=s,
                                  padding=s // 2 + s % 2), slope)
        skips.append(h)
    skips.reverse()
    h = F.conv1d(c, w["hidden_conv.weight"], w.get("hidden_conv.bias"), padding=(ks - 1) // 2)
    for i, s in enumerate(cfg["upsample_scales"]):
        # cat -> LeakyReLU -> ConvTranspose1d(k, stride s, padding s//2 + s%2, output_padding s%2) (uhifigan.py:289-291)
        h = torch.cat((h, skips[i]), dim=1)
        h = F.conv_transpose1d(F.leaky_relu(h, slope), w[f"upsamples.{i}.1.weight"], w.get(f"upsamples.{i}.1.bias"), stride=s,
                               padding=s // 2 + s % 2, output_padding=s % 2)
        h = _mrf(w, "upsamples_mrf", i * nb, h, cfg, slope)
    # LeakyReLU() with the default slope 0.01 -> conv k -> tanh (uhifigan.py:222-235)
    h = F.conv1d(F.leaky_relu(h, 0.01), w["output_conv.1.weight"], w.get("output_conv.1.bias"), padding=(ks - 1) // 2)
    return torch.tanh(h)
