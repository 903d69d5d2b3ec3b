"""CPU restatement of the causal Parallel WaveGAN generator and of ResidualParallelWaveGANDiscriminator (TEST
INFRASTRUCTURE), with the exact references of the causal kernels.  Same conventions as ``oracle/ref_ops.py``
(effective weights keyed like the reference ``state_dict()`` after ``remove_weight_norm()``, fp32 ATen ops); pinned
to golden vectors from the real reference by ``oracle/make_golden_causal_pwg.py``.  Every flag defaults to the
centred model, where these functions compute what ``ref_ops.pwg_generator`` does.

``masks``: optional per-layer dropout masks (already scaled by 1 / (1 - p)), multiplied into each WaveNet layer's
conv input as ``F.dropout`` does in train mode (layers/residual_block.py:114-116); the residual add keeps the
un-dropped x.

All ``file:line`` citations are relative to the reference repository's root."""

import math

import torch
import torch.nn.functional as F

from . import bf16x3, ffma_exact
from .ref_ops import melgan_generator

MELGAN_DEFAULTS = dict(  # MelGANGenerator's constructor defaults (models/melgan.py:24-44)
    in_channels=80, out_channels=1, kernel_size=7, channels=512, upsample_scales=(8, 8, 2, 2), stack_kernel_size=3,
    stacks=3, negative_slope=0.2, use_final_nonlinear_activation=True, use_causal_conv=False,
)


def wavenet_padding(kernel_size, dilation, causal):
    """(left, right) zero padding of the dilated conv once the causal tail crop is applied"""
    return ((kernel_size - 1) * dilation, 0) if causal else ((kernel_size - 1) // 2 * dilation,) * 2


def wavenet_residual_block(w, prefix, x, c, dilation, kernel_size=3, causal=False, mask=None):
    """WaveNetResidualBlock.forward (layers/residual_block.py:102-140); ``causal`` pads (K-1)*dilation and keeps the
    first T outputs (:73-77, :118); ``mask``: the dropout mask of the conv input."""
    residual = x
    xd = x if mask is None else x * mask
    g = F.conv1d(F.pad(xd, wavenet_padding(kernel_size, dilation, causal)), w[f"{prefix}.conv.weight"],
                 w.get(f"{prefix}.conv.bias"), dilation=dilation)
    half = g.shape[1] // 2
    xa, xb = g[:, :half], g[:, half:]
    if c is not None:
        ca = F.conv1d(c, w[f"{prefix}.conv1x1_aux.weight"])
        xa, xb = xa + ca[:, :half], xb + ca[:, half:]
    z = torch.tanh(xa) * torch.sigmoid(xb)
    s = F.conv1d(z, w[f"{prefix}.conv1x1_skip.weight"], w.get(f"{prefix}.conv1x1_skip.bias"))
    x = (F.conv1d(z, w[f"{prefix}.conv1x1_out.weight"], w.get(f"{prefix}.conv1x1_out.bias")) + residual) * math.sqrt(0.5)
    return x, s


def upsample_stages(w, c, scales, prefix, causal=False):
    """UpsampleNetwork.forward (layers/upsample.py:112-128): per scale a nearest repeat and a 1 x (2s+1) FIR shared by
    all rows; causal: the FIR pads 2s on the left and the tail is cropped (:98-100, :124-125)."""
    for i, s in enumerate(scales):
        c = torch.repeat_interleave(c, s, dim=-1)
        fir = w[f"{prefix}.up_layers.{2 * i + 1}.weight"].reshape(1, 1, -1)
        B, C, T = c.shape
        pad = (2 * s, 0) if causal else (s, s)
        c = F.conv1d(F.pad(c.reshape(B * C, 1, T), pad), fir).reshape(B, C, T)
    return c


def pwg_upsample_net(w, c, cfg, prefix="upsample_net"):
    """The generator's conditioning network: ConvInUpsampleNetwork (default; causal conv_in has acw + 1 taps and
    drops its last acw frames when acw > 0, upsample.py:156-194), UpsampleNetwork, or a MelGANGenerator without its
    final tanh (parallel_wavegan.py:108-118)."""
    causal = bool(cfg.get("use_causal_conv", False))
    kind = cfg.get("upsample_net", "ConvInUpsampleNetwork")
    scales = cfg["upsample_scales"]
    if kind == "MelGANGenerator":
        sub = {k[len(prefix) + 1:]: v for k, v in w.items() if k.startswith(prefix + ".")}
        mcfg = dict(MELGAN_DEFAULTS, **cfg.get("upsample_params", {}), use_final_nonlinear_activation=False, use_causal_conv=causal)
        return melgan_generator(sub, c, mcfg)
    if kind == "ConvInUpsampleNetwork":
        acw = cfg.get("aux_context_window", 0)
        c = F.conv1d(c, w[f"{prefix}.conv_in.weight"])
        if causal and acw > 0:
            c = c[:, :, :-acw]
        return upsample_stages(w, c, scales, f"{prefix}.upsample", causal)
    assert kind == "UpsampleNetwork", kind
    return upsample_stages(w, c, scales, prefix, causal)


def pwg_generator(w, z, c, cfg, masks=None):
    """ParallelWaveGANGenerator.forward (models/parallel_wavegan.py:144-173) with ``use_causal_conv`` and the
    upsample-net choice taken from ``cfg``."""
    causal = bool(cfg.get("use_causal_conv", False))
    c = pwg_upsample_net(w, c, cfg)
    assert c.shape[-1] == z.shape[-1]
    x = F.conv1d(z, w["first_conv.weight"], w["first_conv.bias"])
    skips = 0
    lps = cfg["layers"] // cfg["stacks"]
    for layer in range(cfg["layers"]):
        x, h = wavenet_residual_block(w, f"conv_layers.{layer}", x, c, 2 ** (layer % lps), cfg["kernel_size"], causal,
                                      None if masks is None else masks[layer])
        skips = skips + h
    skips = skips * math.sqrt(1.0 / cfg["layers"])
    x = F.relu(skips)
    x = F.conv1d(x, w["last_conv_layers.1.weight"], w["last_conv_layers.1.bias"])
    x = F.relu(x)
    return F.conv1d(x, w["last_conv_layers.3.weight"], w["last_conv_layers.3.bias"])


def residual_pwg_discriminator(w, x, cfg, masks=None):
    """ResidualParallelWaveGANDiscriminator.forward (models/parallel_wavegan.py:466-489)."""
    slope = cfg.get("nonlinear_activation_params", {"negative_slope": 0.2}).get("negative_slope", 0.2)
    causal = bool(cfg.get("use_causal_conv", False))
    x = F.leaky_relu(F.conv1d(x, w["first_conv.0.weight"], w["first_conv.0.bias"]), slope)
    skips = 0
    lps = cfg["layers"] // cfg["stacks"]
    for layer in range(cfg["layers"]):
        x, h = wavenet_residual_block(w, f"conv_layers.{layer}", x, None, 2 ** (layer % lps), cfg.get("kernel_size", 3), causal,
                                      None if masks is None else masks[layer])
        skips = skips + h
    x = skips * math.sqrt(1.0 / cfg["layers"])
    x = F.conv1d(F.leaky_relu(x, slope), w["last_conv_layers.1.weight"], w["last_conv_layers.1.bias"])
    return F.conv1d(F.leaky_relu(x, slope), w["last_conv_layers.3.weight"], w["last_conv_layers.3.bias"])


# --------------------------------------------------------------------------------------------- exact references
def bf16x3_wavenet_layer(x, c, w_conv, *args, causal=False, **kw):
    """``oracle.bf16x3.wavenet_layer`` with a causal dilated conv.  A causal K-tap conv is the centred (2K-1)-tap conv
    whose last K-1 taps are zero: zero weights add exact zeros and do not change the guard's grid, so the emulation
    stays exact and in the kernels' order."""
    if causal:
        G, R, K = w_conv.shape
        w_conv = torch.cat([w_conv, torch.zeros(G, R, K - 1, dtype=w_conv.dtype)], -1)
    return bf16x3.wavenet_layer(x, c, w_conv, *args, **kw)


def upsample_fir(x, fir, scale, causal=False):
    """``oracle.ffma_exact.upsample_fir``; causal: y[r, o] = sum_k f[k] x[r, (o + k - 2s) / s]"""
    if not causal:
        return ffma_exact.upsample_fir(x, fir, scale)
    s = scale
    f = fir.double().reshape(1, 1, -1)
    xr = x.double().repeat_interleave(s, dim=-1)
    sh = xr.shape
    y = F.conv1d(F.pad(xr.reshape(-1, 1, sh[-1]), (2 * s, 0)), f).reshape(sh)
    bound = F.conv1d(F.pad(xr.abs().reshape(-1, 1, sh[-1]), (2 * s, 0)), f.abs()).reshape(sh)
    ex = bf16x3.Exactness(float(bound.max()), bf16x3.grid(x) * bf16x3.grid(fir)) & bf16x3.Exactness(float(fir.double().abs().sum()), bf16x3.grid(fir))
    return y.float(), ex


def upsample_fir_backward_x(gy, fir, scale, causal=False):
    """``oracle.ffma_exact.upsample_fir_backward_x``; causal: the adjoint of the causal stage in x"""
    if not causal:
        return ffma_exact.upsample_fir_backward_x(gy, fir, scale)
    s = scale
    f = fir.double().reshape(1, 1, -1)
    sh = gy.shape
    T = sh[-1] // s

    def adj(v, ff):
        full = F.conv_transpose1d(v.reshape(-1, 1, sh[-1]), ff)  # stretched positions -2s .. T s - 1 (+ 2s past the end)
        return full[:, :, 2 * s: 2 * s + T * s].reshape(*sh[:-1], T, s).sum(-1)

    gx = adj(gy.double(), f)
    return gx.float(), bf16x3.Exactness(float(adj(gy.double().abs(), f.abs()).max()), bf16x3.grid(gy) * bf16x3.grid(fir))


def upsample_fir_backward_f(x, gy, scale, causal=False):
    """``oracle.ffma_exact.upsample_fir_backward_f``; causal: df[k] = RN32(sum gy[r, o] x[r, (o + k - 2s) / s])"""
    if not causal:
        return ffma_exact.upsample_fir_backward_f(x, gy, scale)
    s = scale
    xr = F.pad(x.double().repeat_interleave(s, dim=-1), (2 * s, 0))
    g = gy.double()
    Ts = g.shape[-1]
    df = torch.stack([(g * xr[..., k:k + Ts]).sum() for k in range(2 * s + 1)])
    row = (g.abs().sum(-1) * x.double().abs().amax(-1)).reshape(-1)
    gg = bf16x3.grid(x) * bf16x3.grid(gy)
    ex = bf16x3.Exactness(float(row.max()) if row.numel() else 0.0, gg) & ffma_exact._double_exactness(row.sum() * 3, gg)
    return df.float(), ex
