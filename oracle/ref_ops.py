"""CPU restatement of the reference's hot-path algorithms (TEST INFRASTRUCTURE).

Every function takes the *effective* (weight-norm folded) weights as a flat dict
keyed exactly like the reference ``state_dict()`` after ``remove_weight_norm()``
and computes in fp32 with plain torch CPU functional ops -- the same ATen ops
the reference modules call -- so that it can (a) be pinned against golden
vectors generated from the real reference (``oracle/make_golden.py``) and
(b) travel to the GPU box, where ``/root/reference`` does not exist.

All ``file:line`` citations are relative to ``/root/reference/``.
Parity status: pinned (see ``tests/test_oracle_golden.py``).
"""

import math

import numpy as np
import torch
import torch.nn.functional as F

# --------------------------------------------------------------------------
# weight (re-)parametrisation
# --------------------------------------------------------------------------


def fold_weight_norm(sd):
    """``w = g * v / ||v||`` over all dims but 0 (torch.nn.utils.weight_norm,
    dim=0; applied at hifigan.py:221-231, melgan.py:192-202,
    parallel_wavegan.py:187-195).  Keys ``X.weight_g``/``X.weight_v`` become
    ``X.weight``; everything else is passed through."""
    out = {}
    for k, v in sd.items():
        if k.endswith(".weight_g"):
            base = k[: -len("_g")]
            vv = sd[base + "_v"].float()
            g = v.float()
            dims = tuple(range(1, vv.dim()))
            norm = vv.pow(2).sum(dim=dims, keepdim=True).sqrt()
            out[base] = g * vv / norm
        elif k.endswith(".weight_v") and (k[: -len("_v")] + "_g") in sd:
            continue
        else:
            out[k] = v
    return out


def spectral_norm_weight(w_orig, u, n_power_iterations=1, eps=1e-12, training=True):
    """torch.nn.utils.spectral_norm forward (hifigan.py:613-621 applies it to
    MSD scale 0).  Returns (w, u_new, v_new)."""
    w_mat = w_orig.reshape(w_orig.shape[0], -1)
    v = None
    if training:
        for _ in range(n_power_iterations):
            v = F.normalize(torch.mv(w_mat.t(), u), dim=0, eps=eps)
            u = F.normalize(torch.mv(w_mat, v), dim=0, eps=eps)
    else:
        raise ValueError("eval-mode spectral norm needs the stored v")
    sigma = torch.dot(u, torch.mv(w_mat, v))
    return w_orig / sigma, u, v


# --------------------------------------------------------------------------
# independent float64 direct-loop convolutions (cross-check of ATen on tiny cases)
# --------------------------------------------------------------------------


def np_conv1d(x, w, b=None, stride=1, padding=0, dilation=1, groups=1):
    """Direct definition of cross-correlation conv1d in float64 numpy."""
    x = np.asarray(x, np.float64)
    w = np.asarray(w, np.float64)
    b = None if b is None else np.asarray(b, np.float64)
    B, Cin, T = x.shape
    Cout, Cin_g, K = w.shape
    xp = np.zeros((B, Cin, T + 2 * padding))
    xp[:, :, padding : padding + T] = x
    Tout = (T + 2 * padding - dilation * (K - 1) - 1) // stride + 1
    y = np.zeros((B, Cout, Tout))
    cog = Cout // groups
    for co in range(Cout):
        g = co // cog
        for ci in range(Cin_g):
            for k in range(K):
                seg = xp[:, g * Cin_g + ci, k * dilation : k * dilation + stride * (Tout - 1) + 1 : stride]
                y[:, co, :] += w[co, ci, k] * seg
        if b is not None:
            y[:, co, :] += b[co]
    return y


def np_conv_transpose1d(x, w, b=None, stride=1, padding=0, output_padding=0):
    """Direct definition of ConvTranspose1d (weight (Cin, Cout, K)) in float64."""
    x = np.asarray(x, np.float64)
    w = np.asarray(w, np.float64)
    B, Cin, T = x.shape
    _, Cout, K = w.shape
    full = np.zeros((B, Cout, (T - 1) * stride + K + output_padding))
    for ci in range(Cin):
        for co in range(Cout):
            for k in range(K):
                full[:, co, k : k + (T - 1) * stride + 1 : stride] += x[:, ci, :] * w[ci, co, k]
    Tout = (T - 1) * stride - 2 * padding + K + output_padding
    y = full[:, :, padding : padding + Tout]
    if b is not None:
        y = y + np.asarray(b, np.float64)[None, :, None]
    return y


# --------------------------------------------------------------------------
# HiFi-GAN generator   (models/hifigan.py:23-267, layers/residual_block.py:143-258)
# --------------------------------------------------------------------------

HIFIGAN_V1 = dict(
    in_channels=80,
    out_channels=1,
    channels=512,
    kernel_size=7,
    upsample_scales=(8, 8, 2, 2),
    upsample_kernel_sizes=(16, 16, 4, 4),
    resblock_kernel_sizes=(3, 7, 11),
    resblock_dilations=((1, 3, 5), (1, 3, 5), (1, 3, 5)),
    use_additional_convs=True,
    bias=True,
    negative_slope=0.1,
)


def causal_conv1d(x, weight, bias, dilation=1, mode="constant"):
    """CausalConv1d.forward (layers/causal_conv.py:32-43): pad (k-1)*d on BOTH sides, conv, keep the first T."""
    n = (weight.shape[-1] - 1) * dilation
    xp = F.pad(x, (n, n), mode=mode) if n else x
    return F.conv1d(xp, weight, bias, dilation=dilation)[:, :, : x.shape[2]]


def causal_conv_transpose1d(x, weight, bias, stride):
    """CausalConvTranspose1d.forward (layers/causal_conv.py:68-79): replicate-pad one frame on the
    left, transposed conv without padding, drop ``stride`` samples on each side."""
    xp = F.pad(x, (1, 0), mode="replicate")
    return F.conv_transpose1d(xp, weight, bias, stride=stride)[:, :, stride:-stride]


def hifigan_resblock(w, prefix, x, kernel_size, dilations, use_additional_convs=True, slope=0.1, causal=False):
    """HiFiGANResidualBlock.forward (layers/residual_block.py:243-258)."""
    for idx, d in enumerate(dilations):
        if causal:  # residual_block.py:194-209, 227-241: Sequential(act, CausalConv1d)
            xt = causal_conv1d(F.leaky_relu(x, slope), w[f"{prefix}.convs1.{idx}.1.conv.weight"], w.get(f"{prefix}.convs1.{idx}.1.conv.bias"), d)
            if use_additional_convs:
                xt = causal_conv1d(F.leaky_relu(xt, slope), w[f"{prefix}.convs2.{idx}.1.conv.weight"], w.get(f"{prefix}.convs2.{idx}.1.conv.bias"), 1)
            x = xt + x
            continue
        xt = F.conv1d(
            F.leaky_relu(x, slope),
            w[f"{prefix}.convs1.{idx}.1.weight"],
            w.get(f"{prefix}.convs1.{idx}.1.bias"),
            dilation=d,
            padding=(kernel_size - 1) // 2 * d,
        )
        if use_additional_convs:
            xt = F.conv1d(
                F.leaky_relu(xt, slope),
                w[f"{prefix}.convs2.{idx}.1.weight"],
                w.get(f"{prefix}.convs2.{idx}.1.bias"),
                padding=(kernel_size - 1) // 2,
            )
        x = xt + x
    return x


def hifigan_generator(w, c, cfg=HIFIGAN_V1):
    """HiFiGANGenerator.forward (models/hifigan.py:173-192); ``use_causal_conv`` selects the
    CausalConv1d / CausalConvTranspose1d wiring (hifigan.py:80-91, 108-121, 143-158)."""
    ks = cfg["kernel_size"]
    slope = cfg.get("negative_slope", 0.1)
    nb = len(cfg["resblock_kernel_sizes"])
    causal = bool(cfg.get("use_causal_conv", False))
    if causal:
        c = causal_conv1d(c, w["input_conv.conv.weight"], w.get("input_conv.conv.bias"))
    else:
        c = F.conv1d(c, w["input_conv.weight"], w.get("input_conv.bias"), padding=(ks - 1) // 2)
    for i, s in enumerate(cfg["upsample_scales"]):
        if causal:
            c = causal_conv_transpose1d(F.leaky_relu(c, slope), w[f"upsamples.{i}.1.deconv.weight"], w.get(f"upsamples.{i}.1.deconv.bias"), s)
        else:
            # hifigan.py:94-107: LeakyReLU -> ConvTranspose1d(k=2s, stride s, pad s//2+s%2, out_pad s%2)
            c = F.conv_transpose1d(
                F.leaky_relu(c, slope),
                w[f"upsamples.{i}.1.weight"],
                w.get(f"upsamples.{i}.1.bias"),
                stride=s,
                padding=s // 2 + s % 2,
                output_padding=s % 2,
            )
        cs = 0.0
        for j in range(nb):
            cs = cs + hifigan_resblock(
                w,
                f"blocks.{i * nb + j}",
                c,
                cfg["resblock_kernel_sizes"][j],
                cfg["resblock_dilations"][j],
                cfg.get("use_additional_convs", True),
                slope,
                causal,
            )
        c = cs / nb
    # hifigan.py:139-151: LeakyReLU() with the *default* slope 0.01, conv k, tanh
    if causal:
        return torch.tanh(causal_conv1d(F.leaky_relu(c, 0.01), w["output_conv.1.conv.weight"], w.get("output_conv.1.conv.bias")))
    c = F.conv1d(F.leaky_relu(c, 0.01), w["output_conv.1.weight"], w.get("output_conv.1.bias"), padding=(ks - 1) // 2)
    return torch.tanh(c)


# --------------------------------------------------------------------------
# MelGAN / multi-band MelGAN generator (models/melgan.py:17-257, layers/residual_stack.py)
# --------------------------------------------------------------------------

MB_MELGAN_V2 = dict(  # egs/csmsc/voc1/conf/multi_band_melgan.v2.yaml:35-45
    in_channels=80,
    out_channels=4,
    kernel_size=7,
    channels=384,
    upsample_scales=(5, 5, 3),
    stack_kernel_size=3,
    stacks=4,
    negative_slope=0.2,
    use_final_nonlinear_activation=True,
)


def melgan_layer_index(cfg):
    """Sequential indices of the parametrised layers of ``self.melgan``
    (melgan.py:68-156): returns a list of ("conv"|"convt"|"stack"|"final", idx, meta)."""
    plan = []
    idx = 0
    causal = bool(cfg.get("use_causal_conv", False))
    if causal:
        plan.append(("conv_in", idx, None))  # [CausalConv1d]
        idx += 1
    else:
        plan.append(("conv_in", idx + 1, None))  # [ReflectionPad, Conv1d]
        idx += 2
    for i, s in enumerate(cfg["upsample_scales"]):
        plan.append(("convt", idx + 1, (i, s)))  # [act, ConvTranspose1d | CausalConvTranspose1d]
        idx += 2
        for j in range(cfg["stacks"]):
            plan.append(("stack", idx, (i, j)))
            idx += 1
    plan.append(("conv_out", idx + (1 if causal else 2), None))  # [act, (pad,) conv, (tanh)]
    return plan


def melgan_residual_stack(w, prefix, c, kernel_size, dilation, slope, causal=False):
    """ResidualStack.forward (layers/residual_stack.py:75-85; causal wiring :56-70)."""
    h = F.leaky_relu(c, slope)
    if causal:
        h = causal_conv1d(h, w[f"{prefix}.stack.1.conv.weight"], w.get(f"{prefix}.stack.1.conv.bias"), dilation, mode="reflect")
        h = F.leaky_relu(h, slope)
        h = F.conv1d(h, w[f"{prefix}.stack.3.weight"], w.get(f"{prefix}.stack.3.bias"))
        return h + F.conv1d(c, w[f"{prefix}.skip_layer.weight"], w.get(f"{prefix}.skip_layer.bias"))
    h = F.pad(h, ((kernel_size - 1) // 2 * dilation,) * 2, mode="reflect")
    h = F.conv1d(h, w[f"{prefix}.stack.2.weight"], w.get(f"{prefix}.stack.2.bias"), dilation=dilation)
    h = F.leaky_relu(h, slope)
    h = F.conv1d(h, w[f"{prefix}.stack.4.weight"], w.get(f"{prefix}.stack.4.bias"))
    return h + F.conv1d(c, w[f"{prefix}.skip_layer.weight"], w.get(f"{prefix}.skip_layer.bias"))


def melgan_generator(w, c, cfg=MB_MELGAN_V2):
    """MelGANGenerator.forward (models/melgan.py:168-178)."""
    ks = cfg["kernel_size"]
    slope = cfg.get("negative_slope", 0.2)
    sk = cfg.get("stack_kernel_size", 3)
    causal = bool(cfg.get("use_causal_conv", False))
    for kind, idx, meta in melgan_layer_index(cfg):
        p = f"melgan.{idx}"
        if causal and kind == "conv_in":
            c = causal_conv1d(c, w[p + ".conv.weight"], w.get(p + ".conv.bias"), mode="reflect")
        elif causal and kind == "convt":
            c = causal_conv_transpose1d(F.leaky_relu(c, slope), w[p + ".deconv.weight"], w.get(p + ".deconv.bias"), meta[1])
        elif causal and kind == "conv_out":
            c = causal_conv1d(F.leaky_relu(c, slope), w[p + ".conv.weight"], w.get(p + ".conv.bias"), mode="reflect")
            if cfg.get("use_final_nonlinear_activation", True):
                c = torch.tanh(c)
        elif kind == "conv_in":
            c = F.conv1d(F.pad(c, ((ks - 1) // 2,) * 2, mode="reflect"), w[p + ".weight"], w.get(p + ".bias"))
        elif kind == "convt":
            _, s = meta
            c = F.conv_transpose1d(
                F.leaky_relu(c, slope),
                w[p + ".weight"],
                w.get(p + ".bias"),
                stride=s,
                padding=s // 2 + s % 2,
                output_padding=s % 2,
            )
        elif kind == "stack":
            _, j = meta
            c = melgan_residual_stack(w, p, c, sk, sk**j, slope, causal)
        else:
            c = F.leaky_relu(c, slope)
            c = F.conv1d(F.pad(c, ((ks - 1) // 2,) * 2, mode="reflect"), w[p + ".weight"], w.get(p + ".bias"))
            if cfg.get("use_final_nonlinear_activation", True):
                c = torch.tanh(c)
    return c


# --------------------------------------------------------------------------
# StyleMelGAN generator (models/style_melgan.py:22-270, layers/tade_res_block.py)
# --------------------------------------------------------------------------

STYLE_MELGAN_V1 = dict(  # egs/csmsc/voc1/conf/style_melgan.v1.yaml:31-50
    in_channels=128,
    aux_channels=80,
    channels=64,
    out_channels=1,
    kernel_size=9,
    dilation=2,
    noise_upsample_scales=(11, 2, 2, 2),
    noise_upsample_negative_slope=0.2,
    upsample_scales=(2, 2, 2, 2, 2, 2, 2, 2, 1),
    gated_function="softmax",
)


def _nearest(x, factor):
    """torch.nn.Upsample(scale_factor=factor, mode="nearest") on (B, C, T)."""
    return F.interpolate(x, scale_factor=factor, mode="nearest") if factor != 1 else F.interpolate(x, scale_factor=1, mode="nearest")


def tade_layer(w, prefix, x, c, kernel_size, upsample_factor):
    """TADELayer.forward (layers/tade_res_block.py:56-75)."""
    pad = (kernel_size - 1) // 2
    x = F.instance_norm(x)  # InstanceNorm1d: no affine, no running stats, eps 1e-5, biased variance
    c = _nearest(c, upsample_factor)
    c = F.conv1d(c, w[f"{prefix}.aux_conv.0.weight"], w.get(f"{prefix}.aux_conv.0.bias"), padding=pad)
    cg = F.conv1d(c, w[f"{prefix}.gated_conv.0.weight"], w.get(f"{prefix}.gated_conv.0.bias"), padding=pad)
    cg1, cg2 = cg.split(cg.size(1) // 2, dim=1)
    return cg1 * _nearest(x, upsample_factor) + cg2, c


def tade_res_block(w, prefix, x, c, kernel_size, dilation, upsample_factor, gated_function="softmax"):
    """TADEResBlock.forward (layers/tade_res_block.py:135-160)."""
    gate = (lambda t: torch.softmax(t, dim=1)) if gated_function == "softmax" else torch.sigmoid
    pad = (kernel_size - 1) // 2
    residual = x
    x, c = tade_layer(w, f"{prefix}.tade1", x, c, kernel_size, 1)
    x = F.conv1d(x, w[f"{prefix}.gated_conv1.weight"], w.get(f"{prefix}.gated_conv1.bias"), padding=pad)
    xa, xb = x.split(x.size(1) // 2, dim=1)
    x = gate(xa) * torch.tanh(xb)
    x, c = tade_layer(w, f"{prefix}.tade2", x, c, kernel_size, upsample_factor)
    x = F.conv1d(x, w[f"{prefix}.gated_conv2.weight"], w.get(f"{prefix}.gated_conv2.bias"), dilation=dilation, padding=pad * dilation)
    xa, xb = x.split(x.size(1) // 2, dim=1)
    x = gate(xa) * torch.tanh(xb)
    return _nearest(residual, upsample_factor) + x, c


def style_melgan_generator(w, c, z, cfg=STYLE_MELGAN_V1):
    """StyleMelGANGenerator.forward (models/style_melgan.py:140-160) with an explicit noise tensor
    z (B, in_channels, T_z): x = noise_upsample(z); x, c = block(x, c) ...; tanh(output_conv(x))."""
    slope = cfg.get("noise_upsample_negative_slope", 0.2)
    x = z
    for i, s in enumerate(cfg["noise_upsample_scales"]):
        x = F.conv_transpose1d(x, w[f"noise_upsample.{2 * i}.weight"], w.get(f"noise_upsample.{2 * i}.bias"), stride=s,
                               padding=s // 2 + s % 2, output_padding=s % 2)
        x = F.leaky_relu(x, slope)
    for i, s in enumerate(cfg["upsample_scales"]):
        x, c = tade_res_block(w, f"blocks.{i}", x, c, cfg["kernel_size"], cfg["dilation"], s, cfg.get("gated_function", "softmax"))
    pad = (cfg["kernel_size"] - 1) // 2
    return torch.tanh(F.conv1d(x, w["output_conv.0.weight"], w.get("output_conv.0.bias"), padding=pad))


# --------------------------------------------------------------------------
# PQMF (layers/pqmf.py)
# --------------------------------------------------------------------------


def kaiser_window(M, beta):
    """scipy.signal.windows.kaiser(M, beta) (symmetric) -- restated with np.i0,
    the reference calls it at layers/pqmf.py:45."""
    n = np.arange(0, M)
    alpha = (M - 1) / 2.0
    return np.i0(beta * np.sqrt(1 - ((n - alpha) / alpha) ** 2.0)) / np.i0(beta)


def pqmf_filters(subbands=4, taps=62, cutoff_ratio=0.142, beta=9.0):
    """design_prototype_filter + cosine modulation (layers/pqmf.py:14-48, 61-104).
    Returns (analysis (N,1,taps+1), synthesis (1,N,taps+1)) fp32 tensors."""
    omega_c = np.pi * cutoff_ratio
    with np.errstate(invalid="ignore", divide="ignore"):
        h_i = np.sin(omega_c * (np.arange(taps + 1) - 0.5 * taps)) / (np.pi * (np.arange(taps + 1) - 0.5 * taps))
    h_i[taps // 2] = np.cos(0) * cutoff_ratio
    h_proto = h_i * kaiser_window(taps + 1, beta)
    h_an = np.zeros((subbands, taps + 1))
    h_sy = np.zeros((subbands, taps + 1))
    for k in range(subbands):
        ph = (2 * k + 1) * (np.pi / (2 * subbands)) * (np.arange(taps + 1) - (taps / 2))
        h_an[k] = 2 * h_proto * np.cos(ph + (-1) ** k * np.pi / 4)
        h_sy[k] = 2 * h_proto * np.cos(ph - (-1) ** k * np.pi / 4)
    return torch.from_numpy(h_an).float().unsqueeze(1), torch.from_numpy(h_sy).float().unsqueeze(0)


def pqmf_analysis(x, analysis_filter):
    """PQMF.analysis (layers/pqmf.py:120-131): pad taps/2, conv 1->N, keep every N-th."""
    n, _, k = analysis_filter.shape
    y = F.conv1d(F.pad(x, ((k - 1) // 2,) * 2), analysis_filter)
    return y[..., ::n].contiguous()


def pqmf_synthesis(x, synthesis_filter):
    """PQMF.synthesis (layers/pqmf.py:133-149): zero-stuff by N with gain N
    (conv_transpose1d with the identity ``updown_filter * N``), pad, conv N->1."""
    _, n, k = synthesis_filter.shape
    B, _, T = x.shape
    z = torch.zeros(B, n, T * n, dtype=x.dtype)
    z[..., ::n] = x * n
    return F.conv1d(F.pad(z, ((k - 1) // 2,) * 2), synthesis_filter)


# --------------------------------------------------------------------------
# Parallel WaveGAN generator (models/parallel_wavegan.py:21-261, layers/upsample.py,
# layers/residual_block.py:43-140)
# --------------------------------------------------------------------------

PWG_V1 = dict(  # egs/ljspeech/voc1/conf/parallel_wavegan.v1.yaml:28-46
    in_channels=1,
    out_channels=1,
    kernel_size=3,
    layers=30,
    stacks=3,
    residual_channels=64,
    gate_channels=128,
    skip_channels=64,
    aux_channels=80,
    aux_context_window=2,
    upsample_scales=(4, 4, 4, 4),
)


def pwg_upsample_net(w, c, cfg=PWG_V1, prefix="upsample_net"):
    """ConvInUpsampleNetwork.forward (layers/upsample.py:178-194): conv_in
    (k = 2*ctx+1, no padding, no bias) then per scale: nearest repeat along T and
    a 1 x (2s+1) FIR shared by all mel bins (upsample.py:112-128)."""
    c = F.conv1d(c, w[f"{prefix}.conv_in.weight"])
    for i, s in enumerate(cfg["upsample_scales"]):
        c = torch.repeat_interleave(c, s, dim=-1)
        fir = w[f"{prefix}.upsample.up_layers.{2 * i + 1}.weight"].reshape(1, 1, -1)  # (1,1,1,2s+1)
        B, C, T = c.shape
        c = F.conv1d(c.reshape(B * C, 1, T), fir, padding=s).reshape(B, C, T)
    return c


def wavenet_residual_block(w, prefix, x, c, dilation, kernel_size=3):
    """WaveNetResidualBlock.forward (layers/residual_block.py:102-140), dropout 0."""
    residual = x
    g = F.conv1d(
        x,
        w[f"{prefix}.conv.weight"],
        w.get(f"{prefix}.conv.bias"),
        dilation=dilation,
        padding=(kernel_size - 1) // 2 * dilation,
    )
    half = g.shape[1] // 2
    xa, xb = g[:, :half], g[:, half:]
    if c is not None:
        ca = F.conv1d(c, w[f"{prefix}.conv1x1_aux.weight"])
        xa, xb = xa + ca[:, :half], xb + ca[:, half:]
    z = torch.tanh(xa) * torch.sigmoid(xb)
    s = F.conv1d(z, w[f"{prefix}.conv1x1_skip.weight"], w.get(f"{prefix}.conv1x1_skip.bias"))
    x = (F.conv1d(z, w[f"{prefix}.conv1x1_out.weight"], w.get(f"{prefix}.conv1x1_out.bias")) + residual) * math.sqrt(0.5)
    return x, s


def pwg_generator(w, z, c, cfg=PWG_V1):
    """ParallelWaveGANGenerator.forward (models/parallel_wavegan.py:144-173)."""
    c = pwg_upsample_net(w, c, cfg)
    assert c.shape[-1] == z.shape[-1]
    x = F.conv1d(z, w["first_conv.weight"], w["first_conv.bias"])
    skips = 0
    lps = cfg["layers"] // cfg["stacks"]
    for layer in range(cfg["layers"]):
        x, h = wavenet_residual_block(w, f"conv_layers.{layer}", x, c, 2 ** (layer % lps), cfg["kernel_size"])
        skips = skips + h
    skips = skips * math.sqrt(1.0 / cfg["layers"])
    x = F.relu(skips)
    x = F.conv1d(x, w["last_conv_layers.1.weight"], w["last_conv_layers.1.bias"])
    x = F.relu(x)
    x = F.conv1d(x, w["last_conv_layers.3.weight"], w["last_conv_layers.3.bias"])
    return x


# --------------------------------------------------------------------------
# STFT / mel losses (losses/stft_loss.py, losses/mel_loss.py)
# --------------------------------------------------------------------------


def hann_window(n):
    """torch.hann_window(n) (periodic): 0.5 - 0.5 cos(2 pi i / n)."""
    return 0.5 - 0.5 * torch.cos(2.0 * math.pi * torch.arange(n, dtype=torch.float64) / n)


def windowed_frames(x, fft_size, hop_size, win_length, window="hann"):
    """The frames ``torch.stft(center=True, pad_mode='reflect')`` transforms (losses/stft_loss.py:31-33):
    reflect-pad n_fft/2, frame t = padded[t*hop : t*hop+n_fft], times a window of win_length centred inside n_fft:
    periodic Hann (``window="hann"``), all ones (``window=None``) or the given (win_length,) tensor.
    x: (B, T) -> (B, frames, n_fft) in x's dtype (the window is taken to float64, then rounded to it)."""
    B, T = x.shape
    pad = fft_size // 2
    xp = F.pad(x.unsqueeze(1), (pad, pad), mode="reflect").squeeze(1)
    n_frames = 1 + T // hop_size
    idx = torch.arange(fft_size).unsqueeze(0) + hop_size * torch.arange(n_frames).unsqueeze(1)
    frames = xp[:, idx]  # (B, frames, n_fft)
    win = torch.zeros(fft_size, dtype=torch.float64)
    left = (fft_size - win_length) // 2
    if isinstance(window, torch.Tensor):
        win[left : left + win_length] = window.detach().cpu().double()
    else:
        win[left : left + win_length] = hann_window(win_length) if window == "hann" else 1.0
    return frames * win.to(x.dtype)


def stft_power(x, fft_size, hop_size, win_length, window="hann"):
    """|STFT|^2: rFFT of :func:`windowed_frames`.  x: (B, T) -> (B, frames, bins), in x's dtype (fp32 for
    parity with the reference, float64 as the exact oracle of the fp32 kernels)."""
    spec = torch.fft.rfft(windowed_frames(x, fft_size, hop_size, win_length, window), dim=-1)
    return spec.real**2 + spec.imag**2


def stft_mag(x, fft_size, hop_size, win_length, window="hann"):
    """stft() of losses/stft_loss.py:16-40: sqrt(clamp(re^2+im^2, 1e-7))."""
    return torch.sqrt(torch.clamp(stft_power(x, fft_size, hop_size, win_length, window), min=1e-7))


def mr_stft_loss(x, y, fft_sizes=(1024, 2048, 512), hop_sizes=(120, 240, 50), win_lengths=(600, 1200, 240), windows=None):
    """MultiResolutionSTFTLoss.forward (losses/stft_loss.py:146-170) -> (sc, mag).  ``windows``: one window per
    resolution as :func:`windowed_frames` takes it (default Hann)."""
    if x.dim() == 3:
        x = x.reshape(-1, x.shape[2])
        y = y.reshape(-1, y.shape[2])
    sc = 0.0
    mag = 0.0
    windows = ["hann"] * len(fft_sizes) if windows is None else windows
    for n, h, wl, w in zip(fft_sizes, hop_sizes, win_lengths, windows):
        xm = stft_mag(x, n, h, wl, w)
        ym = stft_mag(y, n, h, wl, w)
        sc = sc + torch.norm(ym - xm, p="fro") / torch.norm(ym, p="fro")  # stft_loss.py:61
        mag = mag + F.l1_loss(torch.log(ym), torch.log(xm))  # stft_loss.py:82
    return sc / len(fft_sizes), mag / len(fft_sizes)


def slaney_mel_filterbank(sr, n_fft, n_mels=80, fmin=0.0, fmax=None):
    """``librosa.filters.mel(sr, n_fft, n_mels, fmin, fmax)`` (htk=False,
    norm='slaney'), called at losses/mel_loss.py:52-58.  librosa is a third-party
    dependency absent from /root/reference (setup.py:29 ``librosa>=0.8.0``);
    this restates its published algorithm: Slaney mel scale (linear below 1 kHz,
    log above), triangular filters, area normalisation 2/(f[m+2]-f[m]).
    Returns (n_mels, 1 + n_fft//2) float32.  Parity: the matrix values are
    unpinned inside the reference itself (SURVEY.md 8c); cross-checked against
    torchaudio.functional.melscale_fbanks in tests."""
    if fmax is None:
        fmax = sr / 2.0

    def hz_to_mel(f):
        f = np.asarray(f, dtype=np.float64)
        f_sp = 200.0 / 3
        mels = f / f_sp
        min_log_hz = 1000.0
        min_log_mel = min_log_hz / f_sp
        logstep = np.log(6.4) / 27.0
        return np.where(f >= min_log_hz, min_log_mel + np.log(np.maximum(f, 1e-10) / min_log_hz) / logstep, mels)

    def mel_to_hz(m):
        m = np.asarray(m, dtype=np.float64)
        f_sp = 200.0 / 3
        freqs = f_sp * m
        min_log_hz = 1000.0
        min_log_mel = min_log_hz / f_sp
        logstep = np.log(6.4) / 27.0
        return np.where(m >= min_log_mel, min_log_hz * np.exp(logstep * (m - min_log_mel)), freqs)

    n_bins = 1 + n_fft // 2
    fftfreqs = np.linspace(0, sr / 2.0, n_bins)
    mel_f = mel_to_hz(np.linspace(hz_to_mel(fmin), hz_to_mel(fmax), n_mels + 2))
    fdiff = np.diff(mel_f)
    ramps = mel_f[:, None] - fftfreqs[None, :]
    weights = np.zeros((n_mels, n_bins))
    for i in range(n_mels):
        lower = -ramps[i] / fdiff[i]
        upper = ramps[i + 2] / fdiff[i + 1]
        weights[i] = np.maximum(0, np.minimum(lower, upper))
    enorm = 2.0 / (mel_f[2 : n_mels + 2] - mel_f[:n_mels])
    weights *= enorm[:, None]
    return weights.astype(np.float32)


def mel_spectrogram(x, melmat, fft_size=1024, hop_size=256, win_length=None, eps=1e-10, log_base=10.0, window="hann"):
    """MelSpectrogram.forward (losses/mel_loss.py:81-110).  melmat: (bins, n_mels), in x's dtype."""
    if x.dim() == 3:
        x = x.reshape(-1, x.shape[2])
    win_length = fft_size if win_length is None else win_length
    amp = torch.sqrt(torch.clamp(stft_power(x, fft_size, hop_size, win_length, window), min=eps))
    mel = torch.clamp(torch.matmul(amp, melmat), min=eps)
    if log_base is None:
        out = torch.log(mel)
    elif log_base == 2.0:
        out = torch.log2(mel)
    elif log_base == 10.0:
        out = torch.log10(mel)
    else:
        raise ValueError(log_base)
    return out.transpose(1, 2)


def mel_loss(y_hat, y, melmat, **kw):
    """MelSpectrogramLoss.forward (losses/mel_loss.py:150-165)."""
    return F.l1_loss(mel_spectrogram(y_hat, melmat, **kw), mel_spectrogram(y, melmat, **kw))


# --------------------------------------------------------------------------
# Discriminators (models/hifigan.py:270-864, models/melgan.py:260-534,
# models/parallel_wavegan.py:264-371).  Weights: effective (norm-folded) dict.
# --------------------------------------------------------------------------


def hifigan_period_discriminator(w, prefix, x, period, n_layers=5, strides=(3, 3, 3, 3, 1), slope=0.1, k0=5, k1=3):
    """HiFiGANPeriodDiscriminator.forward (hifigan.py:354-381)."""
    b, c, t = x.shape
    if t % period != 0:
        n_pad = period - (t % period)
        x = F.pad(x, (0, n_pad), "reflect")
        t += n_pad
    x = x.view(b, c, t // period, period)
    outs = []
    for i in range(n_layers):
        x = F.conv2d(x, w[f"{prefix}.convs.{i}.0.weight"], w.get(f"{prefix}.convs.{i}.0.bias"), stride=(strides[i], 1), padding=((k0 - 1) // 2, 0))
        x = F.leaky_relu(x, slope)
        outs.append(x)
    x = F.conv2d(x, w[f"{prefix}.output_conv.weight"], w.get(f"{prefix}.output_conv.bias"), padding=((k1 - 1) // 2, 0))
    outs.append(torch.flatten(x, 1, -1))
    return outs


def hifigan_scale_discriminator(w, prefix, x, strides=(2, 2, 4, 4, 1), groups=(4, 16, 16, 16, 16), ks=(15, 41, 5, 3), slope=0.1):
    """HiFiGANScaleDiscriminator.forward (hifigan.py:586-601)."""
    outs = []
    x = F.leaky_relu(F.conv1d(x, w[f"{prefix}.layers.0.0.weight"], w.get(f"{prefix}.layers.0.0.bias"), padding=(ks[0] - 1) // 2), slope)
    outs.append(x)
    for i, (s, g) in enumerate(zip(strides, groups)):
        p = f"{prefix}.layers.{i + 1}.0"
        x = F.leaky_relu(F.conv1d(x, w[p + ".weight"], w.get(p + ".bias"), stride=s, padding=(ks[1] - 1) // 2, groups=g), slope)
        outs.append(x)
    n = len(strides)
    p = f"{prefix}.layers.{n + 1}.0"
    x = F.leaky_relu(F.conv1d(x, w[p + ".weight"], w.get(p + ".bias"), padding=(ks[2] - 1) // 2), slope)
    outs.append(x)
    p = f"{prefix}.layers.{n + 2}"
    x = F.conv1d(x, w[p + ".weight"], w.get(p + ".bias"), padding=(ks[3] - 1) // 2)
    outs.append(x)
    return outs


def hifigan_msmpd(w, x, scales=3, periods=(2, 3, 5, 7, 11)):
    """HiFiGANMultiScaleMultiPeriodDiscriminator.forward (hifigan.py:850-864), v1 config:
    AvgPool1d(4, 2, padding=2) between scales (hifigan.py:758-775)."""
    outs = []
    xs = x
    for i in range(scales):
        outs.append(hifigan_scale_discriminator(w, f"msd.discriminators.{i}", xs))
        xs = F.avg_pool1d(xs, 4, 2, padding=2)
    for i, p in enumerate(periods):
        outs.append(hifigan_period_discriminator(w, f"mpd.discriminators.{i}", x, p))
    return outs


def melgan_discriminator(w, prefix, x, downsample_scales=(4, 4, 4, 4), kernel_sizes=(5, 3), channels=16, max_ch=1024, slope=0.2):
    """MelGANDiscriminator.forward (melgan.py:364-379)."""
    outs = []
    k0 = kernel_sizes[0] * kernel_sizes[1]
    x = F.leaky_relu(F.conv1d(F.pad(x, ((k0 - 1) // 2,) * 2, mode="reflect"), w[f"{prefix}.layers.0.1.weight"], w.get(f"{prefix}.layers.0.1.bias")), slope)
    outs.append(x)
    in_chs = channels
    for i, s in enumerate(downsample_scales):
        p = f"{prefix}.layers.{i + 1}.0"
        x = F.leaky_relu(F.conv1d(x, w[p + ".weight"], w.get(p + ".bias"), stride=s, padding=s * 5, groups=in_chs // 4), slope)
        outs.append(x)
        in_chs = min(in_chs * s, max_ch)
    n = len(downsample_scales)
    p = f"{prefix}.layers.{n + 1}.0"
    x = F.leaky_relu(F.conv1d(x, w[p + ".weight"], w.get(p + ".bias"), padding=(kernel_sizes[0] - 1) // 2), slope)
    outs.append(x)
    p = f"{prefix}.layers.{n + 2}"
    x = F.conv1d(x, w[p + ".weight"], w.get(p + ".bias"), padding=(kernel_sizes[1] - 1) // 2)
    outs.append(x)
    return outs


def melgan_msd(w, x, scales=3, **kw):
    """MelGANMultiScaleDiscriminator.forward (melgan.py:478-493): AvgPool1d(4,2,1,count_include_pad=False)."""
    outs = []
    for i in range(scales):
        outs.append(melgan_discriminator(w, f"discriminators.{i}", x, **kw))
        x = F.avg_pool1d(x, 4, 2, padding=1, count_include_pad=False)
    return outs


def style_melgan_discriminator(w, x, starts, window_sizes=(512, 1024, 2048, 4096),
                               pqmf_params=((1, None, None, None), (2, 62, 0.26700, 9.0), (4, 62, 0.14200, 9.0), (8, 62, 0.07949, 9.0)),
                               downsample_scales=(4, 4, 4, 1), max_ch=512):
    """StyleMelGANDiscriminator.forward (style_melgan.py:310-337).  ``starts``: the window positions in call order
    (repeats * len(window_sizes) values of ``np.random.randint(T - ws)``)."""
    outs = []
    n = len(window_sizes)
    for r, s0 in enumerate(starts):
        idx = r % n
        ws = window_sizes[idx]
        x_ = x[:, :, s0 : s0 + ws]
        if idx > 0:
            an, _ = pqmf_filters(*pqmf_params[idx])
            x_ = pqmf_analysis(x_, an)
        outs.append(melgan_discriminator(w, f"discriminators.{idx}", x_, downsample_scales=downsample_scales, max_ch=max_ch))
    return outs


def pwg_discriminator(w, x, layers=10, kernel_size=3, slope=0.2):
    """ParallelWaveGANDiscriminator.forward (parallel_wavegan.py:337-349): dilation i for layer i>0."""
    for i in range(layers - 1):
        d = 1 if i == 0 else i
        p = f"conv_layers.{2 * i}"
        x = F.leaky_relu(F.conv1d(x, w[p + ".weight"], w.get(p + ".bias"), dilation=d, padding=(kernel_size - 1) // 2 * d), slope)
    p = f"conv_layers.{2 * (layers - 1)}"
    return F.conv1d(x, w[p + ".weight"], w.get(p + ".bias"), padding=(kernel_size - 1) // 2)


def fold_spectral_norm_eval(sd):
    """Eval-mode spectral norm (no power iteration): w = w_orig / (u . (W v)); keys X.weight_orig,
    X.weight_u, X.weight_v -> X.weight."""
    out = {}
    for k, v in sd.items():
        if k.endswith(".weight_orig"):
            base = k[: -len("_orig")]
            wm = v.reshape(v.shape[0], -1)
            sigma = torch.dot(sd[base + "_u"], torch.mv(wm, sd[base + "_v"]))
            out[base] = v / sigma
        elif k.endswith(".weight_u") or (k.endswith(".weight_v") and (k[: -len("_v")] + "_orig") in sd):
            continue
        else:
            out[k] = v
    return out


# --------------------------------------------------------------------------
# GAN losses (losses/adversarial_loss.py, losses/feat_match_loss.py), default flags
# --------------------------------------------------------------------------


def generator_adv_loss(outputs, loss_type="mse", average=True):
    tot = 0.0
    for i, o in enumerate(outputs):
        o = o[-1] if isinstance(o, (list, tuple)) else o
        tot = tot + (F.mse_loss(o, torch.ones_like(o)) if loss_type == "mse" else -o.mean())
    return tot / (i + 1) if average else tot


def discriminator_adv_loss(outputs_hat, outputs, loss_type="mse", average=True):
    real = fake = 0.0
    for i, (oh, o) in enumerate(zip(outputs_hat, outputs)):
        oh = oh[-1] if isinstance(oh, (list, tuple)) else oh
        o = o[-1] if isinstance(o, (list, tuple)) else o
        if loss_type == "mse":
            real = real + F.mse_loss(o, torch.ones_like(o))
            fake = fake + F.mse_loss(oh, torch.zeros_like(oh))
        else:
            real = real - torch.mean(torch.min(o - 1, torch.zeros_like(o)))
            fake = fake - torch.mean(torch.min(-oh - 1, torch.zeros_like(oh)))
    return (real / (i + 1), fake / (i + 1)) if average else (real, fake)


def feature_match_loss(feats_hat, feats, average_by_layers=True, average_by_discriminators=True, include_final_outputs=False):
    tot = 0.0
    for i, (fh, f) in enumerate(zip(feats_hat, feats)):
        if not include_final_outputs:
            fh, f = fh[:-1], f[:-1]
        li = 0.0
        for j, (a, b) in enumerate(zip(fh, f)):
            li = li + F.l1_loss(a, b)
        if average_by_layers:
            li = li / (j + 1)
        tot = tot + li
    return tot / (i + 1) if average_by_discriminators else tot
