"""Host-side mirror of ``parallel_wavegan.layers`` (names, ctor kwargs, state-dict keys).

The ``torch.nn`` modules below are *parameter containers*: they give the same
``state_dict()`` layout as the reference (including ``weight_g``/``weight_v`` under
weight norm) but no torch arithmetic runs in ``forward`` -- every forward is a
sequence of ``libpwgb.so`` kernel calls (``ops``).
"""
import math

import numpy as np
import torch

from . import ops
from .capi import PwgbError


def effective_weight(m):
    """Weight a conv container currently represents.

    * plain parameter (after ``remove_weight_norm``): ``m.weight``
    * weight norm (``weight_g``, ``weight_v``): ``g * v / ||v||`` -- the same
      ``torch._weight_norm`` primitive ``torch.nn.utils.weight_norm`` calls in its
      pre-forward hook (which never runs here because the container is not called)
    * spectral norm (``weight_orig``, ``weight_u``): one power iteration in training
      mode, as ``torch.nn.utils.spectral_norm`` does (hifigan.py:613-621).
    """
    if hasattr(m, "weight_g"):
        return torch._weight_norm(m.weight_v, m.weight_g, 0)
    if hasattr(m, "weight_orig"):
        w = m.weight_orig
        w_mat = w.reshape(w.shape[0], -1)
        if m.training:
            with torch.no_grad():
                v = torch.nn.functional.normalize(torch.mv(w_mat.t(), m.weight_u), dim=0, eps=1e-12)
                u = torch.nn.functional.normalize(torch.mv(w_mat, v), dim=0, eps=1e-12)
                m.weight_v.copy_(v)
                m.weight_u.copy_(u)
        u, v = m.weight_u.clone(), m.weight_v.clone()
        sigma = torch.dot(u, torch.mv(w_mat, v))
        return w / sigma
    return m.weight


def activation_slope(name, params):
    """Map the reference's (nonlinear_activation, params) to a LeakyReLU slope."""
    if name == "LeakyReLU":
        return float((params or {}).get("negative_slope", 0.01))
    if name == "ReLU":
        return 0.0
    raise PwgbError(f"nonlinear_activation={name!r} has no sm_90a kernel (supported: LeakyReLU, ReLU)")


class Conv1d(torch.nn.Conv1d):
    """Conv1d with kaiming init (layers/residual_block.py:19-30)."""

    def reset_parameters(self):
        torch.nn.init.kaiming_normal_(self.weight, nonlinearity="relu")
        if self.bias is not None:
            torch.nn.init.constant_(self.bias, 0.0)


class Conv1d1x1(Conv1d):
    """1x1 Conv1d (layers/residual_block.py:33-40)."""

    def __init__(self, in_channels, out_channels, bias):
        super().__init__(in_channels, out_channels, kernel_size=1, padding=0, dilation=1, bias=bias)


class CausalConv1d(torch.nn.Module):
    """layers/causal_conv.py:12-43.  Container with the reference's ``pad`` / ``conv`` children;
    the forward is ONE conv launch with left-only padding ``(k - 1) * d`` (the reference pads both
    sides and crops the tail, which never reads the right padding)."""

    def __init__(self, in_channels, out_channels, kernel_size, dilation=1, bias=True,
                 pad="ConstantPad1d", pad_params={"value": 0.0}):
        super().__init__()
        self.pad = getattr(torch.nn, pad)((kernel_size - 1) * dilation, **pad_params)
        self.conv = torch.nn.Conv1d(in_channels, out_channels, kernel_size, dilation=dilation, bias=bias)
        self.pad_mode = pad_mode_of(pad, pad_params)
        self.left = (kernel_size - 1) * dilation
        self.dilation = dilation

    def forward(self, x, **fuse):
        return ops.conv1d(x, effective_weight(self.conv), self.conv.bias, dilation=self.dilation,
                          padding=(self.left, 0), pad_mode=self.pad_mode, **fuse)


class CausalConvTranspose1d(torch.nn.Module):
    """layers/causal_conv.py:46-79: ``deconv(pad_left_1(x))[:, :, stride:-stride]``.  The crop of
    ``stride`` samples per side is the transposed conv's own ``padding=stride``, so the forward is the
    one-frame left pad (a copy) plus ONE poly-phase launch."""

    def __init__(self, in_channels, out_channels, kernel_size, stride, bias=True,
                 pad="ReplicationPad1d", pad_params={}):
        super().__init__()
        if pad not in ("ReplicationPad1d", "ConstantPad1d", "ReflectionPad1d"):
            raise PwgbError(f"CausalConvTranspose1d: pad={pad!r} has no sm_90a kernel")
        self.pad = getattr(torch.nn, pad)((1, 0), **pad_params)
        self.deconv = torch.nn.ConvTranspose1d(in_channels, out_channels, kernel_size, stride, bias=bias)
        self.stride = stride

    def forward(self, x, pre_slope=1.0):
        # the pending activation commutes with every supported pad (lrelu(0) == 0), so it stays fused
        x = self.pad(x)  # (B, C, T + 1): data movement only
        return ops.conv_transpose1d(x.contiguous(), effective_weight(self.deconv), self.deconv.bias,
                                    stride=self.stride, padding=self.stride, pre_slope=pre_slope)


class HiFiGANResidualBlock(torch.nn.Module):
    """layers/residual_block.py:143-258: 3 x [LReLU -> conv(k, d) -> LReLU -> conv(k, 1)] + x."""

    def __init__(
        self,
        kernel_size=3,
        channels=512,
        dilations=(1, 3, 5),
        bias=True,
        use_additional_convs=True,
        nonlinear_activation="LeakyReLU",
        nonlinear_activation_params={"negative_slope": 0.1},
        use_causal_conv=False,
    ):
        super().__init__()
        assert kernel_size % 2 == 1, "Kernel size must be odd number."
        self.use_causal_conv = use_causal_conv
        self.kernel_size = kernel_size
        self.dilations = tuple(dilations)
        self.use_additional_convs = use_additional_convs
        self.slope = activation_slope(nonlinear_activation, nonlinear_activation_params)
        act = getattr(torch.nn, nonlinear_activation)
        self.convs1 = torch.nn.ModuleList()
        if use_additional_convs:
            self.convs2 = torch.nn.ModuleList()
        for d in dilations:
            if use_causal_conv:
                conv1 = CausalConv1d(channels, channels, kernel_size, dilation=d, bias=bias)
            else:
                conv1 = torch.nn.Conv1d(channels, channels, kernel_size, 1, dilation=d, bias=bias, padding=(kernel_size - 1) // 2 * d)
            self.convs1 += [torch.nn.Sequential(act(**nonlinear_activation_params), conv1)]
            if use_additional_convs:
                if use_causal_conv:
                    conv2 = CausalConv1d(channels, channels, kernel_size, dilation=1, bias=bias)
                else:
                    conv2 = torch.nn.Conv1d(channels, channels, kernel_size, dilation=1, bias=bias, padding=(kernel_size - 1) // 2)
                self.convs2 += [torch.nn.Sequential(act(**nonlinear_activation_params), conv2)]

    def forward(self, x, out=None, accumulate=False, out_scale=1.0):
        """Returns block(x); optionally ``out (+)= out_scale * block(x)`` fused into the last conv
        (inference only -- under autograd the caller sums the block outputs with ScaledSumFn)."""
        k = self.kernel_size
        n = len(self.dilations)
        for idx, d in enumerate(self.dilations):
            last = idx == n - 1
            c1 = self.convs1[idx][1]
            tail = dict(out=out, accumulate=accumulate, out_scale=out_scale) if last else {}
            if self.use_causal_conv:
                if self.use_additional_convs:
                    xt = c1(x, pre_slope=self.slope)
                    x = self.convs2[idx][1](xt, pre_slope=self.slope, residual=x, **tail)
                else:
                    x = c1(x, pre_slope=self.slope, residual=x, **tail)
            elif self.use_additional_convs:
                c2 = self.convs2[idx][1]
                w1, w2 = effective_weight(c1), effective_weight(c2)
                # inference at 32 / 64 channels: both convs in one launch, the intermediate never leaves the SM
                y = ops.resblock_pair(x, w1, c1.bias, w2, c2.bias, kernel_size=k, dilation=d, slope=self.slope, **tail)
                if y is None:
                    xt = ops.conv1d(x, w1, c1.bias, dilation=d, padding=(k - 1) // 2 * d, pre_slope=self.slope)
                    y = ops.conv1d(xt, w2, c2.bias, padding=(k - 1) // 2, pre_slope=self.slope, residual=x, **tail)
                x = y
            else:
                x = ops.conv1d(x, effective_weight(c1), c1.bias, dilation=d, padding=(k - 1) // 2 * d, pre_slope=self.slope, residual=x, **tail)
        return x


class ResidualStack(torch.nn.Module):
    """layers/residual_stack.py:13-85 (MelGAN): LReLU->ReflPad(d)->conv k3 dil d->LReLU->1x1, + 1x1 skip."""

    def __init__(
        self,
        kernel_size=3,
        channels=32,
        dilation=1,
        bias=True,
        nonlinear_activation="LeakyReLU",
        nonlinear_activation_params={"negative_slope": 0.2},
        pad="ReflectionPad1d",
        pad_params={},
        use_causal_conv=False,
    ):
        super().__init__()
        self.use_causal_conv = use_causal_conv
        if not use_causal_conv:
            assert (kernel_size - 1) % 2 == 0, "Not support even number kernel size."
        self.pad_mode = pad_mode_of(pad, pad_params)
        self.kernel_size = kernel_size
        self.dilation = dilation
        self.slope = activation_slope(nonlinear_activation, nonlinear_activation_params)
        act = getattr(torch.nn, nonlinear_activation)
        if not use_causal_conv:
            self.stack = torch.nn.Sequential(
                act(**nonlinear_activation_params),
                getattr(torch.nn, pad)((kernel_size - 1) // 2 * dilation, **pad_params),
                torch.nn.Conv1d(channels, channels, kernel_size, dilation=dilation, bias=bias),
                act(**nonlinear_activation_params),
                torch.nn.Conv1d(channels, channels, 1, bias=bias),
            )
        else:
            self.stack = torch.nn.Sequential(
                act(**nonlinear_activation_params),
                CausalConv1d(channels, channels, kernel_size, dilation=dilation, bias=bias, pad=pad, pad_params=pad_params),
                act(**nonlinear_activation_params),
                torch.nn.Conv1d(channels, channels, 1, bias=bias),
            )
        self.skip_layer = torch.nn.Conv1d(channels, channels, 1, bias=bias)

    def forward(self, c):
        k, d = self.kernel_size, self.dilation
        sk = self.skip_layer
        if self.use_causal_conv:
            c2 = self.stack[3]
            h = self.stack[1](c, pre_slope=self.slope)
        else:
            c1, c2 = self.stack[2], self.stack[4]
            h = ops.conv1d(c, effective_weight(c1), c1.bias, dilation=d, padding=(k - 1) // 2 * d, pad_mode=self.pad_mode, pre_slope=self.slope)
        s = ops.conv1d(c, effective_weight(sk), sk.bias)
        return ops.conv1d(h, effective_weight(c2), c2.bias, pre_slope=self.slope, residual=s)


def pad_mode_of(pad, pad_params):
    if pad == "ReflectionPad1d":
        return "reflect"
    if pad == "ReplicationPad1d":
        return "replicate"
    if pad == "ConstantPad1d" and float((pad_params or {}).get("value", 0.0)) == 0.0:
        return "zero"
    raise PwgbError(f"pad={pad!r} {pad_params!r} has no sm_90a kernel (supported: ReflectionPad1d, ReplicationPad1d, zero ConstantPad1d)")


def design_prototype_filter(taps=62, cutoff_ratio=0.142, beta=9.0):
    """Kaiser-window prototype low-pass for the PQMF bank (layers/pqmf.py:14-48); host-side
    float64 numpy like the reference (``scipy.signal.kaiser`` == np.kaiser's definition)."""
    assert taps % 2 == 0, "The number of taps mush be even number."
    assert 0.0 < cutoff_ratio < 1.0, "Cutoff ratio must be > 0.0 and < 1.0."
    omega_c = np.pi * cutoff_ratio
    n = np.arange(taps + 1) - 0.5 * taps
    with np.errstate(invalid="ignore", divide="ignore"):
        h_i = np.sin(omega_c * n) / (np.pi * n)
    h_i[taps // 2] = np.cos(0) * cutoff_ratio
    M = taps + 1
    alpha = (M - 1) / 2.0
    w = np.i0(beta * np.sqrt(1 - ((np.arange(M) - alpha) / alpha) ** 2.0)) / np.i0(beta)
    return h_i * w


class PQMF(torch.nn.Module):
    """Pseudo-QMF analysis / synthesis (layers/pqmf.py:51-149).

    analysis  = one strided FIR launch (the reference's stride-N identity
    ``updown_filter`` conv is the ``stride`` of the kernel -- an exact index op);
    synthesis = one poly-phase transposed FIR launch (no zero-stuffed tensor)."""

    def __init__(self, subbands=4, taps=62, cutoff_ratio=0.142, beta=9.0):
        super().__init__()
        h_proto = design_prototype_filter(taps, cutoff_ratio, beta)
        h_analysis = np.zeros((subbands, len(h_proto)))
        h_synthesis = np.zeros((subbands, len(h_proto)))
        for k in range(subbands):
            ph = (2 * k + 1) * (np.pi / (2 * subbands)) * (np.arange(taps + 1) - (taps / 2))
            h_analysis[k] = 2 * h_proto * np.cos(ph + (-1) ** k * np.pi / 4)
            h_synthesis[k] = 2 * h_proto * np.cos(ph - (-1) ** k * np.pi / 4)
        self.register_buffer("analysis_filter", torch.from_numpy(h_analysis).float().unsqueeze(1))
        self.register_buffer("synthesis_filter", torch.from_numpy(h_synthesis).float().unsqueeze(0))
        updown_filter = torch.zeros((subbands, subbands, subbands)).float()
        for k in range(subbands):
            updown_filter[k, k, 0] = 1.0
        self.register_buffer("updown_filter", updown_filter)
        self.subbands = subbands
        self.taps = taps

    def analysis(self, x):
        """(B, 1, T) -> (B, subbands, T // subbands)."""
        return ops.conv1d(x, self.analysis_filter, None, stride=self.subbands, padding=self.taps // 2)

    def synthesis(self, x):
        """(B, subbands, T // subbands) -> (B, 1, T).  Transposed-FIR form of
        ``conv1d(pad(zero_stuff(x) * N), synthesis_filter)``: w[b, 0, k'] = N * h[b, taps - k']."""
        n = self.subbands
        w = (self.synthesis_filter[0].flip(-1) * float(n)).unsqueeze(1).contiguous()  # (N, 1, taps+1)
        return ops.conv_transpose1d(x, w, None, stride=n, padding=self.taps // 2, output_padding=n - 1)


# --------------------------------------------------------------------------
# Parallel WaveGAN blocks (layers/residual_block.py:43-140, layers/upsample.py)
# --------------------------------------------------------------------------


class WaveNetResidualBlock(torch.nn.Module):
    """layers/residual_block.py:43-140.  ``forward(x, c, skips)`` runs the fused layer and
    accumulates the skip branch in place; it returns the new residual stream."""

    def __init__(
        self,
        kernel_size=3,
        residual_channels=64,
        gate_channels=128,
        skip_channels=64,
        aux_channels=80,
        dropout=0.0,
        dilation=1,
        bias=True,
        use_causal_conv=False,
    ):
        super().__init__()
        if use_causal_conv:
            raise PwgbError("WaveNetResidualBlock(use_causal_conv=True) has no sm_90a kernel yet")
        if dropout != 0.0:
            raise PwgbError("WaveNetResidualBlock(dropout>0) has no sm_90a kernel (all reference configs use 0.0)")
        assert (kernel_size - 1) % 2 == 0, "Not support even number kernel size."
        self.dropout = dropout
        self.dilation = dilation
        self.aux_channels = aux_channels
        self.use_causal_conv = use_causal_conv
        padding = (kernel_size - 1) // 2 * dilation
        self.conv = Conv1d(residual_channels, gate_channels, kernel_size, padding=padding, dilation=dilation, bias=bias)
        self.conv1x1_aux = Conv1d1x1(aux_channels, gate_channels, bias=False) if aux_channels > 0 else None
        gate_out_channels = gate_channels // 2
        self.conv1x1_out = Conv1d1x1(gate_out_channels, residual_channels, bias=bias)
        self.conv1x1_skip = Conv1d1x1(gate_out_channels, skip_channels, bias=bias)
        self._cache = {}

    def forward(self, x, c, skips=None):
        """x: (B, R, T); c: (B, aux[_padded], T) or None; skips: (B, S, T) accumulated in place.
        Returns (x_out, skips) -- with ``skips=None`` a fresh zero tensor is used so that the pair
        equals the reference's ``(x, s)`` (layers/residual_block.py:140)."""
        aux = self.conv1x1_aux
        if torch.is_grad_enabled() and (x.requires_grad or next(self.parameters()).requires_grad):
            if skips is not None:
                raise PwgbError("in-place skip accumulation is inference-only; use the returned skip tensor under autograd")
            return self._forward_train(x, c)  # (x_out, s): the reference's pair, differentiable
        if skips is None:
            skips = torch.zeros((x.shape[0], self.conv1x1_skip.out_channels, x.shape[2]), device=x.device, dtype=x.dtype)
        x_out = ops.wavenet_layer(
            x, c,
            effective_weight(self.conv), self.conv.bias,
            effective_weight(aux) if aux is not None else None,
            effective_weight(self.conv1x1_skip), self.conv1x1_skip.bias,
            effective_weight(self.conv1x1_out), self.conv1x1_out.bias,
            self.dilation, skips, self.aux_channels, cache=self._cache,
            key=ops.param_key(self.conv, aux, self.conv1x1_skip, self.conv1x1_out),
        )
        return x_out, skips


def _wn_train(self, x, c):
    """Differentiable composition of the layer (every op's forward and backward is a libpwgb kernel):
    g = conv_dil(x) + W_aux c ; z = gate(g) ; s = W_skip z ; x' = (W_out z + x) * sqrt(0.5)."""
    from .autograd import GateFn

    k = self.conv.kernel_size[0]
    g = ops.conv1d(x, effective_weight(self.conv), self.conv.bias, dilation=self.dilation, padding=(k - 1) // 2 * self.dilation)
    if c is not None:
        wa = effective_weight(self.conv1x1_aux)
        if c.shape[1] != wa.shape[1]:  # conditioning stored channel-padded (zeros): pad the weight columns
            wa = torch.nn.functional.pad(wa, (0, 0, 0, c.shape[1] - wa.shape[1]))
        g = ops.conv1d(c, wa, None, residual=g)
    z = GateFn.apply(g)
    s = ops.conv1d(z, effective_weight(self.conv1x1_skip), self.conv1x1_skip.bias)
    xo = ops.conv1d(z, effective_weight(self.conv1x1_out), self.conv1x1_out.bias, residual=x, out_scale=math.sqrt(0.5))
    return xo, s


WaveNetResidualBlock._forward_train = _wn_train


class Stretch2d(torch.nn.Module):
    """layers/upsample.py:16-45 (parameter-free; fused into the FIR stage kernel)."""

    def __init__(self, x_scale, y_scale, mode="nearest"):
        super().__init__()
        if mode != "nearest" or y_scale != 1:
            raise PwgbError("Stretch2d: only nearest time-axis stretching has an sm_90a kernel")
        self.x_scale, self.y_scale, self.mode = x_scale, y_scale, mode


class Conv2d(torch.nn.Conv2d):
    """layers/upsample.py:48-59: box-filter initialised Conv2d (container for the FIR taps)."""

    def reset_parameters(self):
        self.weight.data.fill_(1.0 / np.prod(self.kernel_size))
        if self.bias is not None:
            torch.nn.init.constant_(self.bias, 0.0)


class UpsampleNetwork(torch.nn.Module):
    """layers/upsample.py:62-128."""

    def __init__(self, upsample_scales, nonlinear_activation=None, nonlinear_activation_params={},
                 interpolate_mode="nearest", freq_axis_kernel_size=1, use_causal_conv=False):
        super().__init__()
        if use_causal_conv or nonlinear_activation is not None or freq_axis_kernel_size != 1:
            raise PwgbError("UpsampleNetwork: causal / nonlinear / freq-axis-kernel variants have no sm_90a kernel yet")
        self.use_causal_conv = use_causal_conv
        self.upsample_scales = list(upsample_scales)
        self.up_layers = torch.nn.ModuleList()
        for scale in upsample_scales:
            self.up_layers += [Stretch2d(scale, 1, interpolate_mode)]
            self.up_layers += [Conv2d(1, 1, kernel_size=(1, scale * 2 + 1), padding=(0, scale), bias=False)]

    def forward(self, c, out_channels=None):
        """(B, C, T') -> (B, C [padded to out_channels], T' * prod(scales))."""
        n = len(self.upsample_scales)
        for i, s in enumerate(self.upsample_scales):
            fir = effective_weight(self.up_layers[2 * i + 1])
            oc = out_channels if i == n - 1 else None
            if torch.is_grad_enabled() and (c.requires_grad or fir.requires_grad):
                from .autograd import UpsampleFirFn

                c = UpsampleFirFn.apply(c, fir, s, oc)
            else:
                c = ops.upsample_fir(c, fir, s, out_channels=oc)
        return c


class ConvInUpsampleNetwork(torch.nn.Module):
    """layers/upsample.py:131-194."""

    def __init__(self, upsample_scales, nonlinear_activation=None, nonlinear_activation_params={},
                 interpolate_mode="nearest", freq_axis_kernel_size=1, aux_channels=80, aux_context_window=0,
                 use_causal_conv=False):
        super().__init__()
        if use_causal_conv:
            raise PwgbError("ConvInUpsampleNetwork(use_causal_conv=True) has no sm_90a kernel yet")
        self.aux_context_window = aux_context_window
        self.use_causal_conv = False
        kernel_size = 2 * aux_context_window + 1
        self.conv_in = Conv1d(aux_channels, aux_channels, kernel_size=kernel_size, bias=False)
        self.upsample = UpsampleNetwork(upsample_scales, nonlinear_activation, nonlinear_activation_params,
                                        interpolate_mode, freq_axis_kernel_size, use_causal_conv)

    def forward(self, c, out_channels=None):
        c_ = ops.conv1d(c, effective_weight(self.conv_in), None)  # no padding: input already carries the context
        return self.upsample(c_, out_channels=out_channels)


# --------------------------------------------------------------------------
# StyleMelGAN blocks (layers/tade_res_block.py)
# --------------------------------------------------------------------------


class TADELayer(torch.nn.Module):
    """layers/tade_res_block.py:13-75: x_norm modulated by two convs of the (upsampled) conditioning."""

    def __init__(self, in_channels=64, aux_channels=80, kernel_size=9, bias=True, upsample_factor=2, upsample_mode="nearest"):
        super().__init__()
        if upsample_mode != "nearest":
            raise PwgbError(f"TADELayer: upsample_mode={upsample_mode!r} has no sm_90a kernel (nearest only)")
        self.norm = torch.nn.InstanceNorm1d(in_channels)  # parameter-free container (eps read from it)
        self.aux_conv = torch.nn.Sequential(
            torch.nn.Conv1d(aux_channels, in_channels, kernel_size, 1, bias=bias, padding=(kernel_size - 1) // 2))
        self.gated_conv = torch.nn.Sequential(
            torch.nn.Conv1d(in_channels, in_channels * 2, kernel_size, 1, bias=bias, padding=(kernel_size - 1) // 2))
        self.upsample = torch.nn.Upsample(scale_factor=upsample_factor, mode=upsample_mode)
        self.upsample_factor = int(upsample_factor)
        self.pad = (kernel_size - 1) // 2

    def forward(self, x, c, pre_slope=1.0):
        """(B, C, T), (B, aux, T') -> (B, C, T * f), (B, C, T' * f); ``pre_slope``: pending LeakyReLU on x."""
        f = self.upsample_factor
        xn = ops.instance_norm(x, eps=self.norm.eps, pre_slope=pre_slope)
        c = ops.upsample_nearest(c, f)
        ac, gc = self.aux_conv[0], self.gated_conv[0]
        c = ops.conv1d(c, effective_weight(ac), ac.bias, padding=self.pad)
        cg = ops.conv1d(c, effective_weight(gc), gc.bias, padding=self.pad)
        return ops.tade_combine(cg, xn, f), c


class TADEResBlock(torch.nn.Module):
    """layers/tade_res_block.py:78-160."""

    def __init__(self, in_channels=64, aux_channels=80, kernel_size=9, dilation=2, bias=True, upsample_factor=2,
                 upsample_mode="nearest", gated_function="softmax"):
        super().__init__()
        if gated_function not in ("softmax", "sigmoid"):
            raise ValueError(f"{gated_function} is not supported.")
        self.tade1 = TADELayer(in_channels, aux_channels, kernel_size, bias, 1, upsample_mode)
        self.gated_conv1 = torch.nn.Conv1d(in_channels, in_channels * 2, kernel_size, 1, bias=bias, padding=(kernel_size - 1) // 2)
        self.tade2 = TADELayer(in_channels, in_channels, kernel_size, bias, upsample_factor, upsample_mode)
        self.gated_conv2 = torch.nn.Conv1d(in_channels, in_channels * 2, kernel_size, 1, bias=bias, dilation=dilation,
                                           padding=(kernel_size - 1) // 2 * dilation)
        self.upsample = torch.nn.Upsample(scale_factor=upsample_factor, mode=upsample_mode)
        self.gated_function_name = gated_function
        self.upsample_factor = int(upsample_factor)
        self.pad = (kernel_size - 1) // 2
        self.dilation = dilation

    def forward(self, x, c):
        """(B, C, T), (B, aux, T) -> (B, C, T * f), (B, C, T * f)."""
        residual = x
        x, c = self.tade1(x, c)
        g1 = self.gated_conv1
        x = ops.tade_gate(ops.conv1d(x, effective_weight(g1), g1.bias, padding=self.pad), None, 1, self.gated_function_name)
        x, c = self.tade2(x, c)
        g2 = self.gated_conv2
        x = ops.conv1d(x, effective_weight(g2), g2.bias, dilation=self.dilation, padding=self.pad * self.dilation)
        # gate + nearest-upsampled residual in one pass
        return ops.tade_gate(x, residual, self.upsample_factor, self.gated_function_name), c


# --------------------------------------------------------------------------
# layers/layer_norm.py, layers/duration_predictor.py, layers/length_regulator.py
# --------------------------------------------------------------------------
class LayerNorm(torch.nn.LayerNorm):
    """layers/layer_norm.py:10-40: torch.nn.LayerNorm(nout, eps=1e-12) over dimension ``dim``.  dim = 1 of a
    (B, C, T) tensor is pwgb_channel_layernorm_forward on the channel-major layout; dim = -1 of (N, C) is the same
    kernel on the (N, C, 1) view."""

    def __init__(self, nout, dim=-1):
        super().__init__(nout, eps=1e-12)
        self.dim = dim

    def forward(self, x):
        if self.dim == 1 and x.dim() == 3:
            return ops.channel_layer_norm(x, self.weight, self.bias, self.eps)
        if self.dim in (-1, x.dim() - 1):
            shape = x.shape
            y = ops.channel_layer_norm(x.reshape(-1, shape[-1], 1), self.weight, self.bias, self.eps)
            return y.reshape(shape)
        raise PwgbError(f"LayerNorm(dim={self.dim}) of a {x.dim()}-D tensor has no sm_90a kernel (dim=1 of (B, C, T) or the last dim)")


class DurationPredictor(torch.nn.Module):
    """layers/duration_predictor.py:17-116 (FastSpeech duration predictor).  Each layer is Conv1d (k, "same" padding)
    with the ReLU fused into its epilogue, LayerNorm over channels (its own kernel: it spans the conv's 128-column
    chunks) and dropout; the final Linear(n_chans, 1) runs as a k = 1 conv with one output channel.  ``forward`` takes
    (B, Tmax, idim) like the reference; the channel-major (B, idim, Tmax) tensor the generators hold, transposed, is
    read in place."""

    def __init__(self, idim, n_layers=2, n_chans=384, kernel_size=3, dropout_rate=0.1, offset=1.0):
        super().__init__()
        self.offset = offset
        self.conv = torch.nn.ModuleList()
        for idx in range(n_layers):
            in_chans = idim if idx == 0 else n_chans
            self.conv += [
                torch.nn.Sequential(
                    torch.nn.Conv1d(in_chans, n_chans, kernel_size, stride=1, padding=(kernel_size - 1) // 2),
                    torch.nn.ReLU(),
                    LayerNorm(n_chans, dim=1),
                    torch.nn.Dropout(dropout_rate),
                )
            ]
        self.linear = torch.nn.Linear(n_chans, 1)

    def _log_durations(self, xs, x_masks):
        """(B, Tmax, idim) -> (B, Tmax) log-domain durations (duration_predictor.py:71-77)."""
        if x_masks is not None:
            raise PwgbError("DurationPredictor: x_masks has no sm_90a kernel (the generators never pass one)")
        h = xs.transpose(1, -1)  # (B, idim, Tmax)
        for f in self.conv:
            conv, ln, drop = f[0], f[2], f[3]
            if h.shape[1] != conv.in_channels:
                raise PwgbError(f"DurationPredictor: input has {h.shape[1]} channels, the first conv expects {conv.in_channels}")
            h = ops.conv1d(h, effective_weight(conv), conv.bias, padding=conv.padding[0], post_act="lrelu", post_slope=0.0)
            h = ln(h)
            h = ops.dropout(h, drop.p, self.training)
        lin = self.linear
        w = lin.weight.reshape(1, lin.in_features, 1)
        if ops._needs_grad(h, w, lin.bias):
            from .autograd import conv1d as conv1d_grad

            y = conv1d_grad(h, w, lin.bias)
        else:
            y = ops.conv1d_raw(h, w, lin.bias)
        return y.reshape(y.shape[0], y.shape[2])

    def forward(self, xs, x_masks=None):
        """Log-domain durations (B, Tmax) (duration_predictor.py:90-102)."""
        return self._log_durations(xs, x_masks)

    def inference(self, xs, x_masks=None):
        """int64 durations clamp(round(exp(x) - offset), min=0) (B, Tmax) (duration_predictor.py:104-116)."""
        ds, _ = ops.duration_round(self._log_durations(xs, x_masks), self.offset, zero_rule=False)
        return ds


class LengthRegulator(torch.nn.Module):
    """layers/length_regulator.py:47-98: row b repeats xs[b, j] ds[b, j] times and the rows are zero-padded to the
    largest total.  When the whole batch sums to zero, rows summing to zero are set to all ones first, in place on
    ``ds`` (length_regulator.py:87-95).  The repeat is the embed kernel with xs as the table (row b * Tmax + j); sizing
    the output reads the row totals on the host (see ``ops.regulated_length``).  Under autograd the table gradient goes
    through pwgb_symbol_embed_backward, which serves at most 8192 table rows: B * Tmax <= 8192 (larger raises
    PwgbError).  The generators regulate their embedding tables directly and do not go through this module."""

    def __init__(self, pad_value=0.0):
        super().__init__()
        self.pad_value = pad_value

    def forward(self, xs, ds, alpha=1.0):
        """xs (B, Tmax, D), ds (B, Tmax) int64 -> (B, T*, D)."""
        if alpha != 1.0:
            raise PwgbError("LengthRegulator: alpha != 1.0 has no sm_90a kernel (the generators never pass it)")
        if self.pad_value != 0.0:
            raise PwgbError("LengthRegulator: pad_value != 0 has no sm_90a kernel")
        B, S, D = xs.shape
        _, totals = ops.duration_round(None, ds=ds)
        if B * S == 0:
            return xs.new_zeros((B, 0, D))
        idx = torch.arange(B * S, device=xs.device, dtype=torch.int64).reshape(B, 1, S)
        y = ops.symbol_embed(idx, xs.reshape(B * S, D), ds=ds, t_out=ops.regulated_length(totals))
        return y.transpose(1, 2)


class VQCodebook(torch.nn.Module):
    """layers/vector_quantize_codebook.py:17-75: the (num_embeds, embed_dim) codebook ``embedding.weight``, initialised
    U(-1 / num_embeds, 1 / num_embeds).  The search reads the channel-major z_e in place (pwgb_vq_forward)."""

    def __init__(self, num_embeds, embed_dim):
        super().__init__()
        self.embedding = torch.nn.Embedding(num_embeds, embed_dim)
        self.embedding.weight.data.uniform_(-1.0 / num_embeds, 1.0 / num_embeds)

    def forward(self, z_e):
        """z_e (B, embed_dim, T) -> nearest-code indices (B, T)."""
        from .functions import vector_quantize

        return vector_quantize(z_e.transpose(2, 1), self.embedding.weight)

    def straight_through(self, z_e):
        """z_e (B, embed_dim, T) -> (z_q_st, z_q), both (B, embed_dim, T): the codes for the decoder, whose gradient goes
        straight through to z_e, and the same codes for the quantisation loss, whose gradient goes to the codebook."""
        z_q_st, z_q, _ = ops.vq(z_e, self.embedding.weight)
        return z_q_st, z_q
