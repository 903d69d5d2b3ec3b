"""Chunked CPU restatement of streaming a centred Parallel WaveGAN with a fixed lookahead (TEST INFRASTRUCTURE), on top of
``oracle/ref_causal_pwg.py``.  It carries the same state as ``parallelwavegan_b200.streaming.PWGLookaheadStream``,
explicitly and in plain tensors.

Every signal runs in "delayed time": a chunk of signal s holds its samples [F * rate_s - look_s, (F + n) * rate_s -
look_s), F being the frames pushed before and look_s the lookahead summed along the layers in front of s:

* conv_in (kernel 2 acw + 1, a valid conv over the ReplicationPad1d(acw) input) on [the last 2 acw frames | chunk]:
  acw frames.  A fresh item's history is its first frame replicated; the flush pushes its last frame replicated, the
  right edge of the pad;
* each FIR stage (scale s): output frame j reads input frames j - 1, j, j + 1, so on [2 history frames | chunk] it is the
  causal stage labelled one frame earlier: look <- look * s + s.  The last stage's lookahead is ``look_c``;
* WaveNet layer l (dilation d_l, kernel K) on [(K - 1) d_l history rows | chunk] is the causal tap pattern with its
  output labelled (K - 1) / 2 d_l samples earlier: it ends at look_x + D_l, D_l = sum_{j <= l} (K - 1) / 2 d_j, look_x
  being the lookahead of first_conv's output.  The conditioning enters a layer through its 1x1 aux conv, at the
  layer's output rows, so layer 0 needs it at look_x + D_0 >= look_c: look_x = max(look_c - D_0, 0) is the tightest;
* the noise is pushed with its frames and runs through a ``look_x``-sample delay line in front of first_conv;
* layer l's residual is its input read (K - 1) / 2 d_l rows back; its conditioning is read off_l = look_x + D_l -
  look_c rows back from a window of the last off_L conditioning rows, and its skip is added at columns
  [off_L - off_l, off_L - off_l + T) of an (off_L + T)-column accumulator whose first T columns are complete after the
  last layer, which then shifts by T;
* the output head is pointwise: ``delay`` = look_x + D_L (PWG v1: 851 + 3069 = 3920 samples).

The whole-signal forward reads zero padding before sample 0 and after the end of every signal, so every signal a later
layer reads is stored as zero outside [0, T_s) (the mask; the end is set by the flush), and so is the output.  ``flush``
pushes ceil(delay / hop) frames with the end set and returns the first ``delay`` samples, so that cat(pushes, flush) ==
[zeros(delay) | whole_utterance].

The knobs inject plausible mistakes, so that the tests can show each one is caught: ``no_mask``, ``undelayed_res`` (the
residual read at the layer's own rows), ``unaligned_skips`` (every layer adds its skip at the same columns),
``undelayed_cond`` (every layer reads the newest conditioning rows), ``undelayed_noise`` (no delay line) and
``flush_zero_edge`` (the flush pushes zero frames instead of the replicated last frame)."""
import math

import torch
import torch.nn.functional as F

from .ref_pwg_stream import _fir_prefix
from .ref_pwg_stream import whole_utterance as _whole
from .ref_stream import drive, keep
from .ref_stream import measured_lookahead as _measured


def whole_utterance(w, z, c, cfg):
    """``ParallelWaveGANGenerator.inference`` (centred) for a batch of whole utterances c (B, aux, T'), z (B, 1, T' * hop)"""
    return _whole(w, z, c, cfg)


def plan(cfg):
    """(conv_in frames of lookahead, [lookahead after each FIR stage], look_x, [D_l], delay) of a centred generator
    config"""
    kind = cfg.get("upsample_net", "ConvInUpsampleNetwork")
    look = cfg.get("aux_context_window", 0) if kind == "ConvInUpsampleNetwork" else 0
    look_in, looks = look, []
    for s in cfg["upsample_scales"]:
        look = look * s + s
        looks.append(look)
    K = cfg["kernel_size"]
    lps = cfg["layers"] // cfg["stacks"]
    D, acc = [], 0
    for l in range(cfg["layers"]):
        acc += (K - 1) // 2 * 2 ** (l % lps)
        D.append(acc)
    look_x = max(look - D[0], 0)
    return look_in, looks, look_x, D, look_x + D[-1]


class PWGLookaheadRef:
    """push(c (B, aux, n), z (B, 1, n * hop)) -> (B, out_channels, n * hop); flush() -> (B, out_channels, delay)."""

    def __init__(self, w, cfg, batch=1, dtype=torch.float64, no_mask=False, undelayed_res=False, unaligned_skips=False,
                 undelayed_cond=False, undelayed_noise=False, flush_zero_edge=False):
        kind = cfg.get("upsample_net", "ConvInUpsampleNetwork")
        assert not cfg.get("use_causal_conv") and kind in ("ConvInUpsampleNetwork", "UpsampleNetwork"), cfg
        assert cfg["kernel_size"] % 2 == 1, cfg
        self.w = {k: v.to(dtype) for k, v in w.items()}
        self.cfg, self.B, self.dtype = cfg, batch, dtype
        self.no_mask, self.undelayed_res, self.unaligned_skips = no_mask, undelayed_res, unaligned_skips
        self.undelayed_cond, self.undelayed_noise, self.flush_zero_edge = undelayed_cond, undelayed_noise, flush_zero_edge
        self.conv_in = kind == "ConvInUpsampleNetwork"
        self.acw = cfg.get("aux_context_window", 0) if self.conv_in else 0
        self.scales = list(cfg["upsample_scales"])
        self.hop = math.prod(self.scales)
        self.K = cfg["kernel_size"]
        lps = cfg["layers"] // cfg["stacks"]
        self.dil = [2 ** (l % lps) for l in range(cfg["layers"])]
        self.look_in, self.looks, self.look_x, self.D, self.delay = plan(cfg)
        self.look_c = self.looks[-1]
        self.off = [self.look_x + d - self.look_c for d in self.D]  # conditioning rows behind the newest, per layer
        self.reset()

    def reset(self):
        cfg, B = self.cfg, self.B
        z = lambda C, H: torch.zeros(B, C, H, dtype=self.dtype)  # noqa: E731
        A, R = cfg["aux_channels"], cfg["residual_channels"]
        self.cin = None  # set from the first frame on the first push
        self.fir = [z(A, 2) for _ in self.scales]
        self.zh = z(cfg.get("in_channels", 1), self.look_x)
        self.ch = z(A, self.off[-1])
        self.wn = [z(R, (self.K - 1) * d) for d in self.dil]
        self.sk = z(cfg["skip_channels"], self.off[-1])
        self.frame, self.end = 0, None

    def _mask(self, y, rate, look):
        if self.no_mask:
            return y
        pos = self.frame * rate - look + torch.arange(y.shape[-1])
        keep = pos >= 0
        if self.end is not None:
            keep &= pos < self.end * rate
        return torch.where(keep, y, torch.zeros((), dtype=y.dtype))

    def _layer(self, l, x, cwin, sw):
        w, K, d = self.w, self.K, self.dil[l]
        p = f"conv_layers.{l}"
        W, T = self.off[-1], x.shape[-1]
        H = (K - 1) * d
        xp = torch.cat([self.wn[l], x], -1)
        self.wn[l] = keep(xp, H)
        g = F.conv1d(xp, w[f"{p}.conv.weight"], w.get(f"{p}.conv.bias"), dilation=d)
        c0 = W if self.undelayed_cond else W - self.off[l]
        ca = F.conv1d(cwin[..., c0:c0 + T], w[f"{p}.conv1x1_aux.weight"])
        half = g.shape[1] // 2
        zt = torch.tanh(g[:, :half] + ca[:, :half]) * torch.sigmoid(g[:, half:] + ca[:, half:])
        s = F.conv1d(zt, w[f"{p}.conv1x1_skip.weight"], w.get(f"{p}.conv1x1_skip.bias"))
        res = x if self.undelayed_res else xp[..., H - (K - 1) // 2 * d:H - (K - 1) // 2 * d + T]
        xo = (F.conv1d(zt, w[f"{p}.conv1x1_out.weight"], w.get(f"{p}.conv1x1_out.bias")) + res) * math.sqrt(0.5)
        k0 = 0 if self.unaligned_skips else W - self.off[l]
        sw[..., k0:k0 + T] += s
        return self._mask(xo, self.hop, self.look_x + self.D[l])

    def push(self, c, z):
        w, cfg = self.w, self.cfg
        c, z = c.to(self.dtype), z.to(self.dtype)
        n = c.shape[-1]
        if self.conv_in:
            P = 2 * self.acw
            if self.cin is None:
                self.cin = c[:, :, :1].expand(-1, -1, P).clone()
            x = torch.cat([self.cin, c], -1)
            self.cin = keep(x, P)
            c = self._mask(F.conv1d(x, w["upsample_net.conv_in.weight"]), 1, self.look_in)
        prefix = _fir_prefix(cfg)
        for i, s in enumerate(self.scales):
            x = torch.cat([self.fir[i], c], -1)  # frames -2, -1, 0 .. n-1 of the stage input
            self.fir[i] = x[:, :, -2:]
            B, C, T = x.shape
            fir = w[f"{prefix}.up_layers.{2 * i + 1}.weight"].reshape(1, 1, -1)
            c = F.conv1d(torch.repeat_interleave(x, s, dim=-1).reshape(B * C, 1, T * s), fir).reshape(B, C, (T - 2) * s)
            c = self._mask(c, math.prod(self.scales[:i + 1]), self.looks[i])
        T = c.shape[-1]
        cwin = torch.cat([self.ch, c], -1)
        self.ch = keep(cwin, self.off[-1])
        zw = torch.cat([self.zh, z], -1)
        self.zh = keep(zw, self.look_x)
        zd = z if self.undelayed_noise else zw[..., :T]
        x = self._mask(F.conv1d(zd, w["first_conv.weight"], w["first_conv.bias"]), self.hop, self.look_x)
        sw = torch.cat([self.sk, torch.zeros(self.B, self.sk.shape[1], T, dtype=self.dtype)], -1)
        for l in range(cfg["layers"]):
            x = self._layer(l, x, cwin, sw)
        self.sk = sw[..., T:]
        h = F.relu(sw[..., :T] * math.sqrt(1.0 / cfg["layers"]))
        h = F.relu(F.conv1d(h, w["last_conv_layers.1.weight"], w["last_conv_layers.1.bias"]))
        y = self._mask(F.conv1d(h, w["last_conv_layers.3.weight"], w["last_conv_layers.3.bias"]), self.hop, self.delay)
        self.frame += n
        return y

    def flush(self):
        self.end = self.frame
        n = -(-self.delay // self.hop)
        A = self.cfg["aux_channels"]
        if self.acw and not self.flush_zero_edge:
            c = self.cin[:, :, -1:].expand(-1, -1, n)
        else:
            c = torch.zeros(self.B, A, n, dtype=self.dtype)
        z = torch.zeros(self.B, self.zh.shape[1], n * self.hop, dtype=self.dtype)
        y = self.push(c, z)[..., :self.delay]
        self.reset()
        return y


def stream(w, z, c, cfg, schedule, **kw):
    """Run ``PWGLookaheadRef`` over c (B, aux, T') and z (B, 1, T' * hop) in chunks of ``schedule`` frames (repeated until
    the utterance is used up; the last chunk is cut short), then flush; returns cat(pushes, flush)."""
    hop = math.prod(cfg["upsample_scales"])
    ref = PWGLookaheadRef(w, cfg, batch=c.shape[0], **kw)
    return drive(lambda j, n: ref.push(c[:, :, j:j + n], z[:, :, j * hop:(j + n) * hop]), c.shape[-1], schedule, ref.flush)


def measured_lookahead(w, cfg, frames):
    """The true lookahead of the centred generator in output samples, measured by autograd on the mel frames at the last
    of ``frames`` frames (``ref_stream.measured_lookahead``)."""
    hop = math.prod(cfg["upsample_scales"])
    g = torch.Generator().manual_seed(3)
    c = torch.randn(1, cfg["aux_channels"], frames, generator=g, dtype=torch.float64, requires_grad=True)
    z = torch.randn(1, cfg.get("in_channels", 1), frames * hop, generator=g, dtype=torch.float64)
    wd = {k: v.double() for k, v in w.items()}
    return _measured(lambda c: whole_utterance(wd, z, c, cfg), c, frames - 1, hop)
