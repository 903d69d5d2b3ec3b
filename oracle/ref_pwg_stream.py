"""Chunked CPU restatement of streaming a causal Parallel WaveGAN (TEST INFRASTRUCTURE), on top of
``oracle/ref_causal_pwg.py``.  It carries the same state as ``parallelwavegan_b200.streaming.CausalPWGStream``,
explicitly and in plain tensors:

* conv_in: the last ``aux_context_window`` frames, a fresh item's replicated from its first frame
  (``ReplicationPad1d`` of ``inference``); conv_in runs as a valid conv on [history | chunk];
* each causal FIR stage: its last two input frames, which stand in for the stage's 2 * scale samples of left padding;
* each WaveNet layer: its last (K - 1) * dilation input samples, which stand in for the conv's left padding.

``whole_utterance`` is the reference it must equal: ``inference`` on the whole utterance.  The knobs ``wn_short``,
``cin_init`` and ``fir_frames`` inject the plausible mistakes (a layer history one row short, a zero-initialised conv_in
history, one FIR frame instead of two), so that the tests can show each of them is caught."""
import math

import torch
import torch.nn.functional as F

from .ref_causal_pwg import wavenet_residual_block
from .ref_stream import drive, keep


def _fir_prefix(cfg):
    return "upsample_net.upsample" if cfg.get("upsample_net", "ConvInUpsampleNetwork") == "ConvInUpsampleNetwork" else "upsample_net"


def whole_utterance(w, z, c, cfg):
    """``ParallelWaveGANGenerator.inference`` for a batch of whole utterances: c (B, aux, T') is edge-padded by
    ``aux_context_window`` frames (ReplicationPad1d) and the generator runs on it.  z: (B, 1, T' * hop)."""
    from .ref_causal_pwg import pwg_generator

    acw = cfg.get("aux_context_window", 0)
    if acw:
        idx = torch.arange(-acw, c.shape[-1] + acw).clamp(0, c.shape[-1] - 1)
        c = c[:, :, idx]
    return pwg_generator(w, z, c, cfg)


class PWGStreamRef:
    """push(c (B, aux, n), z (B, 1, n * hop)) -> (B, out_channels, n * hop), for any n >= 1."""

    def __init__(self, w, cfg, batch=1, dtype=torch.float64, wn_short=0, cin_init="replicate", fir_frames=2):
        kind = cfg.get("upsample_net", "ConvInUpsampleNetwork")
        assert cfg.get("use_causal_conv") and kind in ("ConvInUpsampleNetwork", "UpsampleNetwork"), cfg
        self.w = {k: v.to(dtype) for k, v in w.items()}
        self.cfg, self.B, self.dtype = cfg, batch, dtype
        self.wn_short, self.cin_init, self.fir_frames = wn_short, cin_init, fir_frames
        self.acw = cfg.get("aux_context_window", 0) if kind == "ConvInUpsampleNetwork" else 0
        self.conv_in = kind == "ConvInUpsampleNetwork"
        self.scales = list(cfg["upsample_scales"])
        A, R = cfg["aux_channels"], cfg["residual_channels"]
        lps = cfg["layers"] // cfg["stacks"]
        self.dil = [2 ** (l % lps) for l in range(cfg["layers"])]
        self.H = [(cfg["kernel_size"] - 1) * d for d in self.dil]
        self.cin_hist = None  # set from the first frame on the first push
        self.fir_hist = [torch.zeros(batch, A, 2, dtype=dtype) for _ in self.scales]
        self.wn_hist = [torch.zeros(batch, R, h, dtype=dtype) for h in self.H]

    def push(self, c, z):
        w, cfg = self.w, self.cfg
        c, z = c.to(self.dtype), z.to(self.dtype)
        n = c.shape[-1]
        if self.conv_in:
            if self.acw:
                if self.cin_hist is None:
                    first = c[:, :, :1].expand(-1, -1, self.acw)
                    self.cin_hist = first.clone() if self.cin_init == "replicate" else torch.zeros_like(first)
                x = torch.cat([self.cin_hist, c], -1)
                self.cin_hist = x[:, :, n:]
            else:
                x = c
            c = F.conv1d(x, w["upsample_net.conv_in.weight"])
        prefix = _fir_prefix(cfg)
        for i, s in enumerate(self.scales):
            hist = self.fir_hist[i]
            if self.fir_frames == 1:
                hist = F.pad(hist[:, :, 1:], (1, 0))
            x = torch.cat([hist, c], -1)  # frames -2, -1, 0 .. n-1
            self.fir_hist[i] = x[:, :, -2:]
            B, C, T = x.shape
            fir = w[f"{prefix}.up_layers.{2 * i + 1}.weight"].reshape(1, 1, -1)
            # the stretched history is exactly the 2 s samples of the whole-signal left padding
            c = F.conv1d(torch.repeat_interleave(x, s, dim=-1).reshape(B * C, 1, T * s), fir).reshape(B, C, n * s)
            n *= s
        x = F.conv1d(z, w["first_conv.weight"], w["first_conv.bias"])
        skips = 0
        for l, (d, h) in enumerate(zip(self.dil, self.H)):
            xp = torch.cat([self.wn_hist[l], x], -1)
            # wn_short: the oldest rows of the history lost
            self.wn_hist[l] = keep(xp, h, self.wn_short)
            # the causal layer on [history | chunk]; its outputs over the history rows are discarded
            cp = F.pad(c, (h, 0))
            xo, s = wavenet_residual_block(w, f"conv_layers.{l}", xp, cp, d, cfg["kernel_size"], causal=True)
            x, skips = xo[..., h:], skips + s[..., h:]
        x = F.relu(skips * math.sqrt(1.0 / cfg["layers"]))
        x = F.relu(F.conv1d(x, w["last_conv_layers.1.weight"], w["last_conv_layers.1.bias"]))
        return F.conv1d(x, w["last_conv_layers.3.weight"], w["last_conv_layers.3.bias"])


def stream(w, z, c, cfg, schedule, **kw):
    """Run ``PWGStreamRef`` over c (B, aux, T') and z (B, 1, T' * hop) in chunks of ``schedule`` frames (repeated until
    the utterance is used up; the last chunk is cut short) and return the concatenated output."""
    hop = math.prod(cfg["upsample_scales"])
    ref = PWGStreamRef(w, cfg, batch=c.shape[0], **kw)
    return drive(lambda j, n: ref.push(c[:, :, j:j + n], z[:, :, j * hop:(j + n) * hop]), c.shape[-1], schedule)
