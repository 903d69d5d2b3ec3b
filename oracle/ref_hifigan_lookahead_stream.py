"""Chunked CPU restatement of streaming a centred HiFi-GAN with a fixed lookahead (TEST INFRASTRUCTURE), on top of
``oracle/ref_ops.hifigan_generator``.  It carries the same state as
``parallelwavegan_b200.streaming.HiFiGANLookaheadStream``, explicitly and in plain tensors.

A centred conv (kernel k, dilation d, padding p = (k - 1) * d / 2) over [the (k - 1) * d samples in front of a chunk |
the chunk] computes the whole-signal conv's samples from p before the chunk's first sample on.  So every signal is
carried in "delayed time": a chunk of signal s holds its samples [F * rate_s - look_s, (F + n) * rate_s - look_s), F
being the frames pushed before, and look_s the lookahead summed along the layers in front of s:

* input conv: (K - 1) / 2 frames;
* conv-transpose (kernel 2 s, padding p): s * look + p; the window of [previous input sample | chunk] is exactly those
  samples;
* a ResBlock step x + branch(x): the branch lags x by q = sum of its convs' paddings, and adds x read q samples back;
* MRF: block j reads the level input delta_j = max_i D_i - D_j samples later (D_j: the block's total lag), so every
  block ends at the same lookahead and they sum as in the whole-utterance forward;
* output conv: (K - 1) / 2 samples; the total is ``delay``.

The whole-signal conv reads zero padding before sample 0 and after the signal's end, so every signal is stored as zero
outside [0, T_s) (the mask; the end is set by the flush).  ``flush`` pushes ceil(delay / hop) zero frames with the end
set and returns the first ``delay`` samples, so that cat(pushes, flush) == [zeros(delay) | whole_utterance].

The knobs inject plausible mistakes, so that the tests can show each one is caught: ``no_mask``, ``undelayed_res`` (the
residual read at the branch's own rows), ``unaligned`` (every delta_j zero) and ``flush_no_end`` (the flush pushes zero
frames but leaves the end open).  ``up_replicate`` (a fresh item's conv-transpose history replicates its signal's sample
0, as the causal model's ReplicationPad1d does; the first chunk must reach that sample of every level input) is not a
mistake the output can show.  A fresh item's first chunk of a level input starts at sample a = -look_h (look_h >= 3
from the input conv alone), so its history frame is sample a - 1, and with kernel 2 s and padding p that frame's taps
reach output samples up to (a + 1) * s - 1 - p, all before 0, which the mask zeroes.  (Sample -1 itself would reach up
to s - 1 - p >= 0: it is the lookahead that keeps the history out of the signal.)"""
import math

import torch
import torch.nn.functional as F

from .ref_ops import hifigan_generator
from .ref_stream import conv, drive, keep, rows
from .ref_stream import measured_lookahead as _measured


def whole_utterance(w, c, cfg):
    """``HiFiGANGenerator.inference`` (centred) for a batch of whole utterances c (B, in_channels, T)."""
    return hifigan_generator(w, c, cfg)


class HiFiGANLookaheadRef:
    """push(c (B, in_channels, n)) -> (B, out_channels, n * hop); flush() -> (B, out_channels, delay)."""

    def __init__(self, w, cfg, batch=1, dtype=torch.float64, no_mask=False, undelayed_res=False, unaligned=False,
                 up_replicate=False, flush_no_end=False):
        assert not cfg.get("use_causal_conv"), cfg
        self.w = {k: v.to(dtype) for k, v in w.items()}
        self.cfg, self.B, self.dtype = cfg, batch, dtype
        self.no_mask, self.undelayed_res, self.up_replicate, self.flush_no_end = no_mask, undelayed_res, up_replicate, flush_no_end
        self.slope = cfg.get("negative_slope", 0.1)
        self.ks, self.dils = list(cfg["resblock_kernel_sizes"]), [list(d) for d in cfg["resblock_dilations"]]
        self.scales = list(cfg["upsample_scales"])
        self.nb = len(self.ks)
        self.extra = cfg.get("use_additional_convs", True)
        self.K = cfg["kernel_size"]
        self.hop = math.prod(self.scales)
        ch = [cfg["channels"] // 2 ** i for i in range(len(self.scales) + 1)]
        self.ch = ch
        look = (self.K - 1) // 2
        self.look_in = look
        self.levels = []
        for i, s in enumerate(self.scales):
            look_u = look * s + s // 2 + s % 2
            q = [[(k - 1) * d // 2 + ((k - 1) // 2 if self.extra else 0) for d in ds] for k, ds in zip(self.ks, self.dils)]
            D = [sum(qq) for qq in q]
            delta = [0 if unaligned else max(D) - Dj for Dj in D]
            hl = max(delta[j] + (k - 1) * ds[0] for j, (k, ds) in enumerate(zip(self.ks, self.dils)))
            self.levels.append(dict(s=s, rate=math.prod(self.scales[:i + 1]), look_h=look, look_u=look_u, q=q, delta=delta, hl=hl))
            look = look_u + max(D)
        self.delay = look + (self.K - 1) // 2
        self.reset()

    def reset(self):
        z = lambda C, H: torch.zeros(self.B, C, H, dtype=self.dtype)  # noqa: E731
        ch = self.ch
        self.cin = z(self.cfg["in_channels"], self.K - 1)
        self.up = [z(ch[i], 1) for i in range(len(self.scales))]
        self.lvl = [z(ch[i + 1], lv["hl"]) for i, lv in enumerate(self.levels)]
        self.xh = [[[z(ch[i + 1], (k - 1) * d) for d in ds[1:]] for k, ds in zip(self.ks, self.dils)] for i in range(len(self.scales))]
        self.xth = [[[z(ch[i + 1], k - 1) for _ in ds] for k, ds in zip(self.ks, self.dils)] for i in range(len(self.scales))]
        self.out = z(ch[-1], self.K - 1)
        self.frame, self.end, self.fresh = 0, None, True

    def _mask(self, y, rate, look):
        if self.no_mask:
            return y
        pos = self.frame * rate - look + torch.arange(y.shape[-1])
        keep = pos >= 0
        if self.end is not None:
            keep &= pos < self.end * rate
        return torch.where(keep, y, torch.zeros((), dtype=y.dtype))

    def push(self, c):
        w, slope = self.w, self.slope
        c = c.to(self.dtype)
        n, K = c.shape[-1], self.K
        h = self._mask(conv(self.cin, c, w["input_conv.weight"], w.get("input_conv.bias"), 1, 1.0, K - 1, n), 1, self.look_in)
        self.cin = keep(torch.cat([self.cin, c], -1), K - 1)
        for i, lv in enumerate(self.levels):
            s, rate = lv["s"], lv["rate"]
            # up_replicate: the fresh history is the signal's sample 0 (ReplicationPad1d), held by a first chunk that
            # reaches it
            hist = h[:, :, lv["look_h"]:lv["look_h"] + 1] if self.fresh and self.up_replicate else self.up[i]
            xp = torch.cat([hist, h], -1)
            self.up[i] = xp[:, :, -1:]
            u = F.conv_transpose1d(F.leaky_relu(xp, slope), w[f"upsamples.{i}.1.weight"], w.get(f"upsamples.{i}.1.bias"), stride=s)
            u = self._mask(u[:, :, s:u.shape[-1] - s], rate, lv["look_u"])
            t = u.shape[-1]
            cs = 0.0
            for j, (k, ds) in enumerate(zip(self.ks, self.dils)):
                p = f"blocks.{i * self.nb + j}"
                x, cur = u, lv["look_u"] + lv["delta"][j]
                for idx, d in enumerate(ds):
                    hx, extra = (self.lvl[i], lv["delta"][j]) if idx == 0 else (self.xh[i][j][idx - 1], 0)
                    q = lv["q"][j][idx]
                    xt = conv(hx, x, w[f"{p}.convs1.{idx}.1.weight"], w.get(f"{p}.convs1.{idx}.1.bias"), d, slope, (k - 1) * d + extra, t)
                    xt = self._mask(xt, rate, cur + (k - 1) * d // 2)
                    if self.extra:
                        ht = self.xth[i][j][idx]
                        self.xth[i][j][idx] = keep(torch.cat([ht, xt], -1), k - 1)
                        xt = conv(ht, xt, w[f"{p}.convs2.{idx}.1.weight"], w.get(f"{p}.convs2.{idx}.1.bias"), 1, slope, k - 1, t)
                    res = x if self.undelayed_res else rows(hx, x, -(q + extra), t)
                    if idx > 0:
                        self.xh[i][j][idx - 1] = keep(torch.cat([hx, x], -1), hx.shape[-1])
                    cur += q
                    x = self._mask(xt + res, rate, cur)
                cs = cs + x
            self.lvl[i] = keep(torch.cat([self.lvl[i], u], -1), lv["hl"])
            h = cs / self.nb
        y = torch.tanh(conv(self.out, h, w["output_conv.1.weight"], w.get("output_conv.1.bias"), 1, 0.01, K - 1, h.shape[-1]))
        y = self._mask(y, self.hop, self.delay)
        self.out = keep(torch.cat([self.out, h], -1), K - 1)
        self.frame += n
        self.fresh = False
        return y

    def flush(self):
        if not self.flush_no_end:
            self.end = self.frame
        n = -(-self.delay // self.hop)
        y = self.push(torch.zeros(self.B, self.cfg["in_channels"], n, dtype=self.dtype))[..., :self.delay]
        self.reset()
        return y


def stream(w, c, cfg, schedule, **kw):
    """Run ``HiFiGANLookaheadRef`` over c (B, in_channels, T) in chunks of ``schedule`` frames (repeated until the
    utterance is used up; the last chunk is cut short), then flush; returns cat(pushes, flush)."""
    ref = HiFiGANLookaheadRef(w, cfg, batch=c.shape[0], **kw)
    return drive(lambda j, n: ref.push(c[:, :, j:j + n]), c.shape[-1], schedule, ref.flush)


def measured_lookahead(w, cfg, frames):
    """The true lookahead of the centred generator in output samples, measured by autograd at the last of ``frames``
    frames (``ref_stream.measured_lookahead``)."""
    g = torch.Generator().manual_seed(3)
    c = torch.randn(1, cfg["in_channels"], frames, generator=g, dtype=torch.float64, requires_grad=True)
    wd = {k: v.double() for k, v in w.items()}
    return _measured(lambda c: whole_utterance(wd, c, cfg), c, frames - 1, math.prod(cfg["upsample_scales"]))
