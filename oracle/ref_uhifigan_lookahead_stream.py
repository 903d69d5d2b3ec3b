"""Chunked CPU restatement of streaming a centred U-Net HiFi-GAN (``UHiFiGANGenerator``) with a fixed lookahead (TEST
INFRASTRUCTURE), on top of ``oracle/ref_uhifigan.uhifigan_generator``.  It carries the same state as
``parallelwavegan_b200.streaming.UHiFiGANLookaheadStream``, explicitly and in plain tensors.

Every signal runs in "delayed time", as in ``oracle/ref_hifigan_lookahead_stream.py``: a chunk of a signal with ``rate``
samples per frame and lookahead ``look`` holds its samples [F * rate - look, (F + n) * rate - look), F being the frames
pushed before, and every signal is stored as zero outside [0, T * rate) (the mask; the flush sets the end).  The U-Net
adds three things to the HiFi-GAN plan:

* the encoder runs on the excitation, pushed with its frames (``hop`` samples each): the input conv (lookahead
  (K - 1) / 2), then per level the MRF (the HiFi-GAN level plan, from any level input) and the strided conv (kernel 2 s,
  stride s, padding p = s // 2 + s % 2).  Its output lookahead is the smallest L' for which the push's last output row
  reads only input rows that have arrived, L' = ceil((L + s - p) / s) for input lookahead L; it reads
  [the last H = L' s + p - L input rows | chunk] from row 0, which is s-aligned in the whole signal's padded input
  (whole-signal row (F R' - L') s - p), so the stream's space-to-depth rows are the whole signal's;
* the bottom: hidden_conv on mel frames runs at the deepest skip's lookahead L_N (when that is the larger), on a
  history of L_N + (K - 1) / 2 frames with n outputs; otherwise the skip is delayed;
* each decoder level reads cat(h, skip) through a conv-transpose whose two sources have different lookaheads: the one
  ahead is read back by the difference d from a delay line of d + 1 rows (the conv-transpose's own history row
  included).

``delay`` is the output conv's lookahead.  It is at least the true lookahead of every output phase (the excess comes
from the ceilings at the strided convs); ``measured_lookahead`` measures that by autograd.

The knobs inject plausible mistakes, so that the tests can show each one is caught: ``skip_undelayed`` (every skip read
without its delay), ``mel_undelayed`` (hidden_conv at its own lookahead, labelled as the skip's), ``stride_phase`` (the
strided conv's window one input row late), ``ds_no_end_mask`` (strided conv outputs not masked past the end) and
``s2d_no_hist`` (the strided conv reads zeros in place of its history)."""
import math

import torch
import torch.nn.functional as F

from .ref_stream import conv, drive, keep, rows
from .ref_uhifigan import uhifigan_generator


def whole_utterance(w, e, c, cfg):
    """``UHiFiGANGenerator.inference`` for a batch of whole utterances: excitation e (B, 1, T * hop), c (B, in_channels,
    T) -> (B, out_channels, T * hop)."""
    return uhifigan_generator(w, e, c, cfg)


def _slope(cfg):
    return cfg.get("nonlinear_activation_params", {"negative_slope": 0.1}).get("negative_slope", 0.1)


class _MRF:
    """One level's MRF in delayed time (the HiFi-GAN level plan), from a level input of lookahead ``look_u``."""

    def __init__(self, cfg, channels, rate, look_u, prefix, first):
        self.ks, self.dils = list(cfg["resblock_kernel_sizes"]), [list(d) for d in cfg["resblock_dilations"]]
        self.nb, self.extra = len(self.ks), cfg.get("use_additional_convs", True)
        self.C, self.rate, self.look_u, self.prefix, self.first = channels, rate, look_u, prefix, first
        self.q = [[(k - 1) * d // 2 + ((k - 1) // 2 if self.extra else 0) for d in ds] for k, ds in zip(self.ks, self.dils)]
        D = [sum(qq) for qq in self.q]
        self.lag = max(D)
        self.delta = [self.lag - Dj for Dj in D]
        self.hl = max(self.delta[j] + (k - 1) * ds[0] for j, (k, ds) in enumerate(zip(self.ks, self.dils)))
        self.look_out = look_u + self.lag

    def reset(self, z):
        C = self.C
        self.lvl = z(C, self.hl)
        self.xh = [[z(C, (k - 1) * d) for d in ds[1:]] for k, ds in zip(self.ks, self.dils)]
        self.xth = [[z(C, k - 1) for _ in ds] for k, ds in zip(self.ks, self.dils)]

    def push(self, ref, u):
        w, slope, rate = ref.w, ref.slope, self.rate
        t = u.shape[-1]
        cs = 0.0
        for j, (k, ds) in enumerate(zip(self.ks, self.dils)):
            p = f"{self.prefix}.{self.first + j}"
            x, cur = u, self.look_u + self.delta[j]
            for idx, d in enumerate(ds):
                hx, extra = (self.lvl, self.delta[j]) if idx == 0 else (self.xh[j][idx - 1], 0)
                q = self.q[j][idx]
                xt = conv(hx, x, w[f"{p}.convs1.{idx}.1.weight"], w.get(f"{p}.convs1.{idx}.1.bias"), d, slope, (k - 1) * d + extra, t)
                xt = ref._mask(xt, rate, cur + (k - 1) * d // 2)
                if self.extra:
                    ht = self.xth[j][idx]
                    self.xth[j][idx] = keep(torch.cat([ht, xt], -1), k - 1)
                    xt = conv(ht, xt, w[f"{p}.convs2.{idx}.1.weight"], w.get(f"{p}.convs2.{idx}.1.bias"), 1, slope, k - 1, t)
                res = rows(hx, x, -(q + extra), t)
                if idx > 0:
                    self.xh[j][idx - 1] = keep(torch.cat([hx, x], -1), hx.shape[-1])
                cur += q
                x = ref._mask(xt + res, rate, cur)
            cs = cs + x
        self.lvl = keep(torch.cat([self.lvl, u], -1), self.hl)
        return cs / self.nb


class UHiFiGANLookaheadRef:
    """push(c (B, in_channels, n), e (B, 1, n * hop)) -> (B, out_channels, n * hop); flush() -> (B, out_channels, delay)."""

    def __init__(self, w, cfg, batch=1, dtype=torch.float64, skip_undelayed=False, mel_undelayed=False, stride_phase=False,
                 ds_no_end_mask=False, s2d_no_hist=False):
        self.w = {k: v.to(dtype) for k, v in w.items()}
        self.cfg, self.B, self.dtype = cfg, batch, dtype
        self.skip_undelayed, self.mel_undelayed, self.stride_phase = skip_undelayed, mel_undelayed, stride_phase
        self.ds_no_end_mask, self.s2d_no_hist = ds_no_end_mask, s2d_no_hist
        self.slope = _slope(cfg)
        self.K = cfg.get("kernel_size", 7)
        self.ds_scales, self.us_scales = list(cfg["downsample_scales"]), list(cfg["upsample_scales"])
        self.hop = math.prod(self.us_scales)
        assert math.prod(self.ds_scales) == self.hop, cfg
        nb = len(cfg["resblock_kernel_sizes"])
        C = cfg["channels"]
        pk = (self.K - 1) // 2
        # encoder: per level the MRF, then the strided conv
        look, rate = pk, self.hop
        self.look_in = look
        self.enc = []
        for i, s in enumerate(self.ds_scales):
            mrf = _MRF(cfg, C, rate, look, "downsamples_mrf", i * nb)
            p = s // 2 + s % 2
            L = mrf.look_out
            Lq = -(-(L + s - p) // s)
            rate //= s
            self.enc.append(dict(mrf=mrf, s=s, p=p, C=C, look_in=L, look=Lq, H=Lq * s + p - L, rate=rate))
            look, C = Lq, 2 * C
        # bottom: the deeper of the mel path and the last skip sets the decoder's first lookahead
        L_N = look
        self.look_dec0 = max(L_N, pk)
        self.cin_len = self.look_dec0 + pk
        self.dec = []
        look_h, rate = self.look_dec0, 1
        for i, s in enumerate(self.us_scales):
            e = self.enc[-1 - i]
            assert e["rate"] == rate, (e["rate"], rate)
            D = max(look_h, e["look"])
            p = s // 2 + s % 2
            rate *= s
            look_u = D * s + p
            mrf = _MRF(cfg, C // 2, rate, look_u, "upsamples_mrf", i * nb)
            self.dec.append(dict(s=s, C1=C, d1=D - look_h, d2=D - e["look"], look_u=look_u, mrf=mrf, rate=rate))
            look_h, C = mrf.look_out, C // 2
        self.look_last = look_h
        self.delay = look_h + pk
        self.reset()

    def reset(self):
        z = lambda C, H: torch.zeros(self.B, C, H, dtype=self.dtype)  # noqa: E731
        cfg = self.cfg
        self.ein = z(1, self.K - 1)
        for e in self.enc:
            e["mrf"].reset(z)
            e["hist"] = z(e["C"], e["H"])
        self.cin = z(cfg["in_channels"], self.cin_len)
        C = cfg["channels"] * 2 ** len(self.ds_scales)
        for i, d in enumerate(self.dec):
            d["mrf"].reset(z)
            d["h1"] = z(C, d["d1"] + 1)
            d["h2"] = z(C, d["d2"] + 1)
            C //= 2
        self.out = z(cfg["channels"], self.K - 1)
        self.frame, self.end = 0, None

    def _mask(self, y, rate, look, end=True):
        pos = self.frame * rate - look + torch.arange(y.shape[-1])
        keep = pos >= 0
        if self.end is not None and end:
            keep &= pos < self.end * rate
        return torch.where(keep, y, torch.zeros((), dtype=y.dtype))

    def push(self, c, e):
        w, slope, K = self.w, self.slope, self.K
        c, e = c.to(self.dtype), e.to(self.dtype)
        n = c.shape[-1]
        assert e.shape[-1] == n * self.hop, (e.shape, n)
        # encoder
        h = conv(self.ein, e, w["input_conv.0.weight"], w.get("input_conv.0.bias"), 1, 1.0, K - 1, n * self.hop)
        h = self._mask(F.leaky_relu(h, slope), self.hop, self.look_in)
        self.ein = keep(torch.cat([self.ein, e], -1), K - 1)
        skips = []
        for i, lv in enumerate(self.enc):
            h = lv["mrf"].push(self, h)
            s, H = lv["s"], lv["H"]
            hist = torch.zeros_like(lv["hist"]) if self.s2d_no_hist else lv["hist"]
            xw = torch.cat([hist, h], -1)
            lv["hist"] = keep(xw, H)
            t = n * lv["rate"]
            first = 1 if self.stride_phase else 0
            xw = xw[..., first:first + (t - 1) * s + 2 * s]
            xw = F.pad(xw, (0, (t - 1) * s + 2 * s - xw.shape[-1]))
            y = F.leaky_relu(F.conv1d(xw, w[f"downsamples.{i}.0.weight"], w.get(f"downsamples.{i}.0.bias"), stride=s), slope)
            h = self._mask(y, lv["rate"], lv["look"], end=not self.ds_no_end_mask)
            skips.append(h)
        # bottom: hidden_conv at the decoder's first lookahead
        pad_left = K - 1 if self.mel_undelayed else self.cin_len
        h = conv(self.cin, c, w["hidden_conv.weight"], w.get("hidden_conv.bias"), 1, 1.0, pad_left, n)
        h = self._mask(h, 1, self.look_dec0)
        self.cin = keep(torch.cat([self.cin, c], -1), self.cin_len)
        # decoder
        for i, lv in enumerate(self.dec):
            skip = skips[-1 - i]
            s, t = lv["s"], h.shape[-1]
            d2 = 0 if self.skip_undelayed else lv["d2"]
            x1 = rows(lv["h1"], h, -(lv["d1"] + 1), t + 1)
            x2 = rows(lv["h2"], skip, -(d2 + 1), t + 1)
            lv["h1"] = keep(torch.cat([lv["h1"], h], -1), lv["d1"] + 1)
            lv["h2"] = keep(torch.cat([lv["h2"], skip], -1), lv["d2"] + 1)
            xp = torch.cat([x1, x2], 1)
            u = F.conv_transpose1d(F.leaky_relu(xp, slope), w[f"upsamples.{i}.1.weight"], w.get(f"upsamples.{i}.1.bias"), stride=s)
            u = self._mask(u[:, :, s:u.shape[-1] - s], lv["rate"], lv["look_u"])
            h = lv["mrf"].push(self, u)
        y = torch.tanh(conv(self.out, h, w["output_conv.1.weight"], w.get("output_conv.1.bias"), 1, 0.01, K - 1, h.shape[-1]))
        y = self._mask(y, self.hop, self.delay)
        self.out = keep(torch.cat([self.out, h], -1), K - 1)
        self.frame += n
        return y

    def flush(self):
        self.end = self.frame
        n = -(-self.delay // self.hop)
        y = self.push(torch.zeros(self.B, self.cfg["in_channels"], n, dtype=self.dtype),
                      torch.zeros(self.B, 1, n * self.hop, dtype=self.dtype))[..., :self.delay]
        self.reset()
        return y


def stream(w, e, c, cfg, schedule, **kw):
    """Run ``UHiFiGANLookaheadRef`` over c (B, in_channels, T) and e (B, 1, T * hop) in chunks of ``schedule`` frames
    (repeated until the utterance is used up; the last chunk is cut short), then flush; returns cat(pushes, flush)."""
    ref = UHiFiGANLookaheadRef(w, cfg, batch=c.shape[0], **kw)
    hop = ref.hop
    return drive(lambda j, n: ref.push(c[:, :, j:j + n], e[:, :, j * hop:(j + n) * hop]), c.shape[-1], schedule, ref.flush)


def measured_lookahead(w, cfg, frames, first=2):
    """The true lookahead of every output phase, measured by autograd on the float64 generator: for each output o of
    frame ``first`` (o = first * hop + phase), the last excitation sample k_e(o) and the last mel frame f_c(o) that o
    depends on.  Returns, per phase, (k_e(o) - o, f(o) * hop - o) with f(o) = max(k_e(o) // hop, f_c(o)) the last frame
    o needs: a stream of delay D can emit o when D >= f(o) * hop - o.  Both last inputs are non-decreasing in o, so the
    phases are bisected: an interval whose two ends depend on the same last inputs is constant in between, and only
    about as many gradients as there are steps are taken.  ``frames`` must reach past the dependencies of frame
    ``first`` so the end of the utterance cuts none of them."""
    hop = math.prod(cfg["upsample_scales"])
    g = torch.Generator().manual_seed(3)
    wd = {k: v.double() for k, v in w.items()}
    c = torch.randn(1, cfg["in_channels"], frames, generator=g, dtype=torch.float64, requires_grad=True)
    e = torch.randn(1, 1, frames * hop, generator=g, dtype=torch.float64, requires_grad=True)
    y = whole_utterance(wd, e, c, cfg)
    last = {}

    def deps(o):
        if o not in last:
            ge, gc = torch.autograd.grad(y[0, 0, o], (e, c), retain_graph=True)
            ke = int(torch.nonzero(ge[0, 0]).max())
            fc = int(torch.nonzero(gc[0].abs().sum(0)).max())
            assert ke < frames * hop - hop and fc < frames - 1, "frames too short for the dependencies"
            last[o] = (ke, fc)
        return last[o]

    def fill(a, b):  # deps of every o in [a, b], given monotone last inputs
        if deps(a) == deps(b):
            for o in range(a + 1, b):
                last[o] = last[a]
            return
        if b - a <= 1:
            return
        m = (a + b) // 2
        fill(a, m)
        fill(m, b)

    o0 = first * hop
    fill(o0, o0 + hop - 1)
    out = []
    for o in range(o0, o0 + hop):
        ke, fc = last[o]
        out.append((ke - o, max(ke // hop, fc) * hop - o))
    return out
