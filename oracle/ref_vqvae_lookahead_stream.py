"""Chunked CPU restatement of streaming a VQ-VAE's wav2wav conversion with a fixed lookahead (TEST INFRASTRUCTURE).  It
carries the same state as ``parallelwavegan_b200.streaming.VQVAELookaheadStream``, explicitly and in plain tensors.

Two chains run in delayed time, as in ``oracle/ref_melgan_lookahead_stream.py``: a chunk of signal s holds its samples
[F * rate_s - look_s, (F + n) * rate_s - look_s), F being the frames pushed before, and every signal is zero outside
[0, T_s) (the mask; the flush sets the end).

* encoder (MelGANDiscriminator): the reflect-padded input conv (kernel K0) on [the last K0 - 1 samples | chunk] with the
  edge policy, lookahead (K0 - 1) / 2; each strided conv (kernel K, stride s, padding p, groups) at output lookahead
  L' = ceil((L + K - p - s) / s), as a valid strided conv over the window [the last L' s + p - L input samples | chunk],
  which starts on a stride boundary of the whole signal's padded input; then the two centred stride-1 convs, each
  (K - 1) / 2 more.  The encoder's lookahead is E frames;
* bottleneck: the nearest code of each z_e frame, the local conditioning (after local_embed) from a delay line of E
  frames, and the global embedding;
* decoder: ``MelGANLookaheadRef`` on those frames with its frame counter E frames behind.

``delay`` = E * hop + the decoder's delay.  ``whole_utterance`` is decode(encode(x)).  The knobs inject plausible
mistakes, so that the tests can show each one is caught: ``window_shift`` (a strided window one stride late),
``zero_right_edge`` (zero instead of reflect at the right edge of the input conv), ``short_l_delay`` (the l delay line
one frame short), ``decoder_no_lag`` (the decoder's counter not lagging by E) and ``short_lookahead`` (E one frame
too small)."""
import math

import torch
import torch.nn.functional as F

from .ref_melgan_lookahead_stream import MelGANLookaheadRef
from .ref_stream import drive, keep
from .ref_stream import measured_lookahead as _measured
from .ref_vqvae import _sub, assemble, decoder, encoder, quantize


def _enc_conf(cfg):
    ec = cfg.get("encoder_conf", {})
    return (list(ec.get("downsample_scales", [4, 4, 4, 4])), list(ec.get("kernel_sizes", [5, 3])), ec.get("channels", 16),
            ec.get("max_downsample_channels", 1024))


def _dec_conf(cfg):
    return dict(kernel_size=7, stack_kernel_size=3, negative_slope=0.2, **cfg.get("decoder_conf", {}))


def whole_utterance(w, x, cfg, l=None, g=None):
    """decode(encode(x), l, g) for a batch of whole signals x (B, 1, T)"""
    return decoder(w, assemble(w, F.embedding(quantize(encoder(w, x, cfg), w["codebook.embedding.weight"]),
                                              w["codebook.embedding.weight"]).transpose(1, 2), l, g), cfg)


class VQVAELookaheadRef:
    """push(x (B, 1, n * hop), l, g) -> (B, 1, n * hop); flush() -> (B, 1, delay)."""

    def __init__(self, w, cfg, batch=1, dtype=torch.float64, window_shift=False, zero_right_edge=False, short_l_delay=False,
                 decoder_no_lag=False, short_lookahead=False):
        self.w = {k: v.to(dtype) for k, v in w.items()}
        self.cfg, self.B, self.dtype = cfg, batch, dtype
        self.window_shift, self.zero_right_edge, self.short_l_delay = window_shift, zero_right_edge, short_l_delay
        scales, ks, ch, maxc = _enc_conf(cfg)
        self.hop = math.prod(scales)
        self.slope = 0.2
        self.K0 = ks[0] * ks[1]
        look = self.look0 = (self.K0 - 1) // 2
        self.strided, cin, rate = [], ch, self.hop
        for s in scales:
            K, p = 10 * s + 1, 5 * s
            Lq = -(-(look + K - p - s) // s)
            rate //= s
            self.strided.append(dict(s=s, K=K, p=p, groups=cin // 4, look=Lq, rate=rate, H=Lq * s + p - look))
            cin, look = min(cin * s, maxc), Lq
        self.tail = []
        for k in ks:
            look += (k - 1) // 2
            self.tail.append(dict(k=k, look=look))
        self.E = look - (1 if short_lookahead else 0)
        self.dec_cfg = _dec_conf(cfg)
        self.dec = MelGANLookaheadRef(_sub(self.w, "decoder"), self.dec_cfg, batch=batch, dtype=dtype)
        self.lag = 0 if decoder_no_lag else self.E
        self.delay = self.E * self.hop + self.dec.delay
        self.reset()

    def reset(self):
        self.hist, self.frame, self.end = {}, 0, None
        self.z = []  # z_e of every push, masked (delayed by E frames)
        self.dec.reset()
        self.dec.frame = -self.lag

    def _mask(self, y, rate, look):
        pos = self.frame * rate - look + torch.arange(y.shape[-1])
        keep = pos >= 0
        if self.end is not None:
            keep &= pos < self.end * rate
        return torch.where(keep, y, torch.zeros((), dtype=y.dtype))

    def _window(self, key, x, H):
        hist = self.hist.get(key, x.new_zeros(x.shape[0], x.shape[1], H))
        xp = torch.cat([hist, x], -1)
        self.hist[key] = keep(xp, H)
        return xp

    def _conv0(self, x):
        """the input conv on [K0 - 1 history samples | chunk], reflecting about both ends of the signal"""
        H = self.K0 - 1
        xp = self._window("e0", x, H)
        R = xp.shape[-1]
        u = self.frame * self.hop - H + torch.arange(R)
        v = torch.where(u < 0, -u, u)
        if self.end is not None and not self.zero_right_edge:
            L = self.end * self.hop
            v = torch.where(u >= L, 2 * (L - 1) - u, v)
        r = torch.arange(R) + (v - u)
        xe = torch.where((r >= 0) & (r < R), xp[..., r.clamp(0, R - 1)], torch.zeros((), dtype=xp.dtype))
        if self.zero_right_edge and self.end is not None:
            xe = torch.where(u < self.end * self.hop, xe, torch.zeros((), dtype=xp.dtype))
        y = F.conv1d(xe, self.w["encoder.layers.0.1.weight"], self.w.get("encoder.layers.0.1.bias"))
        return self._mask(F.leaky_relu(y, self.slope), self.hop, self.look0)

    def _encode(self, x):
        h = self._conv0(x)
        for i, lv in enumerate(self.strided):
            xp = self._window(f"s{i}", h, lv["H"])
            if self.window_shift:
                xp = F.pad(xp, (0, lv["s"]))[..., lv["s"]:]
            p = f"encoder.layers.{i + 1}.0"
            y = F.conv1d(xp, self.w[p + ".weight"], self.w.get(p + ".bias"), stride=lv["s"], groups=lv["groups"])
            h = self._mask(F.leaky_relu(y[..., :h.shape[-1] // lv["s"]], self.slope), lv["rate"], lv["look"])
        n = len(self.strided)
        for j, t in enumerate(self.tail):
            p = f"encoder.layers.{n + 1}.0" if j == 0 else f"encoder.layers.{n + 2}"
            y = F.conv1d(self._window(f"t{j}", h, t["k"] - 1), self.w[p + ".weight"], self.w.get(p + ".bias"))
            h = self._mask(F.leaky_relu(y, self.slope) if j == 0 else y, 1, t["look"])
        return h

    def push(self, x, l=None, g=None):
        x = x.to(self.dtype)
        n = x.shape[-1] // self.hop
        z = self._encode(x)
        self.z.append(z)
        cb = self.w["codebook.embedding.weight"]
        codes = F.embedding(quantize(z, cb), cb).transpose(1, 2)
        if l is not None:
            if "local_embed.weight" in self.w:
                l = F.conv1d(l.to(self.dtype), self.w["local_embed.weight"], self.w["local_embed.bias"])
            E = self.E - (1 if self.short_l_delay else 0)
            l = self._window("l", l.to(self.dtype), E)[..., :n]
        dec = assemble({k: v for k, v in self.w.items() if k != "local_embed.weight"}, codes, l, g)
        dec = self._mask(dec, 1, self.E)
        self.dec.end = self.end
        y = self.dec.push(dec)
        self.frame += n
        return y

    def flush(self, l_channels=0, g=None):
        self.end = self.frame
        n = -(-self.delay // self.hop)
        l = torch.zeros(self.B, l_channels, n, dtype=self.dtype) if l_channels else None
        y = self.push(torch.zeros(self.B, 1, n * self.hop, dtype=self.dtype), l, g)[..., :self.delay]
        self.z_e = torch.cat(self.z, -1)[..., self.E:self.E + self.end]
        self.reset()
        return y


def stream(w, x, cfg, schedule, l=None, g=None, **kw):
    """Run ``VQVAELookaheadRef`` over x (B, 1, T * hop) in chunks of ``schedule`` frames (repeated until the signal is
    used up; the last chunk is cut short), then flush; returns cat(pushes, flush)."""
    ref = VQVAELookaheadRef(w, cfg, batch=x.shape[0], **kw)
    hop = ref.hop

    def push(j, n):
        return ref.push(x[..., j * hop:(j + n) * hop], l[..., j:j + n] if l is not None else None, g)

    return drive(push, x.shape[-1] // hop, schedule, lambda: ref.flush(l.shape[1] if l is not None else 0, g)), ref


def measured_lookahead(w, cfg, frames, l=None, g=None):
    """The true lookahead of decode(encode(x)) in output samples, measured by float64 autograd through the encoder and
    the decoder (the codes held at their straight-through values): f * hop - o for the first output sample o that depends
    on any input sample of frame f (a frame well inside the signal; every frame has the same phase), found by a binary
    search.  A push that ends before frame f may only return outputs below f * hop - delay, and output o depends on
    frame f, so no exact stream has a smaller delay."""
    from .ref_vqvae import _StraightThrough, gather

    wd = {k: v.double() for k, v in w.items()}
    hop = math.prod(_enc_conf(cfg)[0])
    gen = torch.Generator().manual_seed(5)
    x = torch.randn(1, 1, frames * hop, generator=gen, dtype=torch.float64, requires_grad=True)
    cb = wd["codebook.embedding.weight"]

    def whole(x):
        z = encoder(wd, x, cfg)
        zq = _StraightThrough.apply(z, gather(cb, quantize(z, cb)))
        return decoder(wd, assemble(wd, zq, l, g), cfg)

    # the outputs read the frame's samples well before the signal's end, and output 0 does not
    return _measured(whole, x, frames - 10, hop, rate=hop)
