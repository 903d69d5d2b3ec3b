"""Chunked CPU restatement of streaming a centred (multi-band) MelGAN with a fixed lookahead (TEST INFRASTRUCTURE).  It
carries the same state as ``parallelwavegan_b200.streaming.MelGANLookaheadStream``, explicitly and in plain tensors.

Every signal runs in "delayed time", as in ``oracle/ref_hifigan_lookahead_stream.py``: a chunk of signal s holds its
samples [F * rate_s - look_s, (F + n) * rate_s - look_s), F being the frames pushed before.  The lookaheads:

* input conv (kernel K, padding (K - 1) / 2): (K - 1) / 2 frames, on [the last K - 1 frames | chunk];
* conv-transpose (kernel 2 s, padding p = s // 2 + s % 2): s * look + p, on [the previous input sample | chunk];
* ResidualStack (dilation d, kernel k, padding P = (k - 1) / 2 * d): h = conv1 on [the last (k - 1) d samples | chunk],
  P behind its input; the 1x1 skip reads the stack input P rows back; look + P;
* output conv: (K - 1) / 2 samples more; with PQMF, ``delay`` = N * look_sub + taps // 2.

Every signal is stored as zero outside [0, T_s) (the mask; the end is set by the flush), which is the zero padding of
the conv-transposes and the PQMF synthesis.  A reflect- or replicate-padded conv instead reads, for an input row whose
sample u lies outside [0, L), the row holding sample -u or 2 (L - 1) - u (reflect) or 0 or L - 1 (replicate) of the
same [history | chunk] window: the edge policy.  For every output inside the signal that row lies in the window, so no
push needs a minimum length; the flush pushes ceil(delay / (hop * N)) zero frames with the end set.

``whole_utterance`` is the reference the stream must equal after ``delay`` leading zeros.  The knobs inject plausible
mistakes, so that the tests can show each one is caught: ``zero_edges`` (zero instead of reflected edges),
``left_only`` (no mirror at the end), ``wrong_axis`` (mirror about -1/2: -u - 1 and 2 L - 1 - u), ``undelayed_skip`` (the
skip conv reads the stack input at its own rows), ``unmasked_pqmf`` (the synthesis output not masked) and
``flush_no_end`` (the flush leaves the end open)."""
import math

import torch
import torch.nn.functional as F

from .ref_ops import melgan_layer_index, pqmf_filters, pqmf_synthesis
from .ref_stream import drive, keep
from .ref_stream import measured_lookahead as _measured

MODES = {"reflect": "reflect", "replicate": "replicate", "zero": "constant"}


def whole_utterance(w, c, cfg, pad="reflect", subbands=None):
    """centred ``MelGANGenerator.inference`` with ``pad`` (and ``model.pqmf`` of ``subbands`` bands) for a batch of
    whole utterances c (B, in_channels, T)"""
    slope = cfg.get("negative_slope", 0.2)
    sk = cfg.get("stack_kernel_size", 3)
    K = cfg.get("kernel_size", 7)

    def conv(x, key, d, P):
        return F.conv1d(F.pad(x, (P, P), mode=MODES[pad]), w[key + ".weight"], w.get(key + ".bias"), dilation=d)

    for kind, idx, meta in melgan_layer_index(dict(cfg, use_causal_conv=False)):
        p = f"melgan.{idx}"
        if kind == "conv_in":
            c = conv(c, p, 1, (K - 1) // 2)
        elif kind == "convt":
            s = meta[1]
            c = F.conv_transpose1d(F.leaky_relu(c, slope), w[p + ".weight"], w.get(p + ".bias"), stride=s, padding=s // 2 + s % 2,
                                   output_padding=s % 2)
        elif kind == "stack":
            d = sk ** meta[1]
            h = conv(F.leaky_relu(c, slope), p + ".stack.2", d, (sk - 1) // 2 * d)
            h = F.conv1d(F.leaky_relu(h, slope), w[p + ".stack.4.weight"], w.get(p + ".stack.4.bias"))
            c = h + F.conv1d(c, w[p + ".skip_layer.weight"], w.get(p + ".skip_layer.bias"))
        else:
            c = conv(F.leaky_relu(c, slope), p, 1, (K - 1) // 2)
            if cfg.get("use_final_nonlinear_activation", True):
                c = torch.tanh(c)
    if subbands:
        c = pqmf_synthesis(c, pqmf_filters(subbands)[1].to(c.dtype))
    return c


def min_frames(cfg, pad="reflect"):
    """the shortest utterance ``inference`` accepts: ReflectionPad1d needs its padding below the signal's length"""
    if pad != "reflect":
        return 1
    K, sk = cfg.get("kernel_size", 7), cfg.get("stack_kernel_size", 3)
    need, rate = [((K - 1) // 2, 1)], 1
    for s in cfg["upsample_scales"]:
        rate *= s
        need += [((sk - 1) // 2 * sk ** j, rate) for j in range(cfg["stacks"])]
    need.append(((K - 1) // 2, rate))
    return max(P // r + 1 for P, r in need)


class MelGANLookaheadRef:
    """push(c (B, in_channels, n)) -> (B, 1, n * hop * subbands); flush() -> (B, 1, delay)."""

    def __init__(self, w, cfg, pad="reflect", subbands=None, batch=1, dtype=torch.float64, zero_edges=False, left_only=False,
                 wrong_axis=False, undelayed_skip=False, unmasked_pqmf=False, flush_no_end=False):
        assert not cfg.get("use_causal_conv"), cfg
        self.w = {k: v.to(dtype) for k, v in w.items()}
        self.cfg, self.pad, self.B, self.dtype = cfg, pad, batch, dtype
        self.zero_edges, self.left_only, self.wrong_axis = zero_edges, left_only, wrong_axis
        self.undelayed_skip, self.unmasked_pqmf, self.flush_no_end = undelayed_skip, unmasked_pqmf, flush_no_end
        self.slope = cfg.get("negative_slope", 0.2)
        self.sk = cfg.get("stack_kernel_size", 3)
        self.K = cfg.get("kernel_size", 7)
        self.plan = melgan_layer_index(dict(cfg, use_causal_conv=False))
        self.hop = math.prod(cfg["upsample_scales"])
        look = (self.K - 1) // 2
        self.look = {}  # layer index -> lookahead of its input signal
        for kind, idx, meta in self.plan:
            self.look[idx] = look
            if kind == "conv_in":
                look = (self.K - 1) // 2
            elif kind == "convt":
                s = meta[1]
                look = look * s + s // 2 + s % 2
            elif kind == "stack":
                look += (self.sk - 1) // 2 * self.sk ** meta[1]
            else:
                look += (self.K - 1) // 2
        self.look_sub = look
        self.N = subbands or 1
        if subbands:
            self.f_syn = pqmf_filters(subbands)[1].to(dtype)
            self.taps = self.f_syn.shape[-1] - 1
            self.delay = subbands * look + self.taps // 2
        else:
            self.delay = look
        self.reset()

    def reset(self):
        self.hist = {}  # layer index -> history (B, C, H)
        self.pq = torch.zeros(self.B, self.N, self.taps // self.N if self.N > 1 else 0, dtype=self.dtype)
        self.frame, self.end = 0, None

    def _mask(self, y, rate, look):
        pos = self.frame * rate - look + torch.arange(y.shape[-1])
        keep = pos >= 0
        if self.end is not None:
            keep &= pos < self.end * rate
        return torch.where(keep, y, torch.zeros((), dtype=y.dtype))

    def _edge(self, xp, rate, in_look):
        """[history | chunk] xp (B, C, R) with the edge policy: rows whose sample lies outside the signal read the row of
        their reflected or replicated sample (zero when it is outside xp)"""
        if self.pad == "zero" or self.zero_edges:
            return xp
        R = xp.shape[-1]
        u = self.frame * rate - in_look + torch.arange(R)
        L = self.end * rate if self.end is not None else None
        v = u.clone()
        if self.pad == "reflect":
            v = torch.where(u < 0, -u - 1 if self.wrong_axis else -u, v)
            if L is not None and not self.left_only:
                v = torch.where(u >= L, 2 * L - 1 - u if self.wrong_axis else 2 * (L - 1) - u, v)
        else:
            v = torch.where(u < 0, torch.zeros_like(u), v)
            if L is not None and not self.left_only:
                v = torch.where(u >= L, torch.full_like(u, L - 1), v)
        r = torch.arange(R) + (v - u)
        inside = (r >= 0) & (r < R)
        out = xp[..., r.clamp(0, R - 1)]
        return torch.where(inside, out, torch.zeros((), dtype=xp.dtype))

    def _conv(self, key, x, wk, d, slope, rate, in_look_x):
        """the centred conv of chunk x (lookahead in_look_x) over [its (k - 1) d history | x], with the edge policy"""
        wt, b = self.w[wk + ".weight"], self.w.get(wk + ".bias")
        H = (wt.shape[-1] - 1) * d
        hist = self.hist.get(key, x.new_zeros(x.shape[0], x.shape[1], H))
        xp = torch.cat([hist, x], -1)
        self.hist[key] = keep(xp, H)
        xe = self._edge(xp, rate, in_look_x + H)
        return F.conv1d(F.leaky_relu(xe, slope), wt, b, dilation=d), hist

    def _synth(self, y):
        """the synthesis window of subband chunk y (B, N, m): m * N samples from N * (first row) - taps // 2 on"""
        N, H = self.N, self.pq.shape[-1]
        full = torch.cat([self.pq, y], -1)
        self.pq = keep(full, H)
        z = torch.zeros(full.shape[0], N, full.shape[-1] * N, dtype=full.dtype)
        z[..., ::N] = full * N
        lead = self.taps - H * N
        z = F.pad(z, (lead, 0)) if lead >= 0 else z[..., -lead:]
        return F.conv1d(z, self.f_syn)

    def push(self, c):
        w, slope, sk = self.w, self.slope, self.sk
        c = c.to(self.dtype)
        n = c.shape[-1]
        rate = 1
        for kind, idx, meta in self.plan:
            p, look = f"melgan.{idx}", self.look[idx]
            if kind == "conv_in":
                c, _ = self._conv(idx, c, p, 1, 1.0, 1, 0)
                c = self._mask(c, 1, (self.K - 1) // 2)
            elif kind == "convt":
                s = meta[1]
                rate *= s
                x = F.leaky_relu(c, slope)
                xp = torch.cat([self.hist.get(idx, x.new_zeros(x.shape[0], x.shape[1], 1)), x], -1)
                self.hist[idx] = xp[:, :, -1:]
                u = F.conv_transpose1d(xp, w[p + ".weight"], w.get(p + ".bias"), stride=s)
                c = self._mask(u[:, :, s:u.shape[-1] - s], rate, look * s + s // 2 + s % 2)
            elif kind == "stack":
                d = sk ** meta[1]
                P = (sk - 1) // 2 * d
                h, hist = self._conv(idx, c, p + ".stack.2", d, slope, rate, look)
                h = F.conv1d(F.leaky_relu(h, slope), w[p + ".stack.4.weight"], w.get(p + ".stack.4.bias"))
                xs = c if self.undelayed_skip else torch.cat([hist, c], -1)[..., hist.shape[-1] - P:hist.shape[-1] - P + c.shape[-1]]
                c = self._mask(h + F.conv1d(xs, w[p + ".skip_layer.weight"], w.get(p + ".skip_layer.bias")), rate, look + P)
            else:
                c, _ = self._conv(idx, c, p, 1, slope, rate, look)
                if self.cfg.get("use_final_nonlinear_activation", True):
                    c = torch.tanh(c)
                c = self._mask(c, rate, self.look_sub)
        if self.N > 1:
            c = self._synth(c)
            if not self.unmasked_pqmf:
                c = self._mask(c, self.hop * self.N, self.delay)
        self.frame += n
        return c

    def flush(self):
        if not self.flush_no_end:
            self.end = self.frame
        n = -(-self.delay // (self.hop * self.N))
        y = self.push(torch.zeros(self.B, self.cfg["in_channels"], n, dtype=self.dtype))[..., :self.delay]
        self.reset()
        return y


def stream(w, c, cfg, schedule, pad="reflect", subbands=None, **kw):
    """Run ``MelGANLookaheadRef`` over c (B, in_channels, T) in chunks of ``schedule`` frames (repeated until the
    utterance is used up; the last chunk is cut short), then flush; returns cat(pushes, flush)."""
    ref = MelGANLookaheadRef(w, cfg, pad=pad, subbands=subbands, batch=c.shape[0], **kw)
    return drive(lambda j, n: ref.push(c[:, :, j:j + n]), c.shape[-1], schedule, ref.flush)


def measured_lookahead(w, cfg, frames, pad="reflect", subbands=None):
    """The true lookahead of the centred generator in output samples, measured by autograd at the last of ``frames``
    frames (``ref_stream.measured_lookahead``)."""
    hop = math.prod(cfg["upsample_scales"]) * (subbands or 1)
    g = torch.Generator().manual_seed(3)
    c = torch.randn(1, cfg["in_channels"], frames, generator=g, dtype=torch.float64, requires_grad=True)
    wd = {k: v.double() for k, v in w.items()}
    return _measured(lambda c: whole_utterance(wd, c, cfg, pad, subbands), c, frames - 1, hop)
