"""Chunked CPU restatement of streaming a causal (multi-band) MelGAN (TEST INFRASTRUCTURE), on top of the pieces of
``oracle/ref_ops``.  It carries the same state as ``parallelwavegan_b200.streaming.CausalMelGANStream``, explicitly and
in plain tensors, one history per signal:

* the input conv: its last kernel_size - 1 mel frames;
* each conv-transpose: the last frame of its input; a fresh item replicates its first frame (``ReplicationPad1d``);
* each ResidualStack: the last (k - 1) * d samples of its input;
* the output conv: its last kernel_size - 1 input samples;
* with PQMF: the last floor(taps / subbands) subband samples, the synthesis filter's reach into the past.

A fresh item's pad comes from the chunk itself: samples P .. 1 (reflect), sample 0 repeated (replicate) or zeros.  Every
causal conv runs as a valid conv on [pad or history | chunk].  The synthesis lags by taps // 2 samples: a push emits
the whole-utterance samples [T0 * N - taps // 2, (T0 + n) * N - taps // 2) (zeros before sample 0), and ``flush``
emits the last taps // 2 against the zero right padding.  ``whole_utterance`` is the reference the stream must equal
(after taps // 2 leading zeros).  The knobs inject plausible mistakes, so that the tests can show each one is caught:
``stack_short`` (each residual-stack history one row short), ``fresh_zero`` (a fresh item's conv histories zero
instead of padded from the chunk), ``up_zero`` (a fresh item's conv-transpose history zero instead of replicated),
``pq_short`` (the PQMF history one row short) and ``flush_edge`` (the flush repeats the last subband sample instead of
reading zeros)."""
import torch
import torch.nn.functional as F

from .ref_ops import causal_conv_transpose1d, melgan_layer_index, pqmf_filters, pqmf_synthesis
from .ref_stream import drive, keep

MODES = {"reflect": "reflect", "replicate": "replicate", "zero": "constant"}


def _causal_whole(x, w, b, d, mode):
    """CausalConv1d.forward with the model's pad (layers/causal_conv.py:32-43)"""
    n = (w.shape[-1] - 1) * d
    xp = F.pad(x, (n, n), mode=MODES[mode]) if n else x
    return F.conv1d(xp, w, b, dilation=d)[:, :, :x.shape[2]]


def whole_utterance(w, c, cfg, pad="reflect", subbands=None):
    """``MelGANGenerator.inference`` (with ``model.pqmf`` of ``subbands`` bands) for a batch of whole utterances c (B, in, T)"""
    slope = cfg.get("negative_slope", 0.2)
    sk = cfg.get("stack_kernel_size", 3)
    for kind, idx, meta in melgan_layer_index(dict(cfg, use_causal_conv=True)):
        p = f"melgan.{idx}"
        if kind == "conv_in":
            c = _causal_whole(c, w[p + ".conv.weight"], w.get(p + ".conv.bias"), 1, pad)
        elif kind == "convt":
            c = causal_conv_transpose1d(F.leaky_relu(c, slope), w[p + ".deconv.weight"], w.get(p + ".deconv.bias"), meta[1])
        elif kind == "stack":
            h = _causal_whole(F.leaky_relu(c, slope), w[p + ".stack.1.conv.weight"], w.get(p + ".stack.1.conv.bias"), sk ** meta[1], pad)
            h = F.conv1d(F.leaky_relu(h, slope), w[p + ".stack.3.weight"], w.get(p + ".stack.3.bias"))
            c = h + F.conv1d(c, w[p + ".skip_layer.weight"], w.get(p + ".skip_layer.bias"))
        else:
            c = _causal_whole(F.leaky_relu(c, slope), w[p + ".conv.weight"], w.get(p + ".conv.bias"), 1, pad)
            if cfg.get("use_final_nonlinear_activation", True):
                c = torch.tanh(c)
    if subbands:
        c = pqmf_synthesis(c, pqmf_filters(subbands)[1].to(c.dtype))
    return c


class MelGANStreamRef:
    """push(c (B, in_channels, n)) -> (B, 1, n * hop * subbands); flush() -> (B, 1, delay)."""

    def __init__(self, w, cfg, pad="reflect", subbands=None, batch=1, dtype=torch.float64, stack_short=0, fresh_zero=False,
                 up_zero=False, pq_short=0, flush_edge=False):
        self.w = {k: v.to(dtype) for k, v in w.items()}
        self.cfg, self.pad, self.B, self.dtype = cfg, pad, batch, dtype
        self.stack_short, self.fresh_zero, self.up_zero, self.pq_short, self.flush_edge = stack_short, fresh_zero, up_zero, pq_short, flush_edge
        self.slope = cfg.get("negative_slope", 0.2)
        self.plan = melgan_layer_index(dict(cfg, use_causal_conv=True))
        self.sk = cfg.get("stack_kernel_size", 3)
        self.hist = {}  # layer index -> history (B, C, H)
        self.N = subbands
        if subbands:
            self.f_syn = pqmf_filters(subbands)[1].to(dtype)
            self.taps = self.f_syn.shape[-1] - 1
            self.D = self.taps // 2
            self.pq = torch.zeros(batch, subbands, self.taps // subbands, dtype=dtype)
        self.fresh = True

    def _conv(self, key, x, w, b, d):
        """a causal conv of the chunk x given its history (or, for a fresh item, the pad read from x)"""
        P = (w.shape[-1] - 1) * d
        if self.fresh:
            if self.fresh_zero or self.pad == "zero":
                h = x.new_zeros(x.shape[0], x.shape[1], P)
            elif self.pad == "reflect":
                h = x[:, :, 1:P + 1].flip(-1)
            else:
                h = x[:, :, :1].expand(-1, -1, P)
        else:
            h = self.hist[key]
        xp = torch.cat([h, x], -1)
        self.hist[key] = keep(xp, P, self.stack_short if key[0] == "stack" else 0)
        return F.conv1d(xp, w, b, dilation=d)

    def _synth(self, y):
        """the synthesis window of subband chunk y (B, N, m), m * N samples lagging by D"""
        N, H = self.N, self.pq.shape[-1]
        full = torch.cat([self.pq, y], -1)
        self.pq = keep(full, H, self.pq_short)
        z = torch.zeros(full.shape[0], N, full.shape[-1] * N, dtype=full.dtype)
        z[..., ::N] = full * N
        lead = self.taps - H * N  # zero-stuffed samples in front of the oldest history row that the filter still reaches
        z = F.pad(z, (lead, 0)) if lead >= 0 else z[..., -lead:]
        return F.conv1d(z, self.f_syn)

    def push(self, c):
        w, slope = self.w, self.slope
        c = c.to(self.dtype)
        for kind, idx, meta in self.plan:
            p = f"melgan.{idx}"
            if kind == "conv_in":
                c = self._conv(("in",), c, w[p + ".conv.weight"], w.get(p + ".conv.bias"), 1)
            elif kind == "convt":
                x = F.leaky_relu(c, slope)  # lrelu commutes with the replicated frame
                hist = x[:, :, :1] if self.fresh and not self.up_zero else self.hist.get(("up", idx), x.new_zeros(x.shape[0], x.shape[1], 1))
                xp = torch.cat([hist, x], -1)
                self.hist[("up", idx)] = xp[:, :, -1:]
                s = meta[1]
                c = F.conv_transpose1d(xp, w[p + ".deconv.weight"], w.get(p + ".deconv.bias"), stride=s)[:, :, s:-s]
            elif kind == "stack":
                h = self._conv(("stack", idx), F.leaky_relu(c, slope), w[p + ".stack.1.conv.weight"], w.get(p + ".stack.1.conv.bias"),
                               self.sk ** meta[1])
                h = F.conv1d(F.leaky_relu(h, slope), w[p + ".stack.3.weight"], w.get(p + ".stack.3.bias"))
                c = h + F.conv1d(c, w[p + ".skip_layer.weight"], w.get(p + ".skip_layer.bias"))
            else:
                c = self._conv(("out",), F.leaky_relu(c, slope), w[p + ".conv.weight"], w.get(p + ".conv.bias"), 1)
                if self.cfg.get("use_final_nonlinear_activation", True):
                    c = torch.tanh(c)
        if self.N:
            y = self._synth(c)
            if self.fresh:
                y[:, :, :self.D] = 0.0
            c = y
        self.fresh = False
        return c

    def flush(self):
        if not self.N:
            return torch.zeros(self.B, 1, 0, dtype=self.dtype)
        rows = -(-self.D // self.N)
        tail = self.pq[:, :, -1:].expand(-1, -1, rows) if self.flush_edge else self.pq.new_zeros(self.B, self.N, rows)
        return self._synth(tail)[:, :, :self.D]


def stream(w, c, cfg, schedule, pad="reflect", subbands=None, first=None, **kw):
    """Run ``MelGANStreamRef`` over c (B, in_channels, T) in chunks of ``schedule`` frames (after a first chunk of ``first``
    frames if given; repeated until the utterance is used up, the last chunk cut short), flush, and return the
    concatenated output"""
    ref = MelGANStreamRef(w, cfg, pad=pad, subbands=subbands, batch=c.shape[0], **kw)
    return drive(lambda j, n: ref.push(c[:, :, j:j + n]), c.shape[-1], schedule, ref.flush, first)
