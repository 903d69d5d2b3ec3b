"""Chunked CPU restatement of streaming a discrete-symbol HiFi-GAN (``DiscreteSymbolHiFiGANGenerator``) with a fixed
lookahead (TEST INFRASTRUCTURE), on top of ``oracle/ref_discrete.py`` and ``oracle/ref_hifigan_lookahead_stream.py``.  It
carries the same state as ``parallelwavegan_b200.streaming.DiscreteSymbolHiFiGANLookaheadStream``, explicitly and in
plain tensors.

The generator is the symbol embedding (+ the speaker embedding of each item's first frame, added to every frame)
followed by the centred HiFi-GAN body.  With every upsampling kernel 2 s and s even, the conv-transpose padding
(k - s) // 2 = s / 2 is the HiFi-GAN one, so the body streams exactly as ``HiFiGANLookaheadRef``: the embedding of a
chunk is that stream's input chunk, and the flush pushes zero frames (the whole utterance's zero right padding; the GPU
stream writes the zeros from the end mask whatever ids the flush pushes).  The one new piece of state is the speaker: it
is latched from the first frame pushed after a reset, because the whole-utterance forward reads ``c[:, 1, 0]`` only.

``chunk_speaker`` injects a plausible mistake: taking the speaker from each chunk's first frame."""
import torch
import torch.nn.functional as F

from .ref_discrete import dsym_generator
from .ref_hifigan_lookahead_stream import HiFiGANLookaheadRef
from .ref_stream import drive


def body_cfg(cfg):
    """the HiFi-GAN configuration of the generator's body, as ``HiFiGANLookaheadRef`` reads it"""
    slope = cfg.get("nonlinear_activation_params", {"negative_slope": 0.1}).get("negative_slope", 0.1)
    return dict(cfg, negative_slope=slope, use_causal_conv=False)


def whole_utterance(w, c, cfg):
    """``DiscreteSymbolHiFiGANGenerator.forward`` on whole utterances c (B, 1 or 2, T)"""
    return dsym_generator(w, c, cfg)


class DSymLookaheadRef:
    """push(c (B, 1 or 2, n) indices) -> (B, out_channels, n * hop); flush() -> (B, out_channels, delay)."""

    def __init__(self, w, cfg, batch=1, dtype=torch.float64, chunk_speaker=False):
        for s, k in zip(cfg["upsample_scales"], cfg["upsample_kernel_sizes"]):
            assert k == 2 * s and s % 2 == 0, (s, k)
        self.w = {k: v.to(dtype) for k, v in w.items()}
        self.cfg, self.B, self.dtype, self.chunk_speaker = cfg, batch, dtype, chunk_speaker
        self.use_spk = cfg.get("num_spk_embs", 128) > 0
        self.body = HiFiGANLookaheadRef(self.w, body_cfg(cfg), batch, dtype)
        self.delay, self.hop = self.body.delay, self.body.hop
        self.spk = None

    def _embed(self, c):
        c = c.long()
        e = F.embedding(c[:, 0], self.w["emb.weight"]).transpose(1, 2)
        if self.use_spk:
            if self.spk is None or self.chunk_speaker:
                self.spk = c[:, 1, 0].clone()
            e = e + F.embedding(self.spk, self.w["spk_emb.weight"]).unsqueeze(2)
        return e

    def push(self, c):
        return self.body.push(self._embed(c))

    def flush(self):
        y = self.body.flush()
        self.spk = None
        return y


def stream(w, c, cfg, schedule, **kw):
    """Run ``DSymLookaheadRef`` over c (B, K, T) in chunks of ``schedule`` frames (repeated until the utterance is used
    up; the last chunk is cut short), then flush; returns cat(pushes, flush)."""
    ref = DSymLookaheadRef(w, cfg, batch=c.shape[0], **kw)
    return drive(lambda j, n: ref.push(c[:, :, j:j + n]), c.shape[-1], schedule, ref.flush)


class DSymDurationLookaheadRef:
    """``DiscreteSymbolDurationGenerator`` (no speakers) streamed for one item: push(ids (m,)) -> (1, out_channels, n *
    hop), flush() -> (1, out_channels, L); ``durations`` lists every finalised duration in order.

    * The duration predictor runs in delayed time: a symbol is final once ``look`` = P = n_layers * (k - 1) / 2 symbols
      after it have arrived, or at the flush.  Its log-duration is computed from the symbols that have arrived, with
      every layer's output (the conv's and the LayerNorm's) zero outside [0, symbols known) -- the whole utterance's zero
      padding.  With ``look`` = P that equals the whole-utterance predictor.
    * Final durations (rounded as ``DurationPredictor.inference``) enter a queue of [id, frames left] entries.
    * The body advances by every queued frame, in power-of-two pushes of ``HiFiGANLookaheadRef``; a run may span pushes.
    * The flush finalises the last P symbols, applies the all-zero rule if the item's total is still 0 (every kept entry
      gets one frame), drains the queue and flushes the body.

    Knobs inject plausible mistakes: ``look`` = 1, ``ln_unmasked`` (LayerNorm output left unmasked outside the signal:
    beta there), ``zero_rule_per_chunk`` (the all-zero rule applied to each push's final durations), ``restart_runs`` (a run
    restarts from its first frame at each body push) and ``flush_no_tail`` (the flush skips the predictor's last P
    symbols)."""

    def __init__(self, w, cfg, dtype=torch.float64, look=None, ln_unmasked=False, zero_rule_per_chunk=False, restart_runs=False,
                 flush_no_tail=False):
        for s, k in zip(cfg["upsample_scales"], cfg["upsample_kernel_sizes"]):
            assert k == 2 * s and s % 2 == 0, (s, k)
        assert cfg.get("num_spk_embs", 128) <= 0
        self.w = {k: v.to(dtype) for k, v in w.items()}
        self.cfg, self.dtype = cfg, dtype
        self.k, self.layers = cfg.get("duration_kernel_size", 3), cfg.get("duration_layers", 2)
        self.P = self.layers * (self.k - 1) // 2
        self.look = self.P if look is None else look
        self.ln_unmasked, self.zero_rule_per_chunk, self.restart_runs, self.flush_no_tail = (ln_unmasked, zero_rule_per_chunk,
                                                                                          restart_runs, flush_no_tail)
        self.body = HiFiGANLookaheadRef(self.w, body_cfg(cfg), 1, dtype)
        self.delay, self.hop = self.body.delay, self.body.hop
        self.syms, self.nfinal, self.queue, self.total, self.durations, self.log_durations = [], 0, [], 0, [], []

    def _log_durations(self):
        w, k, P = self.w, self.k, self.P
        S = len(self.syms)
        e = F.embedding(torch.tensor(self.syms), w["emb.weight"]).t()[None]
        h = F.pad(e, (P + 1, P + 1))
        valid = ((torch.arange(h.shape[-1]) - (P + 1)) >= 0) & ((torch.arange(h.shape[-1]) - (P + 1)) < S)
        p = "duration_predictor"
        for i in range(self.layers):
            h = F.relu(F.conv1d(h, w[f"{p}.conv.{i}.0.weight"], w[f"{p}.conv.{i}.0.bias"], padding=(k - 1) // 2)) * valid
            h = F.layer_norm(h.transpose(1, 2), (h.shape[1],), w[f"{p}.conv.{i}.2.weight"], w[f"{p}.conv.{i}.2.bias"], 1e-12).transpose(1, 2)
            if not self.ln_unmasked:
                h = h * valid
        x = F.linear(h.transpose(1, 2), w[f"{p}.linear.weight"], w[f"{p}.linear.bias"])[0, :, 0]
        return x[P + 1:P + 1 + S]

    def _finalise(self, upto):
        if upto <= self.nfinal:
            return
        x = self._log_durations()[self.nfinal:upto]
        self.log_durations += x.tolist()
        d = torch.clamp(torch.round(x.exp() - self.cfg.get("duration_offset", 1.0)), min=0).long()
        if self.zero_rule_per_chunk and int(d.sum()) == 0:
            d = torch.ones_like(d)
        for j, dj in zip(range(self.nfinal, upto), d.tolist()):
            self.queue.append([self.syms[j], dj, dj, False])
            self.durations.append(dj)
            self.total += dj
        self.nfinal = upto

    def _drain(self):
        n, outs = sum(q[2] for q in self.queue), []
        p = 1 << max(n.bit_length() - 1, 0)
        while n > 0:
            if p <= n:
                q0 = self.queue[0]
                if self.restart_runs and 0 < q0[2] < q0[1] and not q0[3]:  # once per run, so the drain ends
                    q0[2], q0[3] = q0[1], True
                rows = []
                while len(rows) < p:
                    if self.queue[0][2] == 0:
                        self.queue.pop(0)
                        continue
                    rows.append(self.queue[0][0])
                    self.queue[0][2] -= 1
                e = F.embedding(torch.tensor(rows), self.w["emb.weight"]).t()[None]
                outs.append(self.body.push(e))
                n = sum(q[2] for q in self.queue)
                p = 1 << max(n.bit_length() - 1, 0)
                continue
            p >>= 1
        return torch.cat(outs, -1) if outs else torch.zeros(1, self.cfg.get("out_channels", 1), 0, dtype=self.dtype)

    def push(self, ids):
        self.syms += [int(i) for i in ids]
        self._finalise(max(len(self.syms) - self.look, 0))
        return self._drain()

    def flush(self):
        if not self.flush_no_tail:
            self._finalise(len(self.syms))
        if self.total == 0:
            for q in self.queue:
                q[2] = 1
        y = torch.cat([self._drain(), self.body.flush()], -1)
        self.syms, self.nfinal, self.queue, self.total = [], 0, [], 0
        return y


def duration_stream(w, c, cfg, schedule, **kw):
    """Run ``DSymDurationLookaheadRef`` over the symbols c (S,) in pushes of ``schedule`` symbols, then flush; returns
    (cat(pushes, flush), the finalised durations, their log-domain values)."""
    ref = DSymDurationLookaheadRef(w, cfg, **kw)
    y = drive(lambda j, n: ref.push(c[j:j + n]), len(c), schedule, ref.flush)
    return y, torch.tensor(ref.durations), torch.tensor(ref.log_durations, dtype=torch.float64)
