"""Chunked synthesis: mel frames in, waveform out, while the frames are still arriving.  ``CausalPWGStream`` streams a
causal Parallel WaveGAN, ``CausalHiFiGANStream`` a causal HiFi-GAN, ``CausalMelGANStream`` a causal (multi-band) MelGAN,
and ``HiFiGANLookaheadStream``, ``PWGLookaheadStream``, ``MelGANLookaheadStream`` and ``UHiFiGANLookaheadStream`` a centred
HiFi-GAN, a centred Parallel WaveGAN, a centred (multi-band) MelGAN and a centred U-Net HiFi-GAN (excitation pushed with
its frames) with a fixed lookahead and a flush; ``DiscreteSymbolHiFiGANLookaheadStream`` streams a discrete-symbol HiFi-GAN
(HuBERT units in, audio out), ``DiscreteSymbolDurationLookaheadStream`` its duration model (durations predicted as the
units arrive) and ``VQVAELookaheadStream`` a VQ-VAE's wav2wav conversion (audio in, converted audio out) the
same way.

A causal generator's output for frame j depends only on frames <= j, so it can be synthesised as soon as frame j
exists.  ``CausalPWGStream`` carries, per batch slot, everything the whole-utterance forward would read from before
the current chunk:

* conv_in (ConvInUpsampleNetwork): the last ``aux_context_window`` mel frames.  A fresh slot starts from its first
  frame replicated, as ``ReplicationPad1d`` does in ``inference``; conv_in then runs as a valid conv on
  [history | chunk];
* every causal FIR stage of the upsampler: its last two input frames, read by pwgb_upsample_fir_causal_stream_forward;
  these and the conv_in history are updated by one pwgb_stream_carry after the last FIR stage;
* every WaveNet layer l: its last H_l = (kernel - 1) * dilation_l input samples, in the packed residual stream's
  operand layout.  A causal layer reads only those rows in front of sample 0, so one copy per layer boundary
  (pwgb_wnstack_carry) puts the history where the whole-utterance forward has the previous samples, and the unchanged
  fused layer kernel computes the chunk as that forward would.

Every kernel computes each output sample with the same fp32 expression as ``model.inference`` on the whole utterance,
so the concatenated chunks equal it bit for bit as long as both runs take the same kernels (see DESIGN.md).  The
state is zeros for a fresh signal (the whole-utterance zero padding), so ``reset`` is a memset."""
import contextlib

import torch

from . import ops
from .capi import PwgbError
from .layers import ConvInUpsampleNetwork, UpsampleNetwork, effective_weight


def _layer_weights(f, A, causal=True):
    """The packed operand image of one WaveNet layer, shared with ParallelWaveGANGenerator._forward_packed's cache."""
    k = ops.param_key(f.conv, f.conv1x1_aux, f.conv1x1_skip, f.conv1x1_out)
    ent = f._cache.get("wnp")
    if ent is not None and ent[0] == k:
        return ent[1], ent[2]
    return ops.wavenet_packed_weights(effective_weight(f.conv), effective_weight(f.conv1x1_aux), effective_weight(f.conv1x1_skip),
                                      effective_weight(f.conv1x1_out), f.conv1x1_skip.bias, f.conv1x1_out.bias, A,
                                      cache=f._cache, key=k, causal=causal)


def wb(conv):
    """(weight, bias) of a conv container, read once when a stream is built"""
    return effective_weight(conv).detach().contiguous(), (conv.bias.detach() if conv.bias is not None else None)


class _ChunkStream:
    """Plumbing shared by the streams:

    * slot validation, and ``reset`` / ``state_bytes`` over the batch-leading state tensors of ``_state()``;
    * the mel frames of a push, checked, normalised if asked and laid out as (B, C, n);
    * the input conv's history of ``history`` frames: a fresh slot's is filled as the model's pad (``"zero"``,
      ``"replicate"`` or ``"reflect"``) would fill it, and ``_input`` copies [history | chunk] into the entry's ``xin``
      buffer, which the subclass's carry table carries into the history;
    * the fresh slots: a host list, and with ``flags`` the same as device int32 flags (``fresh``) for the kernels that
      read them; the subclass clears those inside the captured push;
    * one cached entry per chunk length (at most ``MAX_CHUNK_LENGTHS``), and one CUDA graph per chunk length captured
      after an eager warm-up whose state changes are undone; the result is cloned once, in ``_run``.

    A subclass provides ``_state()`` (the tensors a push advances, including ``cin_hist``), ``_new_entry(n, xin)`` and
    ``_step(*inputs)``, which writes into the entry's buffers."""

    MAX_CHUNK_LENGTHS = 8

    def _setup(self, model, batch, use_graphs, in_channels, history, pad, flags=False):
        self._check_eval(model)
        self.model = model
        self.dev = next(model.parameters()).device
        if self.dev.type != "cuda":
            raise PwgbError(f"{type(self).__name__}: the model must live on a CUDA device (no CPU fallback)")
        self.B = int(batch)
        if self.B < 1:
            raise PwgbError(f"{type(self).__name__}: batch must be >= 1")
        self.use_graphs = bool(use_graphs)
        self._entries = {}  # chunk frames -> per-length data and "graph"; a graph lives and dies with its entry
        self.in_channels, self.pad = in_channels, pad
        self.cin_hist = self._zeros(self.B, in_channels, history)
        self._fresh = [True] * self.B
        self.fresh = torch.ones(self.B, device=self.dev, dtype=torch.int32) if flags else None

    def _zeros(self, *shape):
        return torch.zeros(shape, device=self.dev, dtype=torch.float32)

    def _empty(self, *shape):
        return torch.empty(shape, device=self.dev, dtype=torch.float32)

    def _check_eval(self, model):
        if model.training:
            raise PwgbError(f"{type(self).__name__}: the model is in train mode; call model.eval() (dropout would apply)")

    def _slots(self, items):
        """``items`` (an index, an iterable of indices or None for every slot) as a checked list"""
        items = range(self.B) if items is None else ([items] if isinstance(items, int) else list(items))
        for b in items:
            if not 0 <= b < self.B:
                raise PwgbError(f"{type(self).__name__}.reset: slot {b} out of range [0, {self.B})")
        return items

    def state_bytes(self):
        """bytes of carried state per slot"""
        return sum(t.numel() * t.element_size() for t in self._state()) // self.B

    def reset(self, items=None):
        """Restart slots ``items`` (an index or an iterable of indices; None: every slot) as fresh signals.  The other
        slots continue unaffected."""
        for b in self._slots(items):
            for h in self._state():
                h[b].zero_()
            self._fresh[b] = True
            if self.fresh is not None:
                self.fresh[b] = 1

    def _frames(self, c, normalize_before):
        """c: (B, n, C) mel frames ((n, C) when batch == 1) -> (B, C, n) contiguous on the device"""
        m = self.model
        self._check_eval(m)
        c = torch.as_tensor(c, dtype=torch.float32, device=self.dev)
        if c.dim() == 2 and self.B == 1:
            c = c.unsqueeze(0)
        if c.dim() != 3 or c.shape[0] != self.B or c.shape[2] != self.in_channels or c.shape[1] < 1:
            raise PwgbError(f"{type(self).__name__}.push: c must be ({self.B}, n >= 1, {self.in_channels}), got {tuple(c.shape)}")
        if normalize_before:
            c = (c - m.mean) / m.scale
        return c.transpose(1, 2).contiguous()

    def _start(self, c):
        """Fill the input-conv history of the fresh slots from their first chunk c (B, C, n) as the pad would: frames
        P .. 1 (reflect), frame 0 repeated (replicate) or the reset's zeros."""
        P = self.cin_hist.shape[-1]
        for b in range(self.B):
            if self._fresh[b] and P and self.pad != "zero":
                self.cin_hist[b].copy_(c[b, :, 1:P + 1].flip(-1) if self.pad == "reflect" else c[b, :, :1].expand(-1, P))
        self._fresh = [False] * self.B

    def _input(self, ent, c):
        """[history | chunk] in the entry's xin buffer, the input of the input conv"""
        P = self.cin_hist.shape[-1]
        xin = ent["xin"]
        xin[:, :, :P].copy_(self.cin_hist)
        xin[:, :, P:].copy_(c)
        return xin

    def _entry(self, n):
        ent = self._entries.get(n)
        if ent is None:
            if len(self._entries) >= self.MAX_CHUNK_LENGTHS:
                self._entries.clear()
            xin = self._empty(self.B, self.in_channels, self.cin_hist.shape[-1] + n)
            ent = self._entries[n] = self._new_entry(n, xin)
            ent["xin"] = xin
        return ent

    def _replay(self, n, inputs):
        ent = self._entry(n)
        if "graph" not in ent:
            static = [t.clone() for t in inputs]
            # one eager warm-up (packs weights, sets kernel attributes, fills the per-shape caches) advances the state
            # and clears the flags: both are restored before the capture, which itself runs nothing
            carried = self._state() + ([self.fresh] if self.fresh is not None else [])
            snap = [t.clone() for t in carried]
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                self._step(*static)
            torch.cuda.current_stream().wait_stream(side)
            for t, s in zip(carried, snap):
                t.copy_(s)
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                out = self._step(*static)
            ent.update(graph=graph, inputs=static, out=out)
        for s, t in zip(ent["inputs"], inputs):
            s.copy_(t)
        ent["graph"].replay()
        return ent["out"]

    def _run(self, n, *inputs):
        """One push; the result is the caller's own tensor (the graph's output and the entry's buffers are reused)"""
        y = self._replay(n, inputs) if self.use_graphs else self._step(*inputs)
        return y.clone()


class _Lookahead:
    """The frame / end counters of a stream with a fixed lookahead, shared by the centred streams: the mask of every launch
    (``_mask``), ``reset`` reopening a slot's end, and ``_flush`` (a push with the flushed slots' end frames set, the other
    slots' state restored around it, then the flushed slots reset).  Mixed in before the stream's base class."""

    OPEN = 2 ** 31 - 1  # the end frame of a slot whose signal has not ended
    subbands = 1  # output samples per frame are hop * subbands (a multi-band MelGAN's PQMF synthesis sets its own)

    def _counters(self):
        """the frame counters, the open end frames, and the empty history of the input conv's launch on [history | chunk]"""
        self.frame = torch.zeros(self.B, device=self.dev, dtype=torch.int32)
        self.end = torch.full((self.B,), self.OPEN, device=self.dev, dtype=torch.int32)
        self._nohist = self._zeros(self.B, self.in_channels, 0)

    def reset(self, items=None):
        super().reset(items)
        for b in self._slots(items):
            self.end[b] = self.OPEN

    def _mask(self, rate, look):
        return (self.frame, self.end, rate, look)

    def _flush_frames(self):
        """the frames of a flush push: the fewest whose output covers ``delay`` samples"""
        return -(-self.delay // (self.hop * self.subbands))

    @contextlib.contextmanager
    def _keeping_others(self, items):
        """Restores the state (and the fresh flags) of every slot but ``items`` (a checked list) after the block, so those
        slots continue exactly as if it had not run."""
        keep = [b for b in range(self.B) if b not in items]
        carried = self._state() + ([self.fresh] if self.fresh is not None else [])
        snap = [t[keep].clone() for t in carried] if keep else []
        yield
        for t, s in zip(carried, snap):
            t[keep] = s

    def _flush(self, items, inputs):
        """The first ``delay`` samples of the flush push ``inputs()`` (the arguments of ``_run``) for slots ``items`` (a
        checked list); the other slots continue exactly as if it had not happened."""
        sel = torch.tensor(items, device=self.dev, dtype=torch.long)
        with self._keeping_others(items):
            self.end[sel] = self.frame[sel]
            y = self._run(*inputs())[sel, :, :self.delay].contiguous()
        self.reset(items)
        return y


class _PWGStream(_ChunkStream):
    """The weights, histories and noise of a streamed ``ParallelWaveGANGenerator``, shared by the causal stream and the
    centred one with lookahead: the conv_in and FIR weights of the upsampler and one history per FIR stage (its last two
    input frames), the WaveNet shapes and one packed history per layer (its last (K - 1) * d_l input samples), the output
    head, and the generator that draws the noise a push is not given."""

    def _build(self, model, batch, use_graphs, seed, causal):
        from .models import MelGANGenerator, ParallelWaveGANGenerator

        name = type(self).__name__
        if not isinstance(model, ParallelWaveGANGenerator):
            raise PwgbError(f"{name}: expected a ParallelWaveGANGenerator")
        if causal and not model.use_causal_conv:
            raise PwgbError(f"{name}: the model is not causal (use_causal_conv=False); a centred model needs lookahead")
        if not causal and model.use_causal_conv:
            raise PwgbError(f"{name}: the model is causal (use_causal_conv=True); stream it with CausalPWGStream, which has no "
                            "lookahead")
        up = model.upsample_net
        if up is None:
            raise PwgbError(f"{name}: upsample_conditional_features=False is not supported")
        if isinstance(up, MelGANGenerator):
            raise PwgbError(f"{name}: upsample_net='MelGANGenerator' is not supported")
        if isinstance(up, UpsampleNetwork) and model.aux_context_window:
            raise PwgbError(f"{name}: UpsampleNetwork with aux_context_window > 0 has no whole-utterance inference to match")
        conv_in = up.conv_in if isinstance(up, ConvInUpsampleNetwork) else None
        self.acw = model.aux_context_window if conv_in is not None else 0
        self.A = model.aux_channels
        # ReplicationPad1d of inference: a fresh slot's conv_in history is its first frame; the centred conv_in reads acw
        # frames on either side
        self._setup(model, batch, use_graphs, self.A, self.acw if causal else 2 * self.acw, "replicate")
        fir_net = up.upsample if conv_in is not None else up
        self.scales = list(fir_net.upsample_scales)
        self.w_in = wb(conv_in)[0] if conv_in is not None else None
        self.firs = [wb(fir_net.up_layers[2 * i + 1])[0] for i in range(len(self.scales))]
        self.hop = model.upsample_factor
        l0 = model.conv_layers[0]
        self.R, self.G, self.K = l0.conv.in_channels, l0.conv.out_channels, l0.conv.kernel_size[0]
        self.S = l0.conv1x1_skip.out_channels
        self.dmax = max(f.dilation for f in model.conv_layers)
        self.H = [(self.K - 1) * f.dilation for f in model.conv_layers]
        if not ops.WnStack.supported(self.B, self.hop, self.R, self.G, self.S, self.A, self.K, self.dmax, causal):
            raise PwgbError(f"{name}: the fused packed WaveNet stack does not support this configuration "
                            f"(residual {self.R}, gate {self.G}, skip {self.S}, aux {self.A} channels, kernel {self.K})")
        self.w_first = wb(model.first_conv)
        # the output head as in ParallelWaveGANGenerator.forward: sqrt(1/layers) folded into the first 1x1 conv
        w1, b1 = wb(model.last_conv_layers[1])
        self.w_l1, self.w_l3 = (w1 * model._skip_scale, b1), wb(model.last_conv_layers[3])
        dev, B, A = self.dev, self.B, self.A
        self.fir_hist = [self._zeros(B, A, 2) for _ in self.scales]
        self.wn_hist = [torch.zeros((B, self.R * h), device=dev, dtype=torch.int32) for h in self.H]
        self.gen = torch.Generator(device=dev)
        if seed is not None:
            self.gen.manual_seed(int(seed))

    def _noise(self, z, T):
        """z: (B, in_channels, T) noise on the device, drawn from the stream's generator when None"""
        shape = (self.B, self.model.in_channels, T)
        if z is None:
            return torch.randn(shape, device=self.dev, generator=self.gen)
        z = torch.as_tensor(z, dtype=torch.float32, device=self.dev)
        if tuple(z.shape) != shape:
            raise PwgbError(f"{type(self).__name__}.push: z must be {shape}, got {tuple(z.shape)}")
        return z.contiguous()

    @torch.no_grad()
    def push(self, c, z=None, normalize_before=False):
        """c: (B, n, aux) mel frames ((n, aux) when batch == 1); z: optional (B, in_channels, n * hop) noise of those
        frames, drawn from the stream's generator when omitted.  Returns (B, out_channels, n * hop) on the device: the
        frames' samples (causal), or samples [t0 * hop - delay, (t0 + n) * hop - delay) of each slot's utterance (with
        lookahead; t0: the frames pushed before)."""
        c = self._frames(c, normalize_before)
        z = self._noise(z, c.shape[-1] * self.hop)
        self._start(c)
        return self._run(c.shape[-1], z, c)


class CausalPWGStream(_PWGStream):
    """Streams a causal ``ParallelWaveGANGenerator`` chunk by chunk for ``batch`` independent slots.

    ``push(c, z)`` takes the next n >= 1 frames of every slot and returns their n * hop samples; n may change from
    push to push.  For every slot, the concatenated outputs equal ``model.inference(c=all_frames, x=all_noise)``.
    There is no lookahead and no flush.  With ``use_graphs`` each chunk length is captured once into a CUDA graph and
    replayed.  The weights are read when the stream is built and must not change while it is used."""

    def __init__(self, model, batch=1, seed=None, use_graphs=True):
        self._build(model, batch, use_graphs, seed, causal=True)

    def _state(self):
        return [self.cin_hist] + self.fir_hist + self.wn_hist

    def _new_entry(self, n, xin):
        """The conditioning's buffers for an n-frame chunk, the carry table of the conv_in and FIR histories over them,
        and the packed WaveNet stack."""
        dev, B, A = self.dev, self.B, self.A
        ent = dict(stack=ops.WnStack(B, n * self.hop, self.R, self.G, self.S, A, self.K, self.dmax, dev, True),
                   skips=self._empty(B, self.S, n * self.hop))
        ent["cin"] = self._empty(B, A, n) if self.w_in is not None else xin
        entries, x, t = [(xin, self.cin_hist)], ent["cin"], n
        ent["fir"] = []
        for i, s in enumerate(self.scales):
            entries.append((x, self.fir_hist[i]))
            t *= s
            # the last stage writes the first A of the stack's aux_pad channels; the others stay zero
            x = self._zeros(B, self.model._aux_pad, t) if i == len(self.scales) - 1 else self._empty(B, A, t)
            ent["fir"].append(x)
        ent["table"] = ops.stream_carry_table(entries, dev)
        return ent

    def _step(self, z, c):
        """One chunk: z (B, in_channels, n * hop), c (B, aux, n) -> (B, out_channels, n * hop).  Advances the state."""
        m = self.model
        ent = self._entry(c.shape[-1])
        # conditioning: conv_in on [history | chunk], then the causal FIR stages reading their histories; one carry after
        # the last of them updates every history they read
        x = self._input(ent, c)
        if self.w_in is not None:
            x = ops.conv1d(x, self.w_in, None, out=ent["cin"])
        for i, s in enumerate(self.scales):
            x = ops.upsample_fir_causal_stream(x, self.firs[i], s, self.fir_hist[i], out=ent["fir"][i],
                                               out_channels=ent["fir"][i].shape[1])
        ops.stream_carry(ent["table"])
        # the residual stack on the packed stream; each layer's history is carried between the layer launches
        st = ent["stack"]
        st.cur, st.prev = 0, None
        st.pack_c(x)
        st.first_conv(z, *self.w_first)
        skips = ent["skips"]
        layers = m.conv_layers
        L = len(layers)
        st.carry(load=(self.wn_hist[0], self.H[0]))
        for i, f in enumerate(layers):
            packed, bso = _layer_weights(f, self.A)
            st.layer(packed, f.conv.bias, bso, f.dilation, skips, skips_init=(i == 0), write_x=(i < L - 1))
            st.carry(save=(self.wn_hist[i], self.H[i]), load=(self.wn_hist[i + 1], self.H[i + 1]) if i + 1 < L else None)
        h = ops.conv1d(skips, *self.w_l1, pre_slope=0.0)
        # into a fresh tensor, as in inference: given out=, a wide few-channel output conv would not take _conv1d_fewcout
        return ops.conv1d(h, *self.w_l3, pre_slope=0.0)


class PWGLookaheadStream(_Lookahead, _PWGStream):
    """Streams a centred ``ParallelWaveGANGenerator`` (``use_causal_conv=False``, the published checkpoints) chunk by chunk
    for ``batch`` independent slots, with a fixed lookahead of ``delay`` output samples.

    ``push(c, z)`` takes the next n >= 1 mel frames and their n * hop noise samples of every slot and returns n * hop
    samples: the whole-utterance samples from t0 * hop - delay on (t0: the frames pushed before), with zeros before sample
    0.  ``flush(items)`` returns the last ``delay`` samples of those slots and restarts them; the other slots continue as
    if no flush had happened.  For every slot, the concatenated pushes and flush equal ``[zeros(delay) |
    model.inference(all_frames, all_noise)]``.

    Each signal runs in delayed time behind the frames pushed (DESIGN.md §3.9, oracle/ref_pwg_lookahead_stream.py):

    * conv_in (kernel 2 acw + 1) runs on [the last 2 acw frames | chunk], acw frames behind; a fresh slot's history is its
      first frame replicated, and the flush pushes its last frame replicated (both edges of ``ReplicationPad1d``);
    * each FIR stage (scale s) reads [2 history frames | chunk] and is one frame behind its input
      (pwgb_upsample_fir_stream_ext_forward): lookahead look_c = 852 samples for v1 ([4, 4, 4, 4], acw 2);
    * the conditioning enters each WaveNet layer after its dilated conv, so the residual stream runs look_x = look_c -
      (K - 1) / 2 * d_0 behind: the noise goes through a look_x-sample delay line into first_conv;
    * WaveNet layer l is the causal tap pattern over the (K - 1) d_l history rows of the packed stream's left halo
      (pwgb_wnstack_layer_stream_ext_forward), look_x + D_l behind (D_l = sum_{j <= l} (K - 1) / 2 d_j), with its
      residual read (K - 1) / 2 d_l rows back, its conditioning read from a window that keeps the last off_L rows, and its
      skip added into an (off_L + T)-column accumulator at the columns of its output positions; layer 0 initialises them
      and the others add in layer order, as in ``inference``;
    * every signal a later layer reads is masked to +0.0 outside [0, end) (pwgb_stream_ext: device frame counters and end
      frames), the whole-utterance zero padding, and so is the output before sample 0.

    ``delay`` = look_x + D_L: 3920 samples (15.3 frames) for v1, the lookahead autograd measures on the model.  With
    ``use_graphs`` each chunk length is captured once into a CUDA graph and replayed.  The weights are read when the stream
    is built and must not change while it is used."""

    def __init__(self, model, batch=1, seed=None, use_graphs=True):
        self._build(model, batch, use_graphs, seed, causal=False)
        # the plan: lookaheads of conv_in (frames), of each FIR stage's output, of first_conv's output and of each layer's
        look, self.looks = self.acw, []
        self.look_in = self.acw
        for s in self.scales:
            look = look * s + s
            self.looks.append(look)
        self.look_c = look
        self.D, acc = [], 0
        for f in model.conv_layers:
            acc += (self.K - 1) // 2 * f.dilation
            self.D.append(acc)
        self.look_x = max(self.look_c - self.D[0], 0)
        self.off = [self.look_x + d - self.look_c for d in self.D]  # conditioning rows behind the newest, per layer
        self.W = self.off[-1]
        self.delay = self.look_x + self.D[-1]
        B, A = self.B, self.A
        self.z_hist = self._zeros(B, model.in_channels, self.look_x)
        self.c_hist = self._zeros(B, A, self.W)
        self.skip_hist = self._zeros(B, self.S, self.W)
        self._counters()

    def _state(self):
        return [self.cin_hist] + self.fir_hist + [self.z_hist, self.c_hist, self.skip_hist] + self.wn_hist + [self.frame, self.end]

    def _new_entry(self, n, xin):
        """The buffers of an n-frame chunk (conditioning stages, the noise, conditioning and skip windows), the packed
        WaveNet stack, and the carry table of every history but the WaveNet layers'."""
        dev, B, A, T = self.dev, self.B, self.A, n * self.hop
        ent = dict(stack=ops.WnStack(B, T, self.R, self.G, self.S, A, self.K, self.dmax, dev, causal=False, lookahead=True),
                   zw=self._empty(B, self.model.in_channels, self.look_x + T), cw=self._empty(B, A, self.W + T),
                   sw=self._zeros(B, self.S, self.W + T), skips=self._empty(B, self.S, T))
        ent["cin"] = self._empty(B, A, n) if self.w_in is not None else xin
        entries, x, t = [(xin, self.cin_hist)], ent["cin"], n
        ent["fir"] = []
        for i, s in enumerate(self.scales):
            entries.append((x, self.fir_hist[i]))
            t *= s
            x = self._empty(B, A, t)
            ent["fir"].append(x)
        entries += [(ent["zw"], self.z_hist), (ent["cw"], self.c_hist), (ent["sw"], self.skip_hist)]
        ent["table"] = ops.stream_carry_table(entries, dev)
        return ent

    def _step(self, z, c):
        """One chunk: z (B, in_channels, n * hop), c (B, aux, n) -> (B, out_channels, n * hop).  Advances the state."""
        m = self.model
        n = c.shape[-1]
        ent = self._entry(n)
        W, lx, hop = self.W, self.look_x, self.hop
        # conditioning: the masked conv_in on [history | chunk], then the masked FIR stages reading their histories
        x = self._input(ent, c)
        if self.w_in is not None:
            x = ops.conv1d_stream(x, self._nohist, self.w_in, None, pad_left=0, out=ent["cin"], mask=self._mask(1, self.look_in))
        rate = 1
        for i, s in enumerate(self.scales):
            rate *= s
            x = ops.upsample_fir_causal_stream(x, self.firs[i], s, self.fir_hist[i], out=ent["fir"][i], mask=self._mask(rate, self.looks[i]))
        # the windows [history | chunk] of the conditioning, the noise delay line and the skip accumulator
        cw, zw, sw = ent["cw"], ent["zw"], ent["sw"]
        cw[:, :, :W].copy_(self.c_hist)
        cw[:, :, W:].copy_(x)
        zw[:, :, :lx].copy_(self.z_hist)
        zw[:, :, lx:].copy_(z)
        sw[:, :, :W].copy_(self.skip_hist)
        # the residual stack on the packed stream; each layer's history is carried between the layer launches
        st = ent["stack"]
        st.cur, st.prev = 0, None
        cpk, c_rows = st.pack_c_window(cw)
        st.first_conv_stream(zw, *self.w_first, mask=self._mask(hop, lx))
        layers = m.conv_layers
        L = len(layers)
        st.carry(load=(self.wn_hist[0], self.H[0]))
        for i, f in enumerate(layers):
            packed, bso = _layer_weights(f, self.A, causal=False)
            col = W - self.off[i]
            st.layer_stream(packed, f.conv.bias, bso, f.dilation, cpk, c_rows, col, sw, col, self._mask(hop, lx + self.D[i]),
                            skips_init=(i == 0), write_x=(i < L - 1))
            st.carry(save=(self.wn_hist[i], self.H[i]), load=(self.wn_hist[i + 1], self.H[i + 1]) if i + 1 < L else None)
        skips = ent["skips"]
        skips.copy_(sw[:, :, :skips.shape[-1]])
        ops.stream_carry(ent["table"])
        h = ops.conv1d(skips, *self.w_l1, pre_slope=0.0)
        # into a fresh tensor, as in inference: given out=, a wide few-channel output conv would not take _conv1d_fewcout
        y = ops.stream_mask(ops.conv1d(h, *self.w_l3, pre_slope=0.0), self._mask(hop, self.delay))
        self.frame += n
        return y

    @torch.no_grad()
    def flush(self, items=None):
        """The last ``delay`` samples of slots ``items`` (an index, an iterable of indices or None for every slot), as
        (len(items), out_channels, delay); the slots are then reset.  The flush push repeats each slot's last frame (the
        right edge of ReplicationPad1d) with zero noise, and the end frames mask everything past the signal.  The other
        slots' state is restored around it, so they continue exactly as if it had not happened; ending one slot costs a
        ceil(delay / hop)-frame batch push (DESIGN.md §3.9)."""
        n = self._flush_frames()
        P = self.cin_hist.shape[-1]

        def inputs():
            c = self.cin_hist[:, :, P - 1:].expand(-1, -1, n).contiguous() if P else self._zeros(self.B, self.in_channels, n)
            return n, self._zeros(self.B, self.model.in_channels, n * self.hop), c

        return self._flush(list(self._slots(items)), inputs)


class _HiFiGANStream(_ChunkStream):
    """The level, block and carry tables of a streamed ``HiFiGANGenerator``, shared by the causal stream and the centred
    one with lookahead.  Both keep, per slot, one history per signal (convs that read the same tensor share a buffer sized
    by the largest of their histories):

    * the input conv: the last kernel_size - 1 mel frames; it runs on [history | chunk];
    * each conv-transpose: the last frame of its input;
    * each level's input, read by the first dilated conv of every block: max_j (delta_j + (k_j - 1) * d_j0) samples;
    * each ResBlock's later dilated-conv inputs ((k - 1) * d) and second-conv inputs (k - 1);
    * the output conv: its last kernel_size - 1 input samples.

    The convs read their histories in their loaders (pwgb_conv1d_stream_forward / pwgb_conv1d_tc_stream_forward), so no
    [history | chunk] concatenation is made at the waveform rate.  After a ResBlock's last conv one pwgb_stream_carry
    launch updates every history it read; the intermediate signals of each chunk length live in buffers allocated once,
    so the carry tables are built once too.

    A centred conv over [history | chunk] is the causal conv of the stream with its output labelled pad samples earlier,
    so the centred stream runs every signal in "delayed time", ``look`` samples (at the signal's rate) behind the frames
    pushed.  The causal stream is the case where every lookahead and every delay is zero: ``look*`` 0, ``delta`` 0 and
    ``rdelay`` 0 for every conv, and no mask."""

    def _build(self, model, centred):
        B, zeros = self.B, self._zeros
        m = model
        self.slope, self.nb = m.slope, m.num_blocks
        ic = m.input_conv if centred else m.input_conv.conv
        self.w_in = wb(ic)
        look = (ic.kernel_size[0] - 1) // 2 if centred else 0  # lookahead of the current signal, in its samples
        self.look_in = look
        self.hop = 1
        self.levels = []
        for i in range(m.num_upsamples):
            up = m.upsamples[i][1]
            deconv = up if centred else up.deconv
            cin, cout = deconv.in_channels, deconv.out_channels
            s = deconv.stride[0]
            self.hop *= s
            # the window of cat(h, x) is the centred layer's samples from a * s - padding on
            look = look * s + deconv.padding[0] if centred else 0
            look_u = look
            blocks, lvl_hist, look = self._mrf_level([m.blocks[i * self.nb + j] for j in range(self.nb)], cout, look_u, centred)
            self.levels.append(dict(stride=s, channels=cout, w=wb(deconv), up_hist=zeros(B, cin, 1), lvl_hist=lvl_hist,
                                    blocks=blocks, rate=self.hop, look_u=look_u))
        oc = m.output_conv[1] if centred else m.output_conv[1].conv
        self.w_out = wb(oc)
        K_out = oc.kernel_size[0]
        self.out_hist = zeros(B, oc.in_channels, K_out - 1)
        self.out_channels = oc.out_channels
        self.delay = look + (K_out - 1) // 2 if centred else 0

    def _mrf_level(self, blks, cout, look_u, centred):
        """The block tables of one MRF level (ResidualBlocks ``blks`` on ``cout`` channels) whose input has lookahead
        ``look_u``: returns (blocks, the level input's history, the lookahead of the MRF's output)."""
        B, zeros = self.B, self._zeros
        blocks = []
        for blk in blks:
            k, dils = blk.kernel_size, blk.dilations
            convs = []
            for idx, d in enumerate(dils):
                c1 = blk.convs1[idx][1] if centred else blk.convs1[idx][1].conv
                c2 = (blk.convs2[idx][1] if centred else blk.convs2[idx][1].conv) if blk.use_additional_convs else None
                p1 = (k - 1) * d // 2 if centred else 0
                q = p1 + ((k - 1) // 2 if c2 is not None and centred else 0)  # the branch's lag behind its input
                convs.append(dict(d=d, w1=wb(c1), w2=wb(c2) if c2 is not None else None, p1=p1, q=q,
                                  # the input of the dilated conv (idx 0: the level input, shared) and of the second conv
                                  x_hist=zeros(B, cout, (k - 1) * d) if idx > 0 else None,
                                  xt_hist=zeros(B, cout, k - 1) if c2 is not None else None))
            blocks.append(dict(k=k, convs=convs, lag=sum(cv["q"] for cv in convs)))
        # block j reads the level input delta_j samples later, so that every block ends at the same lookahead
        lag = max(b["lag"] for b in blocks)
        for b in blocks:
            b["delta"] = lag - b["lag"]
            cur = look_u + b["delta"]
            for idx, cv in enumerate(b["convs"]):
                # mask lookaheads of the dilated conv's output and of the block step's output; the residual is the
                # step's input, q (and, for the level input, delta_j) rows back
                cv["look1"], cv["look2"] = cur + cv["p1"], cur + cv["q"]
                cv["rdelay"] = cv["q"] + (b["delta"] if idx == 0 else 0)
                cur += cv["q"]
        hl = max(b["delta"] + (b["k"] - 1) * b["convs"][0]["d"] for b in blocks)
        return blocks, zeros(B, cout, hl), look_u + lag

    # ---------------------------------------------------------------------------------------------------- state
    def _histories(self):
        hs = [self.cin_hist, self.out_hist]
        for lv in self.levels:
            hs += [lv["up_hist"], lv["lvl_hist"]]
            for blk in lv["blocks"]:
                hs += [h for cv in blk["convs"] for h in (cv["x_hist"], cv["xt_hist"]) if h is not None]
        return hs

    # ---------------------------------------------------------------------------------------------------- compute
    def _mrf_buffers(self, lv, t, before, after=(), u=None):
        """The buffers of one MRF level over t samples (``u``: its input, allocated when None) and its carry tables, one
        per block; the last block's also carries ``before``, the level input and ``after``."""
        dev, B, empty = self.dev, self.B, self._empty
        C = lv["channels"]
        nd = max(len(b["convs"]) for b in lv["blocks"])
        buf = dict(u=empty(B, C, t) if u is None else u, cs=empty(B, C, t), x=[empty(B, C, t) for _ in range(nd - 1)],
                   xt=[empty(B, C, t) for _ in range(nd)])
        tables = []
        for j, blk in enumerate(lv["blocks"]):
            entries = []
            for idx, cv in enumerate(blk["convs"]):
                if cv["x_hist"] is not None:
                    entries.append((buf["x"][idx - 1], cv["x_hist"]))
                if cv["xt_hist"] is not None:
                    entries.append((buf["xt"][idx], cv["xt_hist"]))
            if j == len(lv["blocks"]) - 1:
                entries += list(before) + [(buf["u"], lv["lvl_hist"])] + list(after)
            tables.append(ops.stream_carry_table(entries, dev))
        buf["tables"] = tables
        return buf

    def _new_entry(self, n, xin):
        """The buffers of every intermediate signal of an n-frame chunk, and the carry tables over them."""
        dev, B, empty = self.dev, self.B, self._empty
        ent = dict(h0=empty(B, self.levels[0]["w"][0].shape[0], n), levels=[])
        t, prev = n, ent["h0"]
        for i, lv in enumerate(self.levels):
            t *= lv["stride"]
            # the level's shared signals are carried after their last reader; the last frames of [history | chunk] are
            # the chunk's
            buf = self._mrf_buffers(lv, t, [(prev, lv["up_hist"])], [(xin, self.cin_hist)] if i == 0 else [])
            ent["levels"].append(buf)
            prev = buf["cs"]
        ent["y"] = empty(B, self.out_channels, t)
        ent["out_table"] = ops.stream_carry_table([(prev, self.out_hist)], dev)
        return ent

    def _mask(self, rate, look):
        """the stream_ext mask of a signal with ``rate`` samples per frame and lookahead ``look`` (None: causal)"""
        return None

    def _levels(self, h, ent, replicate):
        """the conv-transposes and the MRF blocks of one chunk, from the input conv's output h"""
        slope = self.slope
        for lv, buf in zip(self.levels, ent["levels"]):
            rate = lv["rate"]
            u = ops.conv_transpose1d_stream(h, lv["up_hist"], lv["w"][0], lv["w"][1], stride=lv["stride"], replicate=replicate,
                                            pre_slope=slope, out=buf["u"], mask=self._mask(rate, lv["look_u"]))
            h = self._mrf(lv, buf, u)
        return h

    def _mrf(self, lv, buf, u):
        """The MRF blocks of one level on its input u (buf["u"]); returns their average, buf["cs"]"""
        slope, rate, t, cs = self.slope, lv["rate"], u.shape[-1], buf["cs"]
        for j, blk in enumerate(lv["blocks"]):
            k, convs = blk["k"], blk["convs"]
            x = u
            for idx, cv in enumerate(convs):
                d = cv["d"]
                last = idx == len(convs) - 1
                tail = dict(out=cs, accumulate=j > 0, out_scale=1.0 / self.nb) if last else dict(out=buf["x"][idx])
                hx = lv["lvl_hist"] if idx == 0 else cv["x_hist"]
                # block j's first conv reads the level input delta_j rows early: rows [-(P + delta_j), t - delta_j)
                P = (k - 1) * d + (blk["delta"] if idx == 0 else 0)
                res = dict(residual=x, res_hist=hx if cv["rdelay"] else None, res_delay=cv["rdelay"])
                if cv["w2"] is not None:
                    xt = ops.conv1d_stream(x, hx, *cv["w1"], pad_left=P, dilation=d, pre_slope=slope, out=buf["xt"][idx], t_out=t,
                                           mask=self._mask(rate, cv["look1"]))
                    x = ops.conv1d_stream(xt, cv["xt_hist"], *cv["w2"], pad_left=k - 1, pre_slope=slope,
                                          mask=self._mask(rate, cv["look2"]), **res, **tail)
                else:
                    x = ops.conv1d_stream(x, hx, *cv["w1"], pad_left=P, dilation=d, pre_slope=slope, t_out=t,
                                          mask=self._mask(rate, cv["look2"]), **res, **tail)
            ops.stream_carry(buf["tables"][j])
        return cs

    def _output(self, h, ent):
        y = ops.conv1d_stream(h, self.out_hist, *self.w_out, pad_left=self.out_hist.shape[-1], pre_slope=0.01, post_act="tanh",
                              out=ent["y"], mask=self._mask(self.hop, self.delay))
        ops.stream_carry(ent["out_table"])
        return y

    def _centred(self, ent, n):
        """The centred generator of a lookahead stream on the entry's xin = [history | n frames], which its front end has
        filled: the input conv, the levels and the output conv.  Advances the frame counter."""
        h = ops.conv1d_stream(ent["xin"], self._nohist, *self.w_in, pad_left=0, out=ent["h0"], mask=self._mask(1, self.look_in))
        y = self._output(self._levels(h, ent, None), ent)
        self.frame += n
        return y


class CausalHiFiGANStream(_HiFiGANStream):
    """Streams a causal ``HiFiGANGenerator`` (``use_causal_conv=True``) chunk by chunk for ``batch`` independent slots.

    ``push(c)`` takes the next n >= 1 mel frames of every slot and returns their n * hop samples; n may change from push
    to push.  For every slot, the concatenated outputs equal ``model.inference(all_frames)``.  There is no lookahead and
    no flush.  Every conv of the causal generator pads only on the left, so the histories of ``_HiFiGANStream`` hold
    exactly what the whole-utterance forward reads in front of the chunk: zeros for a fresh slot, except that each
    conv-transpose's history replicates its first frame (``ReplicationPad1d``, pwgb_conv_transpose1d_stream_forward with
    the per-slot replicate flags).  With ``use_graphs`` each chunk length is captured once into a CUDA graph and replayed.
    The weights are read when the stream is built and must not change while it is used."""

    def __init__(self, model, batch=1, use_graphs=True):
        from .models import HiFiGANGenerator

        if not isinstance(model, HiFiGANGenerator):
            raise PwgbError("CausalHiFiGANStream: expected a HiFiGANGenerator")
        if not model.use_causal_conv:
            raise PwgbError("CausalHiFiGANStream: the model is not causal (use_causal_conv=False); a centred model needs lookahead")
        ic = model.input_conv
        # the fresh slots' flags are the conv-transposes' replicate flags
        self._setup(model, batch, use_graphs, ic.conv.in_channels, ic.left, "zero", flags=True)
        self._build(model, centred=False)

    def _state(self):
        return self._histories()

    def _step(self, c):
        """One chunk: c (B, in_channels, n) -> (B, out_channels, n * hop).  Advances the state."""
        ent = self._entry(c.shape[-1])
        h = ops.conv1d(self._input(ent, c), *self.w_in, out=ent["h0"])
        y = self._output(self._levels(h, ent, self.fresh), ent)
        self.fresh.zero_()
        return y

    @torch.no_grad()
    def push(self, c, normalize_before=False):
        """c: (B, n, in_channels) mel frames ((n, in_channels) when batch == 1).  Returns (B, out_channels, n * hop) on the
        device."""
        c = self._frames(c, normalize_before)
        self._start(c)
        return self._run(c.shape[-1], c)


class HiFiGANLookaheadStream(_Lookahead, _HiFiGANStream):
    """Streams a centred ``HiFiGANGenerator`` (``use_causal_conv=False``, the published checkpoints) chunk by chunk for
    ``batch`` independent slots, with a fixed lookahead of ``delay`` output samples.

    ``push(c)`` takes the next n >= 1 mel frames of every slot and returns n * hop samples: the whole-utterance samples
    from t0 * hop - delay on (t0: the frames pushed before), with zeros before sample 0.  ``flush(items)`` returns the
    last ``delay`` samples of those slots and restarts them; the other slots continue as if no flush had happened.  For
    every slot, the concatenated pushes and flush equal ``[zeros(delay) | model.inference(all_frames)]``.

    ``delay`` is the sum of the centred paddings along the generator (DESIGN.md §3.8), derived from the module: 3258
    samples (12.7 frames) for HiFi-GAN v1.  Each signal runs in delayed time behind the frames pushed; every conv is the
    causal stream's history conv on [history | chunk], and:

    * every launch masks the samples outside its signal to +0.0 (pwgb_stream_ext: a device frame counter per slot,
      advanced inside the captured push, and an end frame set by the flush), which is the zero padding the
      whole-utterance forward reads there;
    * a ResBlock step x + branch(x) adds its input q samples back (q: the branch's lag), read from the step's history;
    * block j of a level reads the level input delta_j samples later, so that every block ends at the same lookahead and
      the MRF sum accumulates as in ``inference``;
    * the conv-transposes' one-frame histories are zero for a fresh slot (no replication);
    * the flush pushes ceil(delay / hop) zero frames with the slots' end frames set: the mask gives every layer its right
      zero padding, so it is one more push through a cached entry.

    With ``use_graphs`` each chunk length is captured once into a CUDA graph and replayed.  The weights are read when the
    stream is built and must not change while it is used."""

    def __init__(self, model, batch=1, use_graphs=True):
        from .models import HiFiGANGenerator

        if not isinstance(model, HiFiGANGenerator):
            raise PwgbError("HiFiGANLookaheadStream: expected a HiFiGANGenerator")
        if model.use_causal_conv:
            raise PwgbError("HiFiGANLookaheadStream: the model is causal (use_causal_conv=True); stream it with CausalHiFiGANStream, "
                            "which has no lookahead")
        ic = model.input_conv
        self._setup(model, batch, use_graphs, ic.in_channels, ic.kernel_size[0] - 1, "zero")
        self._build(model, centred=True)
        self._counters()

    def _state(self):
        return self._histories() + [self.frame, self.end]

    def _step(self, c):
        """One chunk: c (B, in_channels, n) -> (B, out_channels, n * hop).  Advances the state."""
        n = c.shape[-1]
        ent = self._entry(n)
        # the centred input conv reads [history | chunk]: frames t0 - 3 .. t0 + n - 4 for kernel 7
        self._input(ent, c)
        return self._centred(ent, n)

    @torch.no_grad()
    def push(self, c, normalize_before=False):
        """c: (B, n, in_channels) mel frames ((n, in_channels) when batch == 1).  Returns (B, out_channels, n * hop) on the
        device: samples [t0 * hop - delay, (t0 + n) * hop - delay) of each slot's utterance."""
        c = self._frames(c, normalize_before)
        self._start(c)
        return self._run(c.shape[-1], c)

    @torch.no_grad()
    def flush(self, items=None):
        """The last ``delay`` samples of slots ``items`` (an index, an iterable of indices or None for every slot), computed
        against the zero right padding, as (len(items), out_channels, delay); the slots are then reset.  The other slots'
        state is restored around the flush push, so they continue exactly as if it had not happened.  The flush push covers
        every slot, so ending one slot costs a ceil(delay / hop)-frame batch push (DESIGN.md §3.8)."""
        n = self._flush_frames()
        return self._flush(list(self._slots(items)), lambda: (n, self._zeros(self.B, self.in_channels, n)))


def _check_dsym_levels(name, model):
    for i, up in enumerate(model.upsamples):
        k, s = up[1].kernel_size[0], up[1].stride[0]
        if k != 2 * s or s % 2:
            raise PwgbError(f"{name}: upsampling level {i} has kernel {k} and stride {s}; the stream needs kernel 2 * stride "
                            "and an even stride (padding (k - s) // 2 makes the whole utterance T * s + 1 samples long otherwise)")


class DiscreteSymbolHiFiGANLookaheadStream(_Lookahead, _HiFiGANStream):
    """Streams a ``DiscreteSymbolHiFiGANGenerator`` (HuBERT units in, audio out; the vctk / cvss_c ``hubert_voc1``
    recipes without durations) chunk by chunk for ``batch`` independent slots, with a fixed lookahead of ``delay`` output
    samples.

    ``push(c)`` takes the next n >= 1 frames of every slot: (B, n, 2) (symbol, speaker) indices when the model has
    speakers, else (B, n) or (B, n, 1); int64 or float32 (read as torch's ``c.long()``, NaN as an index outside the table).
    It returns (B, out_channels, n * hop): the whole-utterance samples [t0 * hop - delay, (t0 + n) * hop - delay).
    ``flush(items)`` returns the last ``delay`` samples of those slots and restarts them; the other slots continue as if
    no flush had happened.  For every slot, the concatenated pushes and flush equal ``[zeros(delay) |
    model.inference(all_frames)]``.

    The body after input_conv is ``HiFiGANLookaheadStream``'s (DESIGN.md §3.8, §3.13).  The front end is one launch,
    pwgb_symbol_embed_stream_forward, which writes the chunk's embedding into the input conv's [history | chunk] buffer
    with the fp32 expression of the whole-utterance embed and stores +0.0 at frames past a flushed slot's end.  The
    whole-utterance forward adds the speaker of an item's first frame to every frame, so each slot latches the speaker
    of its first pushed frame on the device, inside the captured push, and a reset unlatches it.  Index and speaker
    values outside their tables give NaN columns, as in the whole utterance.

    ``delay`` comes from the module: 3482 samples (10.9 frames) for the 16 kHz recipes' scales (10, 8, 2, 2) and 4526 for
    the 24 kHz ones (12, 10, 2, 2).  With ``use_graphs`` each chunk length (and index dtype) is captured once into a CUDA
    graph and replayed.  The weights are read when the stream is built and must not change while it is used."""

    def __init__(self, model, batch=1, use_graphs=True):
        from .models import DiscreteSymbolHiFiGANGenerator

        name = "DiscreteSymbolHiFiGANLookaheadStream"
        if type(model) is not DiscreteSymbolHiFiGANGenerator:
            raise PwgbError(f"{name}: expected a DiscreteSymbolHiFiGANGenerator, got {type(model).__name__}")
        self.use_spk = model.num_spk_embs > 0
        if self.use_spk and model.concat_spk_emb:
            raise PwgbError(f"{name}: concat_spk_emb=True is not supported (the model's forward fails on it too)")
        _check_dsym_levels(name, model)
        ic = model.input_conv
        self._setup(model, batch, use_graphs, ic.in_channels, ic.kernel_size[0] - 1, "zero", flags=self.use_spk)
        self._build(model, centred=True)
        self._counters()
        self.table = model.emb.weight.detach()
        self.spk_table = model.spk_emb.weight.detach() if self.use_spk else None
        # each slot's latched speaker row (-2: outside the speaker table); valid while the slot's fresh flag is clear
        self.latch = torch.zeros(self.B, device=self.dev, dtype=torch.int32) if self.use_spk else None
        self._by_dtype = {}  # index dtype -> its chunk-length entries (a captured graph reads its own index buffer)

    def _state(self):
        return self._histories() + [self.frame, self.end] + ([self.latch] if self.use_spk else [])

    def _step(self, c):
        """One chunk: c (B, K, n) indices -> (B, out_channels, n * hop).  Advances the state."""
        n = c.shape[-1]
        ent = self._entry(n)
        xin = ent["xin"]
        P = self.cin_hist.shape[-1]
        xin[:, :, :P].copy_(self.cin_hist)
        ops.symbol_embed_stream(c, self.table, self.spk_table, self.latch, self.fresh, self._mask(1, 0), xin, P)
        if self.use_spk:
            self.fresh.zero_()
        return self._centred(ent, n)

    def _ids(self, c):
        """(B, n[, K]) indices -> (B, K, n) contiguous on the device, int64 or float32"""
        c = torch.as_tensor(c, device=self.dev)
        if c.dtype not in (torch.float32, torch.int64):
            c = c.long()
        K = 2 if self.use_spk else 1
        if c.dim() == 2 and not self.use_spk:
            c = c.unsqueeze(-1)
        if c.dim() != 3 or c.shape[0] != self.B or c.shape[1] < 1 or c.shape[2] != K:
            want = f"({self.B}, n >= 1, 2)" if self.use_spk else f"({self.B}, n >= 1) or ({self.B}, n >= 1, 1)"
            raise PwgbError(f"DiscreteSymbolHiFiGANLookaheadStream.push: c must be {want}, got {tuple(c.shape)}")
        return c.transpose(1, 2).contiguous()

    def _run(self, n, c):
        self._entries = self._by_dtype.setdefault(c.dtype, {})
        return super()._run(n, c)

    @torch.no_grad()
    def push(self, c):
        """c: (B, n, 2) (symbol, speaker) indices, or (B, n) / (B, n, 1) symbols for a model without speakers.  Returns
        (B, out_channels, n * hop) on the device: samples [t0 * hop - delay, (t0 + n) * hop - delay) of each slot's
        utterance."""
        self._check_eval(self.model)
        c = self._ids(c)
        return self._run(c.shape[-1], c)

    @torch.no_grad()
    def flush(self, items=None):
        """The last ``delay`` samples of slots ``items`` (an index, an iterable of indices or None for every slot), computed
        against the zero right padding, as (len(items), out_channels, delay); the slots are then reset.  The flush push
        covers every slot with symbol 0 (the end mask stores the flushed slots' frames as +0.0); the other slots' state,
        speaker latch and fresh flag included, is restored around it."""
        n = self._flush_frames()
        ids = torch.zeros((self.B, 2 if self.use_spk else 1, n), device=self.dev, dtype=torch.int64)
        return self._flush(list(self._slots(items)), lambda: (n, ids))


class DiscreteSymbolDurationLookaheadStream(_Lookahead, _HiFiGANStream):
    """Streams a ``DiscreteSymbolDurationGenerator`` without speakers (the cvss_c ``hubert_voc1`` recipe: deduplicated
    HuBERT units in, audio out, durations predicted as the units arrive) for ``batch`` independent slots.

    ``push(c)`` takes the next m >= 1 symbols of every slot, (B, m) int64 or float32 (the deduplicated units ``synthesis``
    takes), and returns (B, out_channels, n * hop): the next n frames' samples of every slot, n being the fewest frames
    any slot has queued (all slots share one frame clock; a slot with more keeps them queued).  ``flush(items)`` ends
    those slots one at a time and returns a list of their remaining samples, (out_channels, L_b) each; the other slots
    continue as if no flush had happened.  For every slot, the concatenated pushes and flush equal ``[zeros(delay) |
    model.inference(all_symbols)]``, and the durations finalised by the pushes and the flush (``last_durations`` after
    each) equal ``synthesis``'s before its all-zero rule.

    One push runs four stages (DESIGN.md §3.13):

    * the duration predictor at symbol rate, in delayed time P = n_layers * (k - 1) / 2 symbols behind the symbols pushed:
      the symbol embedding (pwgb_symbol_embed_stream_forward, +0.0 past the end) and each conv on [history | chunk]
      (masked, ReLU epilogue), each LayerNorm masked to +0.0 outside the signal (LayerNorm of a zero column is beta, the
      next conv's padding is zero), the Linear as the whole utterance runs it;
    * the final symbols' durations, rounded as pwgb_duration_round rounds them, appended with their ids to a per-slot
      device queue (pwgb_duration_queue_append), which also keeps the queued frame count and the running total;
    * one device-to-host read of the B queued counts (the whole utterance synchronises at the same point), then the body
      advances every slot by n frames in power-of-two pushes (at most log2 captured lengths), each filling the input
      conv's [history | chunk] buffer from the queues (pwgb_symbol_regulate_stream_forward); a symbol's run may start in
      one push and end in a later one;
    * the body is ``HiFiGANLookaheadStream``'s, ``delay`` samples behind.

    The flush of a slot sets its symbol end, pushes P masked symbols, applies the all-zero rule if the slot's total is
    still 0 (its queued symbols, all kept, get duration 1), drains its queue through the body and runs the body's flush.
    A slot that never produces frames stalls the others; ``max_queue`` bounds each slot's queue, and a push that would
    overflow it raises.  The weights are read when the stream is built and must not change while it is used."""

    def __init__(self, model, batch=1, use_graphs=True, max_queue=4096):
        from .models import DiscreteSymbolDurationGenerator

        name = "DiscreteSymbolDurationLookaheadStream"
        if type(model) is not DiscreteSymbolDurationGenerator:
            raise PwgbError(f"{name}: expected a DiscreteSymbolDurationGenerator, got {type(model).__name__}")
        if model.num_spk_embs > 0:
            raise PwgbError(f"{name}: a duration model with speakers is not supported (its forward fails too: the predictor "
                            "is built for in_channels + spk_emb_dim inputs)")
        _check_dsym_levels(name, model)
        ic = model.input_conv
        self._setup(model, batch, use_graphs, ic.in_channels, ic.kernel_size[0] - 1, "zero")
        self._build(model, centred=True)
        self._counters()
        self.table = model.emb.weight.detach()
        dp = model.duration_predictor
        self.offset = float(dp.offset)
        self.pred = []
        for f in dp.conv:
            conv, ln = f[0], f[2]
            if conv.kernel_size[0] % 2 == 0:
                raise PwgbError(f"{name}: the duration predictor's kernel must be odd")
            self.pred.append(dict(w=wb(conv), k=conv.kernel_size[0], ln=(ln.weight.detach(), ln.bias.detach(), float(ln.eps)),
                                  hist=self._zeros(self.B, conv.in_channels, conv.kernel_size[0] - 1)))
        self.P = sum((L["k"] - 1) // 2 for L in self.pred)
        lin = dp.linear
        self.w_lin = (lin.weight.detach().reshape(1, lin.in_features, 1).contiguous(), lin.bias.detach())
        self.sframe = torch.zeros(self.B, device=self.dev, dtype=torch.int32)
        self.send = torch.full((self.B,), self.OPEN, device=self.dev, dtype=torch.int32)
        self.id_hist = torch.zeros((self.B, self.P), device=self.dev, dtype=torch.int64)
        self.max_queue = int(max_queue)
        self.queue = ops.DurationQueue(self.B, self.max_queue, self.dev)
        self._last, self._last_flush = None, None
        self._len = {}

    def _state(self):
        return (self._histories() + [self.frame, self.end, self.sframe, self.send, self.id_hist] + [L["hist"] for L in self.pred]
                + self.queue.tensors())

    def reset(self, items=None):
        super().reset(items)
        for b in self._slots(items):
            self.send[b] = self.OPEN

    # ---------------------------------------------------------------------------------------------------- predictor
    def _predict(self, ids):
        """The predictor on m symbols ids (B, 1, m) int64 of every slot; appends the final symbols to the queues and keeps
        their durations (B, m) (-1: not final) in ``_last``."""
        m = ids.shape[-1]
        smask = lambda look: (self.sframe, self.send, 1, look)  # noqa: E731
        x = self._empty(self.B, self.table.shape[1], m)
        ops.symbol_embed_stream(ids, self.table, None, None, None, smask(0), x, 0)
        look = 0
        for L in self.pred:
            k, hist = L["k"], L["hist"]
            look += (k - 1) // 2
            y = ops.conv1d_stream(x, hist, *L["w"], pad_left=k - 1, post_act="lrelu", post_slope=0.0, mask=smask(look))
            hist.copy_(torch.cat([hist, x], -1)[:, :, -(k - 1):] if k > 1 else hist)
            x = ops.stream_mask(ops.channel_layer_norm(y, *L["ln"]), smask(look))
        logd = ops.conv1d_raw(x, *self.w_lin).reshape(self.B, m)
        idw = torch.cat([self.id_hist, ids[:, 0]], -1)  # column j: symbol sframe - P + j
        if self.P:
            self.id_hist.copy_(idw[:, -self.P:])
        self._last, self._last_flush = torch.empty((self.B, m), device=self.dev, dtype=torch.int64), None
        ops.duration_queue_append(self.queue, logd, idw, smask(self.P), self.P, self.offset, dur_out=self._last)
        self.sframe += m

    def _queued(self, slots=None):
        """the queued frame counts on the host (one device-to-host read); raises on an overflowed queue"""
        q = self.queue.counts.cpu()
        over = [b for b in (range(self.B) if slots is None else slots) if q[b, 1]]
        if over:
            raise PwgbError(f"DiscreteSymbolDurationLookaheadStream: the queue of slot(s) {over} overflowed max_queue = {self.max_queue} "
                            "symbols (a slot stalls while another makes no frames); build the stream with a larger max_queue and "
                            "reset those slots")
        return q[:, 0]

    @property
    def last_durations(self):
        """the durations finalised by the last push or flush, one int64 tensor per slot (a list: slots finalise different
        counts while their first P symbols are in flight)"""
        if self._last_flush is not None:
            return self._last_flush
        if self._last is None:
            return [torch.zeros(0, dtype=torch.int64) for _ in range(self.B)]
        d = self._last.cpu()
        return [row[row >= 0] for row in d]

    # ---------------------------------------------------------------------------------------------------- body
    def _step(self, tn):
        """n frames of every slot's queue (n: tn's length) -> (B, out_channels, n * hop).  Advances the state."""
        n = tn.shape[0]
        ent = self._entry(n)
        xin = ent["xin"]
        P = self.cin_hist.shape[-1]
        xin[:, :, :P].copy_(self.cin_hist)
        ops.symbol_regulate_stream(self.table, self.queue, self._mask(1, 0), xin, P, n)
        return self._centred(ent, n)

    def _body(self, n):
        """n frames in power-of-two pushes, largest first"""
        ys = []
        p = 1 << max(int(n).bit_length() - 1, 0)
        while n > 0:
            if p <= n:
                if p not in self._len:
                    self._len[p] = torch.empty(p, device=self.dev)
                ys.append(self._run(p, self._len[p]))
                n -= p
            p >>= 1
        return torch.cat(ys, -1) if ys else self._zeros(self.B, self.out_channels, 0)

    @torch.no_grad()
    def push(self, c):
        """c: (B, m) symbols (or (B, m, 1)).  Returns (B, out_channels, n * hop) on the device (n may be 0)."""
        self._check_eval(self.model)
        c = torch.as_tensor(c, device=self.dev)
        if c.dim() == 3 and c.shape[-1] == 1:
            c = c[..., 0]
        if c.dim() != 2 or c.shape[0] != self.B or c.shape[1] < 1:
            raise PwgbError(f"DiscreteSymbolDurationLookaheadStream.push: c must be ({self.B}, m >= 1) symbols, got {tuple(c.shape)}")
        if c.dtype not in (torch.float32, torch.int64):
            c = c.long()
        self._predict(c.unsqueeze(1).contiguous())
        return self._body(int(self._queued().min()))

    @torch.no_grad()
    def flush(self, items=None):
        """The remaining samples of slots ``items`` (an index, an iterable of indices or None for every slot), as a list of
        (out_channels, L_b) tensors; the slots are then reset.  Each slot is flushed alone, with the other slots' state
        restored around it; ``last_durations`` then holds the durations the flush finalised."""
        items = list(self._slots(items))
        outs, last = [], [torch.zeros(0, dtype=torch.int64) for _ in range(self.B)]
        n = self._flush_frames()
        for b in items:
            with self._keeping_others([b]):
                self.send[b] = self.sframe[b]
                if self.P:
                    self._predict(torch.zeros((self.B, 1, self.P), device=self.dev, dtype=torch.int64))
                    last[b] = self.last_durations[b]
                zr = torch.zeros(self.B, device=self.dev, dtype=torch.int32)
                zr[b] = 1
                ops.duration_queue_append(self.queue, None, None, (self.frame, self.end), 0, self.offset, zero_rule=zr)
                ys = [self._body(int(self._queued([b])[b]))]
                self.end[b] = self.frame[b]
                if n not in self._len:
                    self._len[n] = torch.empty(n, device=self.dev)
                ys.append(self._run(n, self._len[n])[:, :, :self.delay])
                outs.append(torch.cat(ys, -1)[b])
            self.reset(b)
        self._last_flush = last
        return outs


class _MelGANStream(_ChunkStream):
    """The levels, stacks, histories and carry table of a streamed ``MelGANGenerator`` (full-band, or multi-band with
    ``model.pqmf``), shared by the causal stream and the centred one with lookahead.  Both keep, per slot, one history
    per signal:

    * the input conv: the last kernel_size - 1 mel frames; it runs on [history | chunk];
    * each conv-transpose: the last frame of its input;
    * each ResidualStack: its last (k - 1) * d input samples (the two 1x1 convs need none of their own);
    * the output conv: its last kernel_size - 1 input samples;
    * with PQMF: the last ceil((taps + 1) / subbands) - 1 subband samples of the synthesis input.

    The dilated convs read their histories in their loaders (pwgb_conv1d_stream_forward / pwgb_conv1d_tc_stream_forward),
    and one pwgb_stream_carry launch at the end of a push updates every history."""

    def _build(self, model, centred):
        from .layers import CausalConv1d, CausalConvTranspose1d, ResidualStack

        B, zeros = self.B, self._zeros
        self.slope = model.slope
        mods = list(model.melgan)
        convs = [m for m in mods if isinstance(m, torch.nn.Conv1d if centred else CausalConv1d)]
        ic, oc = convs[0], convs[-1]
        self.w_in = wb(ic if centred else ic.conv)
        self.hop, self.levels = 1, []
        for m in mods[1:]:
            if isinstance(m, torch.nn.ConvTranspose1d if centred else CausalConvTranspose1d):
                if not centred and not isinstance(m.pad, torch.nn.ReplicationPad1d):
                    raise PwgbError("CausalMelGANStream: only the ReplicationPad1d conv-transpose of MelGANGenerator is supported")
                deconv = m if centred else m.deconv
                self.hop *= deconv.stride[0]
                self.levels.append(dict(stride=deconv.stride[0], channels=deconv.out_channels, w=wb(deconv),
                                        up_hist=zeros(B, deconv.in_channels, 1), rate=self.hop, stacks=[]))
            elif isinstance(m, ResidualStack):
                k, d = m.kernel_size, m.dilation
                C = m.skip_layer.in_channels
                c1, c2 = (m.stack[2], m.stack[4]) if centred else (m.stack[1].conv, m.stack[3])
                self.levels[-1]["stacks"].append(dict(k=k, d=d, w1=wb(c1), w2=wb(c2), ws=wb(m.skip_layer), hist=zeros(B, C, (k - 1) * d)))
        oconv = oc if centred else oc.conv
        self.w_out = wb(oconv)
        self.out_hist = zeros(B, oconv.in_channels, oconv.kernel_size[0] - 1)
        self.out_channels = oconv.out_channels
        self.post_act = "tanh" if model.use_final_nonlinear_activation else None
        pq = model.pqmf
        if pq is not None:
            N = pq.subbands
            if self.out_channels != N:
                raise PwgbError(f"{type(self).__name__}: {self.out_channels} output channels for a {N}-band PQMF")
            # PQMF.synthesis's transposed FIR, computed as there; its window lags its input by taps // 2 samples
            self.w_syn = (pq.synthesis_filter[0].flip(-1) * float(N)).unsqueeze(1).contiguous()
            self.subbands, self.pq_pad = N, pq.taps // 2
            self.pq_hist = zeros(B, N, -(-(pq.taps + 1) // N) - 1)
        else:
            self.subbands, self.pq_hist = 1, None

    # ---------------------------------------------------------------------------------------------------- state
    def _histories(self):
        hs = [self.cin_hist, self.out_hist]
        for lv in self.levels:
            hs += [lv["up_hist"]] + [st["hist"] for st in lv["stacks"]]
        return hs + ([self.pq_hist] if self.pq_hist is not None else [])

    # ---------------------------------------------------------------------------------------------------- compute
    def _new_entry(self, n, xin):
        """The buffers of every intermediate signal of an n-frame chunk, and the carry table over them."""
        dev, B, empty = self.dev, self.B, self._empty
        ent = dict(h0=empty(B, self.levels[0]["w"][0].shape[0], n), levels=[])
        entries = [(xin, self.cin_hist)]
        t, prev = n, ent["h0"]
        for lv in self.levels:
            t *= lv["stride"]
            C = lv["channels"]
            buf = dict(u=empty(B, C, t), h=empty(B, C, t), s=empty(B, C, t), x=[empty(B, C, t) for _ in lv["stacks"]])
            entries.append((prev, lv["up_hist"]))
            x = buf["u"]
            for j, st in enumerate(lv["stacks"]):
                entries.append((x, st["hist"]))
                x = buf["x"][j]
            ent["levels"].append(buf)
            prev = x
        entries.append((prev, self.out_hist))
        ent["y"] = empty(B, self.out_channels, t)
        if self.pq_hist is not None:
            entries.append((ent["y"], self.pq_hist))
            ent["wave"] = empty(B, 1, t * self.subbands)
        # every history is read before this one carry, at the end of the push
        ent["table"] = ops.stream_carry_table(entries, dev)
        return ent


class CausalMelGANStream(_MelGANStream):
    """Streams a causal ``MelGANGenerator`` (``use_causal_conv=True``), full-band or multi-band with ``model.pqmf``, chunk
    by chunk for ``batch`` independent slots.

    ``push(c)`` takes the next n mel frames of every slot and returns their n * hop * subbands samples; n may change from
    push to push.  ``flush(items)`` returns the ``delay`` samples the slots still hold and restarts them.  For every slot,
    the concatenated pushes and flush equal ``[zeros(delay) | model.inference(all_frames)]``.  Without PQMF ``delay`` is
    0; with it the centred synthesis filter reads ``taps // 2`` samples ahead, so the stream lags by that many samples
    and the flush computes the tail against the zero right padding.

    Every conv pads only on the left, with the model's pad (reflect, replicate or zero ``ConstantPad1d``).  A reflected
    row -t is sample t of the same signal, so the first push after a reset must hold every such sample:
    ``min_first_frames`` frames (7 for the recipes' kernel-7 input conv; 1 for the other pads).  The stream keeps, per
    slot, one history per signal:

    * the input conv: the last kernel_size - 1 mel frames; a fresh slot starts from what the pad would read (frames
      P .. 1 for reflect, frame 0 repeated for replicate, zeros); it runs as a valid conv on [history | chunk];
    * each conv-transpose: the last frame of its input, replicated from the first frame for a fresh slot;
    * each ResidualStack: its last (k - 1) * d input samples (the two 1x1 convs need none); with replicate padding a
      chunk shorter than that first sets a fresh slot's history to its first sample, since the carry keeps those rows;
    * the output conv: its last kernel_size - 1 input samples;
    * with PQMF: the last ceil((taps + 1) / subbands) - 1 subband samples of the synthesis input.

    The dilated convs read their histories in their loaders (pwgb_conv1d_stream_forward / pwgb_conv1d_tc_stream_forward),
    reflecting or replicating for the slots whose fresh flag is set; the synthesis is a window of the conv-transpose
    (pwgb_conv_transpose1d_window_stream_forward) that writes zeros before sample 0 of a fresh slot.  One
    pwgb_stream_carry launch per push updates every history, and the fresh flags are cleared inside the same captured
    work.  With ``use_graphs`` each chunk length is captured once into a CUDA graph and replayed.  The weights are read
    when the stream is built and must not change while it is used."""

    def __init__(self, model, batch=1, use_graphs=True):
        from .layers import CausalConv1d
        from .models import MelGANGenerator

        if not isinstance(model, MelGANGenerator):
            raise PwgbError("CausalMelGANStream: expected a MelGANGenerator")
        mods = list(model.melgan)
        if not isinstance(mods[0], CausalConv1d):
            raise PwgbError("CausalMelGANStream: the model is not causal (use_causal_conv=False); a centred model needs lookahead")
        ic = mods[0]
        self._setup(model, batch, use_graphs, ic.conv.in_channels, ic.left, model.pad_mode, flags=True)
        self._build(model, centred=False)
        # (left padding, input samples per frame) of every conv the pad applies to
        reflect_need = [(ic.left, 1)] + [((st["k"] - 1) * st["d"], lv["rate"]) for lv in self.levels for st in lv["stacks"]]
        reflect_need.append((self.out_hist.shape[-1], self.hop))
        # the smallest first push after a reset for which every reflected row lies inside the chunk
        self.min_first_frames = max(P // rate + 1 for P, rate in reflect_need) if self.pad == "reflect" else 1
        if self.pq_hist is not None:
            self.delay = self.pq_pad
            # a fresh slot's first window also holds the delay's zeros before sample 0
            self.min_first_frames = max(self.min_first_frames, -(-self.delay // (self.hop * self.subbands)))
        else:
            self.delay = 0

    def _state(self):
        return self._histories()

    # ---------------------------------------------------------------------------------------------------- compute
    def _pad_kw(self, P, rate, n):
        """the history policy of a conv with left padding P over an input of ``rate`` samples per frame"""
        if self.pad == "replicate":
            return dict(replicate=self.fresh)
        if self.pad == "reflect" and P < n * rate:
            # a chunk too short to reflect in never holds a fresh slot (push refuses it)
            return dict(replicate=self.fresh, reflect=True)
        return {}

    def _step(self, c):
        """One chunk: c (B, in_channels, n) -> (B, 1, n * hop * subbands).  Advances the state."""
        n = c.shape[-1]
        ent = self._entry(n)
        h = ops.conv1d(self._input(ent, c), *self.w_in, out=ent["h0"])
        slope = self.slope
        for lv, buf in zip(self.levels, ent["levels"]):
            x = ops.conv_transpose1d_stream(h, lv["up_hist"], lv["w"][0], lv["w"][1], stride=lv["stride"], replicate=self.fresh,
                                            pre_slope=slope, out=buf["u"])
            for j, st in enumerate(lv["stacks"]):
                P = (st["k"] - 1) * st["d"]
                if self.pad == "replicate" and n * lv["rate"] < P:
                    # the carry keeps rows in front of a chunk shorter than the history: a fresh slot's must be its pad
                    torch.where(self.fresh.bool()[:, None, None], x[:, :, :1], st["hist"], out=st["hist"])
                hh = ops.conv1d_stream(x, st["hist"], *st["w1"], pad_left=P, dilation=st["d"], pre_slope=slope, out=buf["h"],
                                       **self._pad_kw(P, lv["rate"], n))
                s = ops.conv1d(x, *st["ws"], out=buf["s"])
                x = ops.conv1d(hh, *st["w2"], pre_slope=slope, residual=s, out=buf["x"][j])
            h = x
        P = self.out_hist.shape[-1]
        y = ops.conv1d_stream(h, self.out_hist, *self.w_out, pad_left=P, pre_slope=slope, post_act=self.post_act, out=ent["y"],
                              **self._pad_kw(P, self.hop, n))
        if self.pq_hist is not None:
            y = ops.conv_transpose1d_window_stream(y, self.pq_hist, self.w_syn, None, stride=self.subbands, padding=self.delay,
                                                   fresh=self.fresh, out=ent["wave"])
        ops.stream_carry(ent["table"])
        self.fresh.zero_()
        return y

    @torch.no_grad()
    def push(self, c, normalize_before=False):
        """c: (B, n, in_channels) mel frames ((n, in_channels) when batch == 1); n >= ``min_first_frames`` for a slot's
        first push after a reset.  Returns (B, 1, n * hop * subbands) on the device."""
        c = self._frames(c, normalize_before)
        n = c.shape[-1]
        fresh = [b for b in range(self.B) if self._fresh[b]]
        if fresh and n < self.min_first_frames:
            raise PwgbError(f"CausalMelGANStream.push: the first push after a reset needs at least {self.min_first_frames} frames "
                            f"(the reflect padding reads that far into the signal), got {n} for slots {fresh}")
        self._start(c)
        return self._run(n, c)

    @torch.no_grad()
    def flush(self, items=None):
        """The last ``delay`` samples of slots ``items`` (an index, an iterable of indices or None for every slot), computed
        against the zero right padding, as (len(items), 1, delay); the slots are then reset."""
        items = self._slots(items)
        if self.pq_hist is None:
            y = torch.zeros((len(items), 1, 0), device=self.dev, dtype=torch.float32)
        else:
            rows = -(-self.delay // self.subbands)
            y = ops.conv_transpose1d_window_stream(None, self.pq_hist, self.w_syn, None, stride=self.subbands, padding=self.delay,
                                                   fresh=self.fresh, flush_rows=rows)
            y = y[list(items), :, :self.delay].contiguous()
        self.reset(items)
        return y


class MelGANLookaheadStream(_Lookahead, _MelGANStream):
    """Streams a centred ``MelGANGenerator`` (``use_causal_conv=False``, the published checkpoints), full-band or
    multi-band with ``model.pqmf``, chunk by chunk for ``batch`` independent slots, with a fixed lookahead of ``delay``
    output samples.

    ``push(c)`` takes the next n >= 1 mel frames of every slot and returns n * hop * subbands samples: the whole-utterance
    samples from t0 * hop * subbands - delay on (t0: the frames pushed before), with zeros before sample 0.
    ``flush(items)`` returns the last ``delay`` samples of those slots and restarts them; the other slots continue as if
    no flush had happened.  For every slot, the concatenated pushes and flush equal ``[zeros(delay) |
    model.inference(all_frames)]``.

    Each signal runs in delayed time behind the frames pushed, as in ``HiFiGANLookaheadStream`` (DESIGN.md §3.10,
    oracle/ref_melgan_lookahead_stream.py): every conv is a history conv on [history | chunk] whose output is labelled
    its padding earlier, and every launch masks the samples outside its signal to +0.0 (pwgb_stream_ext), the zero padding
    the conv-transposes and the PQMF synthesis read.  The model's pad (reflect, replicate or zero ``ConstantPad1d``) sits
    at both ends of every signal a ResidualStack, the input conv or the output conv reads; those convs take the stream
    edge policy instead (pwgb_stream_ext.edge): an input row outside the signal reads the row of [history | chunk] that
    holds its reflected or replicated sample, which for every output inside the signal is in the window.  The lookaheads:
    (K - 1) / 2 frames after the input conv; s * look + s // 2 + s % 2 after a conv-transpose; + (k - 1) / 2 * d after a
    ResidualStack, whose 1x1 skip reads the stack input that many rows back from the stack's history; + (K - 1) / 2 after
    the output conv; with PQMF ``delay`` = subbands * look + taps // 2.  1425 samples for MelGAN v1, 2719 for multi-band
    MelGAN v2 ([8, 4, 2]).

    ``ReflectionPad1d`` needs its padding below the signal's length, so ``inference`` needs ``min_frames`` frames (4 for
    the recipes' [8, 8, 2, 2] and [8, 4, 2] models, 6 for [5, 5, 3]; 1 for the other pads), and ``flush`` refuses a slot
    with fewer.  With ``use_graphs`` each chunk length is captured once into a CUDA graph and replayed.  The weights are
    read when the stream is built and must not change while it is used."""

    def __init__(self, model, batch=1, use_graphs=True):
        from .layers import CausalConv1d
        from .models import MelGANGenerator

        if not isinstance(model, MelGANGenerator):
            raise PwgbError("MelGANLookaheadStream: expected a MelGANGenerator")
        mods = list(model.melgan)
        if isinstance(mods[0], CausalConv1d):
            raise PwgbError("MelGANLookaheadStream: the model is causal (use_causal_conv=True); stream it with CausalMelGANStream, "
                            "which has no lookahead")
        ic = mods[1]
        # a fresh slot's input-conv history stays zero: those frames lie before the signal, where the edge policy reads
        self._setup(model, batch, use_graphs, ic.in_channels, ic.kernel_size[0] - 1, "zero")
        self._plan(model)
        self._counters()
        self._count = [0] * self.B  # frames pushed per slot, on the host

    # the frames the generator's input runs behind the frame counter (VQVAELookaheadStream's decoder: the encoder's
    # lookahead); every mask and edge lookahead of the generator grows by that many frames at its rate
    _shift = 0

    def _plan(self, model):
        """The generator's histories (``_build``) and its plan: the lookahead of each signal, in its own samples, from an
        input conv whose [history | chunk] window starts K - 1 frames before the frame counter"""
        ic = list(model.melgan)[1]
        self._build(model, centred=True)
        self.edge = model.pad_mode
        K_out = self.out_hist.shape[-1] + 1
        look = self.look_in = (ic.kernel_size[0] - 1) // 2
        need = [(look, 1)]  # (padding, input samples per frame) of every conv the pad applies to
        for lv in self.levels:
            s = lv["stride"]
            look = lv["look_u"] = look * s + s // 2 + s % 2
            for st in lv["stacks"]:
                st["P"] = (st["k"] - 1) // 2 * st["d"]
                st["look"] = look
                look += st["P"]
                need.append((st["P"], lv["rate"]))
        self.look_last = look
        self.look_sub = look + (K_out - 1) // 2
        need.append(((K_out - 1) // 2, self.hop))
        self.min_frames = max(P // rate + 1 for P, rate in need) if self.edge == "reflect" else 1
        self.delay = self.subbands * self.look_sub + self.pq_pad if self.pq_hist is not None else self.look_sub

    def _state(self):
        return self._histories() + [self.frame, self.end]

    def reset(self, items=None):
        super().reset(items)
        for b in self._slots(items):
            self._count[b] = 0

    def _step(self, c):
        """One chunk: c (B, in_channels, n) -> (B, out_channels or 1, n * hop * subbands).  Advances the state."""
        n = c.shape[-1]
        ent = self._entry(n)
        y = self._generate(ent, self._input(ent, c), n)
        self.frame += n
        return y

    def _generate(self, ent, xin, n):
        """The generator on the window xin = [history | n frames] of the entry; carries its histories, not the counter"""
        slope, edge, sh = self.slope, self.edge, self._shift

        def mask(rate, look):
            return self._mask(rate, look + sh * rate)

        # the input conv on [history | chunk]: input row r is frame t0 - (K - 1) + r
        h = ops.conv1d_stream(xin, None, *self.w_in, pad_left=0, out=ent["h0"], mask=mask(1, self.look_in), edge=edge,
                              in_lookahead=xin.shape[-1] - n + sh)
        for lv, buf in zip(self.levels, ent["levels"]):
            rate = lv["rate"]
            x = ops.conv_transpose1d_stream(h, lv["up_hist"], lv["w"][0], lv["w"][1], stride=lv["stride"], pre_slope=slope,
                                            out=buf["u"], mask=mask(rate, lv["look_u"]))
            for j, st in enumerate(lv["stacks"]):
                P, look, m = st["P"], st["look"], mask(rate, st["look"] + st["P"])
                hh = ops.conv1d_stream(x, st["hist"], *st["w1"], pad_left=(st["k"] - 1) * st["d"], dilation=st["d"], pre_slope=slope,
                                       out=buf["h"], mask=m, edge=edge, in_lookahead=look + sh * rate)
                # the skip reads the stack input P rows back, as h lags it
                s = ops.conv1d_stream(x, st["hist"], *st["ws"], pad_left=P, t_out=x.shape[-1], out=buf["s"])
                x = ops.conv1d_stream(hh, None, *st["w2"], pad_left=0, pre_slope=slope, residual=s, out=buf["x"][j], mask=m)
            h = x
        y = ops.conv1d_stream(h, self.out_hist, *self.w_out, pad_left=self.out_hist.shape[-1], pre_slope=slope, post_act=self.post_act,
                              out=ent["y"], mask=mask(self.hop, self.look_sub), edge=edge, in_lookahead=self.look_last + sh * self.hop)
        if self.pq_hist is not None:
            y = ops.conv_transpose1d_window_stream(y, self.pq_hist, self.w_syn, None, stride=self.subbands, padding=self.pq_pad,
                                                   out=ent["wave"])
            ops.stream_mask(y, self._mask(self.hop * self.subbands, self.delay))
        ops.stream_carry(ent["table"])
        return y

    @torch.no_grad()
    def push(self, c, normalize_before=False):
        """c: (B, n, in_channels) mel frames ((n, in_channels) when batch == 1).  Returns (B, 1, n * hop * subbands) on
        the device (out_channels rows for a multi-band model without PQMF): samples [t0 * hop * subbands - delay,
        (t0 + n) * hop * subbands - delay) of each slot's utterance."""
        c = self._frames(c, normalize_before)
        self._start(c)
        n = c.shape[-1]
        y = self._run(n, c)
        self._count = [k + n for k in self._count]
        return y

    @torch.no_grad()
    def flush(self, items=None):
        """The last ``delay`` samples of slots ``items`` (an index, an iterable of indices or None for every slot), as
        (len(items), 1, delay); the slots are then reset.  The flush push covers ceil(delay / (hop * subbands)) zero frames
        with the slots' end frames set, so every conv reads its pad about the signal's last sample.  The other slots'
        state is restored around it, so they continue exactly as if it had not happened; ending one slot costs a batch
        push (DESIGN.md §3.10).  A slot with fewer than ``min_frames`` frames raises, with nothing changed."""
        items = list(self._slots(items))
        short = [b for b in items if self._count[b] < self.min_frames]
        if short:
            raise PwgbError(f"MelGANLookaheadStream.flush: slots {short} hold fewer than {self.min_frames} frames "
                            f"({[self._count[b] for b in short]}); inference needs that many for the reflect padding")
        n = self._flush_frames()
        return self._flush(items, lambda: (n, self._zeros(self.B, self.in_channels, n)))


class VQVAELookaheadStream(MelGANLookaheadStream):
    """Streams the wav2wav conversion of a ``VQVAE`` (``decode(encode(x), l, g)``, the vctk / yesno ``vq1`` recipes:
    a ``MelGANDiscriminator`` encoder and a centred ``MelGANGenerator`` decoder) chunk by chunk for ``batch``
    independent slots, with a fixed lookahead of ``delay`` output samples.

    ``push(x, l, g)`` takes the next n * hop samples of every slot (hop = prod(downsample_scales)), their n local
    conditioning frames when the model has them, and the slots' target speaker ids when it has a global embedding, and
    returns n * hop samples: the converted samples from t0 * hop - delay on (t0: the frames pushed before), with zeros
    before sample 0.  ``flush(items)`` returns the last ``delay`` samples of those slots and restarts them; the other
    slots continue as if no flush had happened.  For every slot, the concatenated pushes and flush equal ``[zeros(delay)
    | model.decode(model.encode(all_x), all_l, g)]`` (``encode`` under ``torch.no_grad``, as inference runs it).  A
    slot's speaker may not change inside a signal.

    Two delayed-time chains (DESIGN.md §3.12, oracle/ref_vqvae_lookahead_stream.py), every launch masked outside its
    signal (pwgb_stream_ext):

    * the encoder on the audio: the reflect-padded input conv with the edge policy; each grouped strided conv (kernel K,
      stride s, padding p) at the smallest output lookahead L' = ceil((L + K - p - s) / s) for which the push's last
      output reads only samples that have arrived, on a window [the last L' s + p - L input samples | chunk] that starts
      on a stride boundary of the whole signal's padded input; it runs as ``encode`` runs it: the grouped space-to-depth
      gather read in place (pwgb_s2d_stream_grouped_forward) and the grouped masked stride-1 tensor-core conv where
      ``conv1d`` takes that route, else the grouped masked FFMA strided history conv; then the two centred stride-1 convs.
      The encoder's output lookahead is E whole frames (12 for [4, 4, 2, 2]);
    * the bottleneck, one pwgb_vq_stream_forward per push: the nearest code of each frame (the search of ``encode``),
      gathered with the local conditioning (after ``local_embed``, run on the pushed frames) read from an E-frame delay
      line, and the target speaker's embedding;
    * the decoder: the body of ``MelGANLookaheadStream`` on the frames the bottleneck wrote, E frames behind the frame
      counter, so ``delay`` = E * hop + the decoder's lookahead: 1305 samples (54 ms at 24 kHz) for the vctk recipes,
      1098 for yesno, the lookahead autograd measures on the model.

    ``min_frames`` is the decoder's (the reflect padding of ``decode``); ``flush`` refuses a slot with fewer.  With
    ``use_graphs`` each chunk length is captured once into a CUDA graph and replayed.  The weights and the conv engine
    (``ops.ENGINE``, which picks each strided conv's route as ``encode`` does) are read when the stream is built and must
    not change while it is used."""

    def __init__(self, model, batch=1, use_graphs=True):
        import math

        from .layers import CausalConv1d
        from .models import VQVAE, MelGANDiscriminator

        name = "VQVAELookaheadStream"
        if not isinstance(model, VQVAE):
            raise PwgbError(f"{name}: expected a VQVAE")
        enc, dec = model.encoder, model.decoder
        if not isinstance(enc, MelGANDiscriminator):
            raise PwgbError(f"{name}: the encoder is a {type(enc).__name__}; only MelGANDiscriminator is streamed")
        mods = list(dec.melgan)
        if isinstance(mods[0], CausalConv1d):
            raise PwgbError(f"{name}: the decoder is causal (use_causal_conv=True); only the centred MelGANGenerator is streamed")
        if dec.pqmf is not None:
            raise PwgbError(f"{name}: a decoder with PQMF synthesis is not streamed")
        if model.in_channels != 1:
            raise PwgbError(f"{name}: in_channels {model.in_channels}; the stream takes one audio channel")
        layers = list(enc.layers)
        strided = [q[0] for q in layers[1:-2]]
        down = math.prod(c.stride[0] for c in strided)
        up = math.prod(c.stride[0] for c in mods if isinstance(c, torch.nn.ConvTranspose1d))
        if down != up:
            raise PwgbError(f"{name}: prod(downsample_scales) {down} != prod(upsample_scales) {up}: a frame of audio must give "
                            "one frame of codes")
        self._setup(model, batch, use_graphs, mods[1].in_channels, mods[1].kernel_size[0] - 1, "zero")
        B, zeros = self.B, self._zeros
        # encoder: the reflect-padded input conv, the strided convs, the two centred stride-1 convs
        c0 = [q for q in layers[0] if isinstance(q, torch.nn.Conv1d)][0]
        self.enc_edge, self.enc_slope = enc.pad_mode, enc.slope
        self.w_e0 = wb(c0)
        self.e_hist = zeros(B, 1, c0.kernel_size[0] - 1)
        look = self.look_e0 = (c0.kernel_size[0] - 1) // 2
        rate, self.enc = down, []
        for conv in strided:
            s, K, p, G = conv.stride[0], conv.kernel_size[0], conv.padding[0], conv.groups
            Lq = -(-(look + K - p - s) // s)
            w, b = wb(conv)
            cin_g = conv.in_channels // G
            cgo = (cin_g * s + 31) // 32 * 32
            # the route of ops._conv1d_s2d under no_grad: the grouped space-to-depth and the stride-1 tensor-core conv
            # (its channel conditions, the tensor-core engine), else the FFMA strided conv
            s2d = ops.ENGINE != "simt" and (conv.out_channels // G) % 16 == 0 and cgo <= 2 * cin_g * s
            rate //= s
            self.enc.append(dict(stride=s, groups=G, kernel=K, w=(w, b), w2=ops.s2d_weight(w, s, cgo).contiguous() if s2d else None,
                                 cgo=cgo, rate=rate, look=Lq, cout=conv.out_channels, hist=zeros(B, conv.in_channels, Lq * s + p - look)))
            look = Lq
        self.tail = []
        for q in (layers[-2][0], layers[-1]):
            K, p = q.kernel_size[0], q.padding[0]
            look += K - 1 - p
            self.tail.append(dict(w=wb(q), look=look, cout=q.out_channels, hist=zeros(B, q.in_channels, K - 1)))
        self.E = look
        # bottleneck
        self.codebook = model.codebook.embedding.weight.detach()
        self.local = hasattr(model, "local_embed")
        self.w_le = wb(model.local_embed) if self.local and model.local_embed is not None else None
        self.l_in = (model.local_embed.in_channels if self.w_le is not None else None) if self.local else 0
        self.glob = hasattr(model, "global_embed")
        self.g_table = model.global_embed.weight.detach() if self.glob else None
        # decoder: MelGANLookaheadStream's plan and histories, E frames behind the counter
        self._shift = self.E
        self._plan(dec)
        self.dec_delay = self.delay
        self.delay = self.E * self.hop + self.dec_delay
        Cl = dec.melgan[1].in_channels - self.codebook.shape[1] - (self.g_table.shape[1] if self.glob else 0)
        if self.local and self.l_in is None:
            self.l_in = Cl  # num_local_embeds without local_embed_dim: l goes to the decoder as it is
        self.l_hist = zeros(B, Cl, self.E) if self.local else None
        self._counters()
        self._count = [0] * self.B
        self._g = [None] * self.B  # the speaker of each slot's signal, on the host
        self._nog = torch.zeros(self.B, device=self.dev, dtype=torch.int64)

    def _state(self):
        enc = [self.e_hist] + [lv["hist"] for lv in self.enc] + [t["hist"] for t in self.tail]
        return self._histories() + enc + ([self.l_hist] if self.local else []) + [self.frame, self.end]

    def reset(self, items=None):
        super().reset(items)
        for b in self._slots(items):
            self._g[b] = None

    def _new_entry(self, n, xin):
        """The decoder's buffers and carry table (``MelGANLookaheadStream``), the encoder's and the bottleneck's, and the
        carry table of the encoder's histories and the l delay line"""
        ent = super()._new_entry(n, xin)
        B, empty, hop = self.B, self._empty, self.hop
        ent["e"] = empty(B, 1, n * hop)
        ent["e0"] = empty(B, self.w_e0[0].shape[0], n * hop)
        carry, x = [(ent["e"], self.e_hist)], ent["e0"]
        ent["enc"] = []
        for lv in self.enc:
            t = n * lv["rate"]
            buf = dict(d=empty(B, lv["cout"], t))
            if lv["w2"] is not None:
                buf["xs"] = empty(B, lv["groups"] * lv["cgo"], t + -(-lv["kernel"] // lv["stride"]) - 1)
            carry.append((x, lv["hist"]))
            x = buf["d"]
            ent["enc"].append(buf)
        ent["tail"] = []
        for t in self.tail:
            carry.append((x, t["hist"]))
            x = empty(B, t["cout"], n)
            ent["tail"].append(x)
        if self.local:
            ent["l"] = empty(B, self.l_hist.shape[1], n)
            carry.append((ent["l"], self.l_hist))
        ent["idx"] = torch.empty((B, n), device=self.dev, dtype=torch.int64)
        ent["dec"] = empty(B, xin.shape[1], n)
        ent["enc_table"] = ops.stream_carry_table(carry, self.dev)
        return ent

    def _strided(self, lv, buf, h):
        """a strided conv on [hist | h], as ``MelGANDiscriminator.forward`` runs it on the whole signal: the window starts
        on a stride boundary of the whole signal's padded input, and its outputs are masked"""
        s, G, out = lv["stride"], lv["groups"], buf["d"]
        mask = self._mask(lv["rate"], lv["look"])
        if lv["w2"] is not None:
            xs = ops.s2d_stream(h, lv["hist"], s, buf["xs"].shape[-1], lv["cgo"], out=buf["xs"], groups=G)
            return ops.conv1d_stream(xs, None, lv["w2"], lv["w"][1], pad_left=0, post_act="lrelu", post_slope=self.enc_slope, out=out,
                                     mask=mask, groups=G)
        return ops.conv1d_strided_stream(h, lv["hist"], *lv["w"], stride=s, pad_left=lv["hist"].shape[-1], post_act="lrelu",
                                         post_slope=self.enc_slope, t_out=out.shape[-1], out=out, mask=mask, groups=G)

    def _step(self, e, l, g):
        """One chunk: e (B, 1, n * hop), l (B, l_in, n), g (B,) -> (B, 1, n * hop).  Advances the state."""
        n = e.shape[-1] // self.hop
        ent = self._entry(n)
        ent["e"].copy_(e)
        h = ops.conv1d_stream(ent["e"], self.e_hist, *self.w_e0, pad_left=self.e_hist.shape[-1], post_act="lrelu",
                              post_slope=self.enc_slope, out=ent["e0"], mask=self._mask(self.hop, self.look_e0), edge=self.enc_edge)
        for lv, buf in zip(self.enc, ent["enc"]):
            h = self._strided(lv, buf, h)
        for i, (t, out) in enumerate(zip(self.tail, ent["tail"])):
            act = dict(post_act="lrelu", post_slope=self.enc_slope) if i == 0 else {}
            h = ops.conv1d_stream(h, t["hist"], *t["w"], pad_left=t["hist"].shape[-1], out=out, mask=self._mask(1, t["look"]), **act)
        le = None
        if self.local:
            le = ops.conv1d(l, *self.w_le, out=ent["l"]) if self.w_le is not None else ent["l"].copy_(l)
        _, dec = ops.vq_stream(h, self.codebook, self._mask(1, self.E), l=le, l_hist=self.l_hist, global_table=self.g_table,
                               g=g if self.glob else None, indices=ent["idx"], dec=ent["dec"])
        ops.stream_carry(ent["enc_table"])
        y = self._generate(ent, self._input(ent, dec), n)
        self.frame += n
        return y

    @torch.no_grad()
    def push(self, x, l=None, g=None, return_indices=False):
        """x: (B, n * hop) or (B, 1, n * hop) audio samples, n >= 1; l: (B, num_local_embeds, n) local conditioning frames
        (required when the model has them, refused otherwise); g: (B,) target speaker ids (likewise).  Returns (B, 1, n *
        hop) on the device: samples [t0 * hop - delay, (t0 + n) * hop - delay) of each slot's converted signal; with
        ``return_indices`` also the (B, n) codes of frames t0 - E .. t0 + n - E - 1 (-1 outside the signal)."""
        name = "VQVAELookaheadStream.push"
        self._check_eval(self.model)
        x = torch.as_tensor(x, dtype=torch.float32, device=self.dev)
        if x.dim() == 3 and x.shape[1] == 1:
            x = x[:, 0]
        T = x.shape[-1] if x.dim() == 2 else 0
        if x.dim() != 2 or x.shape[0] != self.B or T < self.hop or T % self.hop:
            raise PwgbError(f"{name}: x must be ({self.B}, n * {self.hop}) or ({self.B}, 1, n * {self.hop}) samples with n >= 1, "
                            f"got {tuple(x.shape)}")
        n = T // self.hop
        if self.local:
            if l is None:
                raise PwgbError(f"{name}: the model has local conditioning; l ({self.B}, {self.l_in}, {n}) is required")
            l = torch.as_tensor(l, dtype=torch.float32, device=self.dev)
            if tuple(l.shape) != (self.B, self.l_in, n):
                raise PwgbError(f"{name}: l must be ({self.B}, {self.l_in}, {n}), got {tuple(l.shape)}")
            l = l.contiguous()
        elif l is not None:
            raise PwgbError(f"{name}: the model has no local conditioning; l must be None")
        else:
            l = self._zeros(self.B, 0, n)
        if self.glob:
            if g is None:
                raise PwgbError(f"{name}: the model has a global embedding; g ({self.B},) target speaker ids are required")
            gl = [int(v) for v in torch.as_tensor(g).reshape(-1).tolist()]
            if len(gl) != self.B:
                raise PwgbError(f"{name}: g must hold {self.B} speaker ids, got {len(gl)}")
            moved = [b for b in range(self.B) if self._g[b] is not None and self._g[b] != gl[b]]
            if moved:
                raise PwgbError(f"{name}: slots {moved} change speaker inside their signal ({[self._g[b] for b in moved]} -> "
                                f"{[gl[b] for b in moved]}); reset them first")
            g = torch.tensor(gl, device=self.dev, dtype=torch.int64)
        elif g is not None:
            raise PwgbError(f"{name}: the model has no global embedding; g must be None")
        else:
            g = self._nog
        y = self._run(n, x.reshape(self.B, 1, T).contiguous(), l, g)
        if self.glob:
            self._g = gl
        self._fresh = [False] * self.B
        self._count = [k + n for k in self._count]
        return (y, self._entries[n]["idx"].clone()) if return_indices else y

    @torch.no_grad()
    def flush(self, items=None):
        """The last ``delay`` samples of slots ``items`` (an index, an iterable of indices or None for every slot), as
        (len(items), 1, delay); the slots are then reset.  The flush push covers ceil(delay / hop) frames of zero audio and
        conditioning with the slots' end frames set, so every conv reads its pad about the signal's last sample; the other
        slots' state is restored around it, so they continue exactly as if it had not happened (DESIGN.md §3.12).  A slot
        with fewer than ``min_frames`` frames raises, with nothing changed."""
        items = list(self._slots(items))
        short = [b for b in items if self._count[b] < self.min_frames]
        if short:
            raise PwgbError(f"VQVAELookaheadStream.flush: slots {short} hold fewer than {self.min_frames} frames "
                            f"({[self._count[b] for b in short]}); decode needs that many for the reflect padding")
        n = self._flush_frames()
        l_ch = self.l_in if self.local else 0

        def inputs():
            g = torch.tensor([v or 0 for v in self._g], device=self.dev, dtype=torch.int64) if self.glob else self._nog
            return n, self._zeros(self.B, 1, n * self.hop), self._zeros(self.B, l_ch, n), g

        return self._flush(items, inputs)


class UHiFiGANLookaheadStream(_Lookahead, _HiFiGANStream):
    """Streams a centred ``UHiFiGANGenerator`` (every recipe: opencpop, opensinger, yesno) chunk by chunk for ``batch``
    independent slots, with a fixed lookahead of ``delay`` output samples.

    ``push(c, excitation)`` takes the next n >= 1 mel frames of every slot and their n * hop excitation samples, and
    returns n * hop samples: the whole-utterance samples from t0 * hop - delay on (t0: the frames pushed before), with
    zeros before sample 0.  ``flush(items)`` returns the last ``delay`` samples of those slots and restarts them; the
    other slots continue as if no flush had happened.  For every slot, the concatenated pushes and flush equal
    ``[zeros(delay) | model.inference(excitation=all_excitation, c=all_frames)]``.

    Each signal runs in delayed time behind the frames pushed, as in ``HiFiGANLookaheadStream`` (DESIGN.md §3.11,
    oracle/ref_uhifigan_lookahead_stream.py), and every launch masks the samples outside its signal to +0.0:

    * the encoder: the input conv on [the last K - 1 excitation samples | chunk], then per level the MRF of the HiFi-GAN
      stream (its block tables, delays and carries, from the level's input) and the strided conv (kernel 2 s, stride s,
      padding p).  Its output lookahead is the smallest L' for which the push's last output reads only input samples
      that have arrived, L' = ceil((L + s - p) / s), and it reads a window [the last L' s + p - L input samples | chunk]
      that starts on a stride boundary of the whole signal's padded input.  It runs as the whole-utterance conv does: the
      space-to-depth gather reading the history in place (pwgb_s2d_stream_forward) and the masked stride-1 tensor-core
      conv where ``conv1d`` takes that route, else the masked FFMA strided history conv
      (pwgb_conv1d_strided_stream_ext_forward);
    * the bottom: hidden_conv runs at the deepest skip's lookahead, on a history of that many frames plus (K - 1) / 2;
    * each decoder level: LeakyReLU -> ConvTranspose1d over cat(h, skip), whose two sources have different lookaheads.
      The skip, which is ahead at every level, is read back by the difference d from a delay line of d + 1 samples by the
      two-source stream conv-transpose (pwgb_conv_transpose1d_cat_stream_ext_forward); then the MRF.  A model whose
      decoder state is ahead of its skip is refused;
    * the output conv as in the HiFi-GAN stream (LeakyReLU 0.01, tanh).

    ``delay`` is the output conv's lookahead: 16231 samples (54.1 frames, 0.68 s at 24 kHz) for the opencpop recipe and
    5050 (19.7 frames) for yesno's.  It is this large because the bottom level's lag is multiplied by every upsample
    scale on the way up; it equals the largest lookahead autograd measures over the output phases of a hop (the last
    frame an output needs, times hop, minus the output's index), so no exact stream can have a smaller one.  With
    ``use_graphs`` each chunk length is captured once into a CUDA graph and replayed.  The weights and the conv engine
    (``ops.ENGINE``, which picks each strided conv's route as ``inference`` does) are read when the stream is built and must
    not change while it is used."""

    def __init__(self, model, batch=1, use_graphs=True):
        import math

        from .models import UHiFiGANGenerator

        name = "UHiFiGANLookaheadStream"
        if not isinstance(model, UHiFiGANGenerator):
            raise PwgbError(f"{name}: expected a UHiFiGANGenerator")
        self._check_eval(model)
        if next(model.parameters()).device.type != "cuda":
            raise PwgbError(f"{name}: the model must live on a CUDA device (no CPU fallback)")
        if model.use_causal_conv:
            raise PwgbError(f"{name}: a causal UHiFiGANGenerator cannot be built")
        if math.prod(model.downsample_scales) != math.prod(model.upsample_scales):
            raise PwgbError(f"{name}: prod(downsample_scales) {math.prod(model.downsample_scales)} != prod(upsample_scales) "
                            f"{math.prod(model.upsample_scales)}: a push must give whole samples at every encoder level")
        for kind, mods in (("downsample", [d[0] for d in model.downsamples]), ("upsample", [u[1] for u in model.upsamples])):
            for conv in mods:
                if conv.kernel_size[0] != 2 * conv.stride[0]:
                    raise PwgbError(f"{name}: a {kind} conv of kernel {conv.kernel_size[0]} and stride {conv.stride[0]}; the stream "
                                    "needs kernel 2 * stride")
        hc = model.hidden_conv
        K = model.kernel_size
        pk = (K - 1) // 2
        B = int(batch)
        self.B = B  # the plan's histories are allocated before _setup, which sizes the mel history from it
        self.dev = next(model.parameters()).device
        self.slope, self.nb = model.slope, model.num_blocks
        self.hop = math.prod(model.upsample_scales)
        zeros = self._zeros
        # encoder: the input conv on the excitation, then per level the MRF and the strided conv
        ic = model.input_conv[0]
        self.w_in = wb(ic)
        self.e_hist = zeros(B, 1, K - 1)
        self.look_in = pk
        look, rate, self.enc = pk, self.hop, []
        for i, s in enumerate(model.downsample_scales):
            conv = model.downsamples[i][0]
            C = conv.in_channels
            blocks, lvl_hist, L = self._mrf_level([model.downsamples_mrf[i * self.nb + j] for j in range(self.nb)], C, look, True)
            p = s // 2 + s % 2
            Lq = -(-(L + s - p) // s)
            w, b = wb(conv)
            cgo = (C * s + 31) // 32 * 32
            # the whole-utterance conv's route, fixed here: the space-to-depth gather and the stride-1 tensor-core conv
            # where ops._conv1d_s2d takes them (its channel conditions, the tensor-core engine), else the FFMA strided conv
            s2d = ops.ENGINE != "simt" and conv.out_channels % 16 == 0 and cgo <= 2 * C * s
            self.enc.append(dict(stride=s, channels=C, rate=rate, look_u=look, blocks=blocks, lvl_hist=lvl_hist, w=(w, b),
                                 w2=ops.s2d_weight(w, s, cgo).contiguous() if s2d else None, cgo=cgo, look_d=Lq,
                                 ds_hist=zeros(B, C, Lq * s + p - L)))
            rate //= s
            look = Lq
        # bottom: the deeper of the mel path and the deepest skip sets the decoder's first lookahead
        look_h = max(look, pk)
        self.look_hc = look_h
        self._setup(model, batch, use_graphs, hc.in_channels, look_h + pk, "zero")
        self.w_hc = wb(hc)
        # decoder: cat(h, skip) -> LeakyReLU -> ConvTranspose1d, then the MRF
        self.levels, rate = [], 1
        for i, s in enumerate(model.upsample_scales):
            e = self.enc[-1 - i]
            up = model.upsamples[i][1]
            C1 = up.in_channels - 2 * e["channels"]
            D = max(look_h, e["look_d"])
            d1, d2 = D - look_h, D - e["look_d"]  # the delay lines of the source ahead
            if d1:
                raise PwgbError(f"{name}: decoder level {i}'s skip runs {d1} samples behind its decoder state; the stream reads "
                                "only the skip through a delay line")
            rate *= s
            look_u = D * s + up.padding[0]
            cout = up.out_channels
            blocks, lvl_hist, look_h = self._mrf_level([model.upsamples_mrf[i * self.nb + j] for j in range(self.nb)], cout, look_u, True)
            self.levels.append(dict(stride=s, channels=cout, C1=C1, w=wb(up), rate=rate, look_u=look_u, blocks=blocks,
                                    lvl_hist=lvl_hist, d1=d1, d2=d2, h1_hist=zeros(B, C1, d1 + 1),
                                    h2_hist=zeros(B, up.in_channels - C1, d2 + 1)))
        oc = model.output_conv[1]
        self.w_out = wb(oc)
        self.out_hist = zeros(B, oc.in_channels, K - 1)
        self.out_channels = oc.out_channels
        self.delay = look_h + pk
        self._counters()

    def _state(self):
        hs = [self.cin_hist, self.out_hist, self.e_hist]
        for lv in self.enc:
            hs += [lv["lvl_hist"], lv["ds_hist"]]
            hs += [h for blk in lv["blocks"] for cv in blk["convs"] for h in (cv["x_hist"], cv["xt_hist"]) if h is not None]
        for lv in self.levels:
            hs += [lv["lvl_hist"], lv["h1_hist"], lv["h2_hist"]]
            hs += [h for blk in lv["blocks"] for cv in blk["convs"] for h in (cv["x_hist"], cv["xt_hist"]) if h is not None]
        return hs + [self.frame, self.end]

    def _new_entry(self, n, xin):
        """The buffers of every intermediate signal of an n-frame chunk, and the carry tables over them."""
        dev, B, empty = self.dev, self.B, self._empty
        ent = dict(e=empty(B, 1, n * self.hop), enc=[], levels=[])
        u = empty(B, self.enc[0]["channels"], n * self.hop)
        misc = [(ent["e"], self.e_hist), (xin, self.cin_hist)]
        for lv in self.enc:
            t = n * lv["rate"]
            buf = self._mrf_buffers(lv, t, [], u=u)
            s = lv["stride"]
            if lv["w2"] is not None:
                buf["xs"] = empty(B, lv["cgo"], t // s + 1)
            u = buf["d"] = empty(B, 2 * lv["channels"], t // s)
            misc.append((buf["cs"], lv["ds_hist"]))
            ent["enc"].append(buf)
        h = ent["h0"] = empty(B, self.w_hc[0].shape[0], n)
        t = n
        for i, lv in enumerate(self.levels):
            skip = ent["enc"][-1 - i]["d"]
            buf = self._mrf_buffers(lv, t * lv["stride"], [])
            misc += [(h, lv["h1_hist"]), (skip, lv["h2_hist"])]
            ent["levels"].append(buf)
            t *= lv["stride"]
            h = buf["cs"]
        ent["y"] = empty(B, self.out_channels, t)
        ent["out_table"] = ops.stream_carry_table([(h, self.out_hist)], dev)
        ent["table"] = ops.stream_carry_table(misc, dev)
        return ent

    def _strided(self, lv, buf, h):
        """the level's strided conv on [ds_hist | h], as ``UHiFiGANGenerator.forward`` runs it on the whole signal: the
        window starts on a stride boundary of the whole signal's padded input, and its outputs are masked"""
        s, out = lv["stride"], buf["d"]
        mask = self._mask(lv["rate"] // s, lv["look_d"])
        if lv["w2"] is not None:
            xs = ops.s2d_stream(h, lv["ds_hist"], s, out.shape[-1] + 1, lv["cgo"], out=buf["xs"])
            return ops.conv1d_stream(xs, None, lv["w2"], lv["w"][1], pad_left=0, post_act="lrelu", post_slope=self.slope, out=out,
                                     mask=mask)
        return ops.conv1d_strided_stream(h, lv["ds_hist"], *lv["w"], stride=s, pad_left=lv["ds_hist"].shape[-1], post_act="lrelu",
                                         post_slope=self.slope, t_out=out.shape[-1], out=out, mask=mask)

    def _step(self, c, e):
        """One chunk: c (B, in_channels, n), e (B, 1, n * hop) -> (B, out_channels, n * hop).  Advances the state."""
        n = c.shape[-1]
        ent = self._entry(n)
        slope = self.slope
        ent["e"].copy_(e)
        K = self.e_hist.shape[-1] + 1
        u = ops.conv1d_stream(ent["e"], self.e_hist, *self.w_in, pad_left=K - 1, post_act="lrelu", post_slope=slope,
                              out=ent["enc"][0]["u"], mask=self._mask(self.hop, self.look_in))
        for lv, buf in zip(self.enc, ent["enc"]):
            u = self._strided(lv, buf, self._mrf(lv, buf, u))
        # hidden_conv on [the last look_hc + (K - 1) / 2 frames | chunk]: n outputs at the decoder's first lookahead
        h = ops.conv1d_stream(self._input(ent, c), self._nohist, *self.w_hc, pad_left=0, t_out=n, out=ent["h0"],
                              mask=self._mask(1, self.look_hc))
        for i, (lv, buf) in enumerate(zip(self.levels, ent["levels"])):
            skip = ent["enc"][-1 - i]["d"]
            # the skip is read d2 samples back from its delay line
            u = ops.conv_transpose1d_cat_stream(h, lv["h1_hist"], skip, lv["h2_hist"], lv["d2"], *lv["w"], stride=lv["stride"],
                                                pre_slope=slope, out=buf["u"], mask=self._mask(lv["rate"], lv["look_u"]))
            h = self._mrf(lv, buf, u)
        ops.stream_carry(ent["table"])
        y = self._output(h, ent)
        self.frame += n
        return y

    @torch.no_grad()
    def push(self, c, excitation, normalize_before=False):
        """c: (B, n, in_channels) mel frames ((n, in_channels) when batch == 1); excitation: (B, n * hop) or (B, n, hop)
        ((n * hop,) or (n, hop) when batch == 1).  ``normalize_before`` normalises c with the model's statistics, as in
        the other streams.  Returns (B, out_channels, n * hop) on the device: samples [t0 * hop - delay, (t0 + n) * hop
        - delay) of each slot's utterance."""
        c = self._frames(c, normalize_before)
        n = c.shape[-1]
        e = torch.as_tensor(excitation, dtype=torch.float32, device=self.dev)
        T = n * self.hop
        shapes = {(self.B, T), (self.B, n, self.hop)} | ({(T,), (n, self.hop)} if self.B == 1 else set())
        if tuple(e.shape) not in shapes:
            raise PwgbError(f"UHiFiGANLookaheadStream.push: excitation must be ({self.B}, {T}) or ({self.B}, {n}, {self.hop}) for "
                            f"{n} frames, got {tuple(e.shape)}")
        self._start(c)
        return self._run(n, c, e.reshape(self.B, 1, T).contiguous())

    @torch.no_grad()
    def flush(self, items=None):
        """The last ``delay`` samples of slots ``items`` (an index, an iterable of indices or None for every slot), computed
        against the zero right padding, as (len(items), out_channels, delay); the slots are then reset.  The flush push
        covers ceil(delay / hop) zero frames and zero excitation with the slots' end frames set; the other slots' state is
        restored around it, so they continue exactly as if it had not happened (DESIGN.md §3.11)."""
        n = self._flush_frames()
        return self._flush(list(self._slots(items)),
                           lambda: (n, self._zeros(self.B, self.in_channels, n), self._zeros(self.B, 1, n * self.hop)))
