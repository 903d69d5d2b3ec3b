"""Chunked synthesis with a causal Parallel WaveGAN: mel frames in, waveform out, while the frames are still arriving.

A causal generator's output for frame j depends only on frames <= j, so it can be synthesised as soon as frame j
exists.  ``CausalPWGStream`` carries, per batch slot, everything the whole-utterance forward would read from before
the current chunk:

* conv_in (ConvInUpsampleNetwork): the last ``aux_context_window`` mel frames.  A fresh slot starts from its first
  frame replicated, as ``ReplicationPad1d`` does in ``inference``; conv_in then runs as a valid conv on
  [history | chunk];
* every causal FIR stage of the upsampler: its last two input frames (pwgb_upsample_fir_causal_stream_forward);
* every WaveNet layer l: its last H_l = (kernel - 1) * dilation_l input samples, in the packed residual stream's
  operand layout.  A causal layer reads only those rows in front of sample 0, so one copy per layer boundary
  (pwgb_wnstack_carry) puts the history where the whole-utterance forward has the previous samples, and the unchanged
  fused layer kernel computes the chunk as that forward would.

Every kernel computes each output sample with the same fp32 expression as ``model.inference`` on the whole utterance,
so the concatenated chunks equal it bit for bit as long as both runs take the same kernels (see DESIGN.md).  The
state is zeros for a fresh signal (the whole-utterance zero padding), so ``reset`` is a memset."""
import torch

from . import ops
from .capi import PwgbError
from .layers import ConvInUpsampleNetwork, UpsampleNetwork, effective_weight


def _layer_weights(f, A):
    """The packed operand image of one WaveNet layer, shared with ParallelWaveGANGenerator._forward_packed's cache."""
    k = ops.param_key(f.conv, f.conv1x1_aux, f.conv1x1_skip, f.conv1x1_out)
    ent = f._cache.get("wnp")
    if ent is not None and ent[0] == k:
        return ent[1], ent[2]
    return ops.wavenet_packed_weights(effective_weight(f.conv), effective_weight(f.conv1x1_aux), effective_weight(f.conv1x1_skip),
                                      effective_weight(f.conv1x1_out), f.conv1x1_skip.bias, f.conv1x1_out.bias, A,
                                      cache=f._cache, key=k, causal=True)


class CausalPWGStream:
    """Streams a causal ``ParallelWaveGANGenerator`` chunk by chunk for ``batch`` independent slots.

    ``push(c, z)`` takes the next n >= 1 frames of every slot and returns their n * hop samples; n may change from
    push to push.  For every slot, the concatenated outputs equal ``model.inference(c=all_frames, x=all_noise)``.
    There is no lookahead and no flush.  With ``use_graphs`` each chunk length is captured once into a CUDA graph and
    replayed.  The model's weights must not change while a stream uses them (the graphs hold the packed images)."""

    MAX_CHUNK_LENGTHS = 8

    def __init__(self, model, batch=1, seed=None, use_graphs=True):
        from .models import MelGANGenerator, ParallelWaveGANGenerator

        if not isinstance(model, ParallelWaveGANGenerator):
            raise PwgbError("CausalPWGStream: expected a ParallelWaveGANGenerator")
        if not model.use_causal_conv:
            raise PwgbError("CausalPWGStream: the model is not causal (use_causal_conv=False); a centred model needs lookahead")
        up = model.upsample_net
        if up is None:
            raise PwgbError("CausalPWGStream: upsample_conditional_features=False is not supported")
        if isinstance(up, MelGANGenerator):
            raise PwgbError("CausalPWGStream: upsample_net='MelGANGenerator' is not supported")
        if isinstance(up, UpsampleNetwork) and model.aux_context_window:
            raise PwgbError("CausalPWGStream: UpsampleNetwork with aux_context_window > 0 has no whole-utterance inference to match")
        self._check_eval(model)
        self.model = model
        self.dev = next(model.parameters()).device
        if self.dev.type != "cuda":
            raise PwgbError("CausalPWGStream: the model must live on a CUDA device (no CPU fallback)")
        self.B = int(batch)
        if self.B < 1:
            raise PwgbError("CausalPWGStream: batch must be >= 1")
        self.conv_in = up.conv_in if isinstance(up, ConvInUpsampleNetwork) else None
        fir_net = up.upsample if isinstance(up, ConvInUpsampleNetwork) else up
        self.scales = list(fir_net.upsample_scales)
        self.firs = [fir_net.up_layers[2 * i + 1] for i in range(len(self.scales))]
        self.hop = model.upsample_factor
        self.acw = model.aux_context_window if self.conv_in is not None else 0
        self.A = model.aux_channels
        l0 = model.conv_layers[0]
        self.R, self.G, self.K = l0.conv.in_channels, l0.conv.out_channels, l0.conv.kernel_size[0]
        self.S = l0.conv1x1_skip.out_channels
        self.dmax = max(f.dilation for f in model.conv_layers)
        self.H = [(self.K - 1) * f.dilation for f in model.conv_layers]
        if not ops.WnStack.supported(self.B, self.hop, self.R, self.G, self.S, self.A, self.K, self.dmax, True):
            raise PwgbError("CausalPWGStream: the fused packed WaveNet stack does not support this configuration "
                            f"(residual {self.R}, gate {self.G}, skip {self.S}, aux {self.A} channels, kernel {self.K})")
        dev, B, A = self.dev, self.B, self.A
        self.cin_hist = torch.zeros((B, A, self.acw), device=dev, dtype=torch.float32) if self.acw else None
        self.fir_hist = [torch.zeros((B * A, 2), device=dev, dtype=torch.float32) for _ in self.scales]
        self.fir_next = [torch.zeros((B * A, 2), device=dev, dtype=torch.float32) for _ in self.scales]
        self.wn_hist = [torch.zeros(B * self.R * h, device=dev, dtype=torch.int32) for h in self.H]
        self._fresh = [True] * B
        self.use_graphs = bool(use_graphs)
        self._entries = {}  # chunk frames -> {"stack": WnStack, "graph": ...}; a graph lives and dies with its stack
        self.gen = torch.Generator(device=dev)
        if seed is not None:
            self.gen.manual_seed(int(seed))

    @staticmethod
    def _check_eval(model):
        if model.training:
            raise PwgbError("CausalPWGStream: the model is in train mode; call model.eval() (dropout would apply)")

    # ---------------------------------------------------------------------------------------------------- state
    def _state(self):
        return ([self.cin_hist] if self.cin_hist is not None else []) + self.fir_hist + self.wn_hist

    def reset(self, items=None):
        """Restart slots ``items`` (an index or an iterable of indices; None: every slot) as fresh signals.  The other
        slots continue unaffected."""
        items = range(self.B) if items is None else ([items] if isinstance(items, int) else list(items))
        A = self.A
        for b in items:
            if not 0 <= b < self.B:
                raise PwgbError(f"CausalPWGStream.reset: slot {b} out of range [0, {self.B})")
            if self.cin_hist is not None:
                self.cin_hist[b].zero_()
            for h in self.fir_hist:
                h[b * A:(b + 1) * A].zero_()
            for h in self.wn_hist:
                h.view(self.B, -1)[b].zero_()
            self._fresh[b] = True

    # ---------------------------------------------------------------------------------------------------- compute
    def _entry(self, n):
        ent = self._entries.get(n)
        if ent is None:
            if len(self._entries) >= self.MAX_CHUNK_LENGTHS:
                self._entries.clear()
            ent = self._entries[n] = {"stack": ops.WnStack(self.B, n * self.hop, self.R, self.G, self.S, self.A, self.K, self.dmax,
                                                           self.dev, True)}
        return ent

    def _step(self, z, c):
        """One chunk: z (B, in_channels, n * hop), c (B, aux, n) -> (B, out_channels, n * hop).  Advances the state."""
        m = self.model
        n = c.shape[-1]
        # conditioning: conv_in on [history | chunk], then the causal FIR stages with their carried frames
        if self.conv_in is not None:
            x = c
            if self.acw:
                x = torch.cat([self.cin_hist, c], -1)
                self.cin_hist.copy_(x[:, :, n:])
            c = ops.conv1d(x, effective_weight(self.conv_in), None)
        last = len(self.scales) - 1
        for i, s in enumerate(self.scales):
            c = ops.upsample_fir_causal_stream(c, effective_weight(self.firs[i]), s, self.fir_hist[i], self.fir_next[i],
                                               out_channels=m._aux_pad if i == last else None)
            self.fir_hist[i].copy_(self.fir_next[i])
        # the residual stack on the packed stream; each layer's history is carried between the layer launches
        st = self._entry(n)["stack"]
        st.cur, st.prev = 0, None
        st.pack_c(c)
        fc = m.first_conv
        st.first_conv(z, effective_weight(fc), fc.bias)
        skips = torch.empty((self.B, self.S, z.shape[-1]), device=z.device, dtype=torch.float32)
        layers = m.conv_layers
        L = len(layers)
        st.carry(load=(self.wn_hist[0], self.H[0]))
        for i, f in enumerate(layers):
            packed, bso = _layer_weights(f, self.A)
            st.layer(packed, f.conv.bias, bso, f.dilation, skips, skips_init=(i == 0), write_x=(i < L - 1))
            st.carry(save=(self.wn_hist[i], self.H[i]), load=(self.wn_hist[i + 1], self.H[i + 1]) if i + 1 < L else None)
        # the output head as in ParallelWaveGANGenerator.forward: sqrt(1/layers) folded into the first 1x1 conv
        l1, l3 = m.last_conv_layers[1], m.last_conv_layers[3]
        h = ops.conv1d(skips, effective_weight(l1) * m._skip_scale, l1.bias, pre_slope=0.0)
        return ops.conv1d(h, effective_weight(l3), l3.bias, pre_slope=0.0)

    def _replay(self, z, c):
        ent = self._entry(c.shape[-1])
        if "graph" not in ent:
            static_z, static_c = z.clone(), c.clone()
            # one eager warm-up (packs weights, sets kernel attributes, fills the per-shape caches) advances the state:
            # it is restored before the capture, which itself runs nothing
            snap = [t.clone() for t in self._state()]
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                self._step(static_z, static_c)
            torch.cuda.current_stream().wait_stream(side)
            for t, s in zip(self._state(), snap):
                t.copy_(s)
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                out = self._step(static_z, static_c)
            ent.update(graph=graph, z=static_z, c=static_c, out=out)
        ent["z"].copy_(z)
        ent["c"].copy_(c)
        ent["graph"].replay()
        return ent["out"].clone()

    @torch.no_grad()
    def push(self, c, z=None, normalize_before=False):
        """c: (B, n, aux) mel frames ((n, aux) when batch == 1); z: optional (B, in_channels, n * hop) noise, drawn from
        the stream's generator when omitted.  Returns (B, out_channels, n * hop) on the device."""
        m = self.model
        self._check_eval(m)
        c = torch.as_tensor(c, dtype=torch.float32, device=self.dev)
        if c.dim() == 2 and self.B == 1:
            c = c.unsqueeze(0)
        if c.dim() != 3 or c.shape[0] != self.B or c.shape[2] != self.A or c.shape[1] < 1:
            raise PwgbError(f"CausalPWGStream.push: c must be ({self.B}, n >= 1, {self.A}), got {tuple(c.shape)}")
        if normalize_before:
            c = (c - m.mean) / m.scale
        c = c.transpose(1, 2).contiguous()
        n = c.shape[-1]
        T = n * self.hop
        if z is None:
            z = torch.randn((self.B, m.in_channels, T), device=self.dev, generator=self.gen)
        else:
            z = torch.as_tensor(z, dtype=torch.float32, device=self.dev)
            if tuple(z.shape) != (self.B, m.in_channels, T):
                raise PwgbError(f"CausalPWGStream.push: z must be ({self.B}, {m.in_channels}, {T}), got {tuple(z.shape)}")
            z = z.contiguous()
        if self.acw and any(self._fresh):  # ReplicationPad1d: a fresh slot's history is its first frame
            for b in range(self.B):
                if self._fresh[b]:
                    self.cin_hist[b].copy_(c[b, :, :1].expand(-1, self.acw))
        self._fresh = [False] * self.B
        return self._replay(z, c) if self.use_graphs else self._step(z, c)
