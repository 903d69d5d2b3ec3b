"""Decode driver -- the GPU side of ``parallel-wavegan-decode`` (bin/decode.py:214-243, SURVEY.md 8f-2).

The reference loops utterances one at a time through ``model.inference`` (host normalisation, one forward of
~80 launches, synchronous float D2H, ``sf.write(..., "PCM_16")``).  Here:

* utterances are sharded over ranks (``i mod world``; no collective) and batched by length;
* feature normalisation ``(c - mean) / scale`` (hifigan.py:264-265), the (T, C) -> (C, T) transpose and the edge
  padding (``ReplicationPad1d(aux_context_window)`` for Parallel WaveGAN) are one kernel per utterance writing straight
  into the batch slot (``pwgb_prep_features``);
* the generator forward of every distinct batch shape is captured once into a CUDA graph and replayed;
* the waveform is quantised to PCM16 on the GPU (``pwgb_pcm16_forward``, libsndfile's rule) and leaves the device
  as int16 through an asynchronous copy into pinned host memory -- an utterance crosses PCIe once each way.

``exact=True`` (default) batches only utterances of EQUAL length, so every waveform equals ``model.inference`` of that
utterance alone; ``exact=False`` pads a length bucket with zero frames (after normalisation) to a multiple of
``bucket_frames`` and crops -- samples within one receptive field of an utterance's end then see the padded tail
instead of the conv's zero padding.

``ragged=True`` (HiFi-GAN and the discrete-symbol HiFi-GAN) batches utterances of ANY lengths: the batch (sorted by
length) is padded to a multiple of ``bucket_frames`` and its per-item frame counts go to the device, where every layer
keeps each item zero past its own end (``HiFiGANGenerator.forward(c, lengths)``).  Every waveform then equals
``model.inference`` of that utterance alone (bit for bit wherever both take the same kernels, DESIGN.md §3.14).  One CUDA
graph per (batch, padded length) serves every mix of lengths, which are a static input of the graph.  A causal
HiFi-GAN needs the padding only.

The discrete-symbol HiFi-GAN decodes units: each input is a (T, 2) (symbol, speaker) or (T, 1) index array, padded
with symbol 0 past its end (and its own speaker).

The U-Net HiFi-GAN decodes mels with their excitations (bin/decode.py:156-230): ``decode(mels, excitations=...)``, one
(T', hop) or (T' * hop,) excitation per utterance, which crosses PCIe once from pinned memory into its batch slot and is
padded with zero samples where the mels get zero frames.  Mels and excitation are the static inputs of the graph."""
import ctypes as C

import numpy as np
import torch

from . import capi, ops, sharding
from .capi import PAD_REPLICATE, PAD_ZERO, PwgbError


def _stream():
    return ops._stream()


class GraphedGenerator:
    """Replays ``fn(*static_inputs)`` from a CUDA graph for every distinct tuple of input shapes.

    The first call with new shapes runs two eager warm-ups on a side stream (packs weights, sets kernel
    attributes, fills every per-shape cache), then captures; later calls copy the inputs into the static
    tensors and replay.  The graph holds the packed weight images: call ``reset()`` after changing weights."""

    def __init__(self, model, max_graphs=16, fn=None):
        self.model = model.eval() if hasattr(model, "eval") else model
        self.fn = fn if fn is not None else self.model
        self.max_graphs = max_graphs
        self._graphs = {}

    def reset(self):
        self._graphs.clear()

    @torch.no_grad()
    def __call__(self, *inputs):
        key = tuple(tuple(t.shape) for t in inputs)
        ent = self._graphs.get(key)
        if ent is None:
            if len(self._graphs) >= self.max_graphs:
                return self.fn(*inputs)
            static_in = [t.clone() for t in inputs]
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                for _ in range(2):
                    self.fn(*static_in)
            torch.cuda.current_stream().wait_stream(side)
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                static_out = self.fn(*static_in)
            ent = (graph, static_in, static_out)
            self._graphs[key] = ent
        graph, static_in, static_out = ent
        for s, t in zip(static_in, inputs):
            s.copy_(t)
        graph.replay()
        return static_out


def pcm16(y):
    """float waveform (any shape, CUDA) -> int16 tensor of the same shape (libsndfile's PCM_16 rule)."""
    if not y.is_cuda or y.dtype != torch.float32:
        raise PwgbError("pcm16: expected a float32 CUDA tensor (no CPU fallback)")
    y = y.contiguous()
    out = torch.empty(y.shape, device=y.device, dtype=torch.int16)
    rc = capi.lib().pwgb_pcm16_forward(C.c_void_p(y.data_ptr()), C.c_void_p(out.data_ptr()), y.numel(), _stream())
    capi.check(rc, "pwgb_pcm16_forward")
    return out


def prep_features(c, out, mean=None, scale=None, pad_left=0, replicate=False):
    """c: (T, C) features on the device -> out: (C, T_out) slot (normalised, transposed, edge-padded)."""
    T, Cc = c.shape
    rc = capi.lib().pwgb_prep_features(C.c_void_p(c.data_ptr()), C.c_void_p(mean.data_ptr()) if mean is not None else None,
                                       C.c_void_p(scale.data_ptr()) if scale is not None else None, C.c_void_p(out.data_ptr()), T, Cc,
                                       int(pad_left), out.shape[-1], PAD_REPLICATE if replicate else PAD_ZERO, _stream())
    capi.check(rc, "pwgb_prep_features")
    return out


def ragged_refusal(model):
    """Why ``Decoder(model, ragged=True)`` cannot batch utterances of different lengths, or None when it can."""
    from . import models

    t = type(model)
    if t is models.HiFiGANGenerator or t is models.DiscreteSymbolHiFiGANGenerator:
        return None
    reasons = {
        models.MelGANGenerator: "MelGAN pads its input by reflection at the signal's end (and multi-band MelGAN's PQMF "
                                "synthesis looks ahead), which a zero-padded batch cannot reproduce per item",
        models.ParallelWaveGANGenerator: "the fused WaveNet stack of Parallel WaveGAN has no per-item length mask",
        models.StyleMelGANGenerator: "StyleMelGAN's InstanceNorm takes statistics over the whole signal",
        models.UHiFiGANGenerator: "the U-Net HiFi-GAN's strided encoder and excitation input have no per-item length mask",
        models.DiscreteSymbolDurationGenerator: "the duration model's regulated length is only known after its predictor runs",
        models.VQVAE: "the VQ-VAE converts waveforms and has no per-item length mask",
    }
    for cls, why in reasons.items():
        if isinstance(model, cls):
            return why
    return f"{t.__name__} has no per-item length mask"


class Decoder:
    def __init__(self, model, use_graphs=True, max_batch=16, exact=True, bucket_frames=32, rank=0, world=1, seed=None,
                 ragged=False):
        self.max_batch, self.exact, self.bucket = int(max_batch), bool(exact), int(bucket_frames)
        self.ragged = bool(ragged)
        # a ragged batch passes per-item lengths to the non-causal HiFi-GAN body; a causal one needs the padding only
        self.masked = False
        if self.ragged:
            if self.max_batch < 1 or self.bucket < 1:
                raise PwgbError(f"Decoder(ragged=True): max_batch ({max_batch}) and bucket_frames ({bucket_frames}) must be positive")
            why = ragged_refusal(model)
            if why is not None:
                raise PwgbError(f"Decoder(ragged=True): {why}")
            if self.bucket % 4:
                raise PwgbError(f"Decoder(ragged=True): bucket_frames must be a multiple of 4 (the fused ResBlock pairs need "
                                f"t % 4 == 0), got {self.bucket}")
            self.masked = not getattr(model, "use_causal_conv", False)
        self.model = model.eval()
        self.dev = next(model.parameters()).device
        if self.dev.type != "cuda":
            raise PwgbError("Decoder: the model must live on a CUDA device (no CPU fallback)")
        self.kind = decoder_kind(model)
        self.rank, self.world = rank, world
        self.gen = torch.Generator(device=self.dev)
        if seed is not None:
            self.gen.manual_seed(int(seed))
        pq = getattr(model, "pqmf", None)

        def fwd(*a):
            y = model(*a)
            return pq.synthesis(y) if pq is not None else y

        def fwd_excitation(c, e):  # the U-Net HiFi-GAN: mels and excitation (its f0 input is unused)
            return model(c, None, e)

        run = fwd_excitation if self.kind == "uhifigan" else fwd
        self.runner = GraphedGenerator(model, fn=run) if use_graphs else run
        self.hop = (int(np.prod(model.upsample_scales)) if self.kind == "uhifigan" else
                    int(getattr(model, "upsample_factor", 0)) or None)
        self.ctx = int(getattr(model, "aux_context_window", 0)) if self.kind == "pwg" else 0

    def _groups(self, lengths, idxs):
        """(padded length, [indices]) batches: equal lengths (exact), length buckets, or (ragged) runs of up to max_batch
        utterances in length order, each padded to a multiple of bucket_frames above its longest"""
        if self.ragged:
            order = sorted(idxs, key=lambda i: (lengths[i], i))
            for k in range(0, len(order), self.max_batch):
                g = order[k : k + self.max_batch]
                yield max(-(-lengths[g[-1]] // self.bucket) * self.bucket, self.bucket), g
            return
        groups = {}
        for i in idxs:
            L = lengths[i]
            key = L if self.exact else -(-L // self.bucket) * self.bucket
            groups.setdefault(key, []).append(i)
        for key in sorted(groups):
            g = groups[key]
            for k in range(0, len(g), self.max_batch):
                yield key, g[k : k + self.max_batch]

    @torch.no_grad()
    def decode(self, mels, normalize_before=False, to_pcm16=True, noises=None, excitations=None):
        """mels: list of (T_i, C) arrays / tensors.  Returns {index: waveform}: int16 numpy arrays of shape (samples,)
        (``to_pcm16``) or float32 device tensors (samples, out_channels).  ``noises`` (Parallel WaveGAN only): optional
        {index: (samples, 1)} noise for reproducibility (``inference(c, x)``).  ``excitations`` (the U-Net HiFi-GAN
        only, and required there): a list aligned with ``mels``, entry i (T_i, hop) or (T_i * hop,)."""
        m = self.model
        idxs = list(sharding.partition(len(mels), self.rank, self.world))
        exc = None
        if self.kind == "uhifigan":
            if normalize_before:
                raise PwgbError("Decoder: the U-Net HiFi-GAN's inference ignores normalize_before; normalise the mels "
                                "before decoding (normalize_before=False)")
            exc = _excitation_rows(excitations, mels, idxs, self.hop)
        elif excitations is not None:
            raise PwgbError(f"Decoder: excitations are an input of the U-Net HiFi-GAN only, not of {type(m).__name__}")
        if self.kind == "style":  # batch-1 inference with its own noise / padding protocol (style_melgan.py:226-262)
            out = {}
            for i in idxs:
                y = m.inference(torch.as_tensor(mels[i], dtype=torch.float32, device=self.dev), normalize_before=normalize_before)
                out[i] = pcm16(y[:, 0]).cpu().numpy() if to_pcm16 else y
            return out
        units = self.kind == "units"
        if units and normalize_before:
            raise PwgbError("Decoder: units are not normalised (normalize_before=False)")
        mean = m.mean if normalize_before else None
        scale = m.scale if normalize_before else None
        if units:
            host = [_unit_rows(x, m.num_spk_embs > 0) for x in (mels[i] for i in idxs)]
        else:
            host = [torch.as_tensor(np.asarray(x, dtype=np.float32) if not isinstance(x, torch.Tensor) else x, dtype=torch.float32) for x in (mels[i] for i in idxs)]
        by_idx = dict(zip(idxs, host))
        lengths = {i: by_idx[i].shape[0] for i in idxs}
        out, pending = {}, []
        for Tb, grp in self._groups(lengths, idxs):
            B, Cc = len(grp), by_idx[grp[0]].shape[1]
            if units:
                # symbol 0 past an item's end (masked before input_conv), the item's own speaker throughout
                cin = torch.zeros((B, Cc, Tb), dtype=torch.int64)
                for b, i in enumerate(grp):
                    u = by_idx[i]
                    cin[b, :, : u.shape[0]] = u.transpose(0, 1)
                    if Cc == 2 and u.shape[0]:
                        cin[b, 1, u.shape[0] :] = u[0, 1]
                cin = cin.pin_memory().to(self.dev, non_blocking=True)
            else:
                cin = torch.empty((B, Cc, Tb + 2 * self.ctx), device=self.dev, dtype=torch.float32)
                for b, i in enumerate(grp):
                    src = by_idx[i]
                    src = src.pin_memory() if not src.is_cuda and not src.is_pinned() else src
                    prep_features(src.to(self.dev, non_blocking=True).contiguous(), cin[b], mean, scale, pad_left=self.ctx, replicate=self.ctx > 0)
            if self.masked:
                lens = torch.tensor([lengths[i] for i in grp], dtype=torch.int32).pin_memory().to(self.dev, non_blocking=True)
                y = self.runner(cin, lens)
            elif self.kind == "pwg":
                hop = m.upsample_factor
                z = torch.randn((B, 1, Tb * hop), device=self.dev, generator=self.gen)
                if noises:
                    for b, i in enumerate(grp):
                        if i in noises:
                            nz = torch.as_tensor(noises[i], dtype=torch.float32).to(self.dev).reshape(-1)
                            z[b, 0, : nz.numel()] = nz
                y = self.runner(z, cin)
            elif exc is not None:
                e = torch.empty((B, 1, Tb * self.hop), device=self.dev, dtype=torch.float32)
                for b, i in enumerate(grp):
                    src = exc[i]
                    src = src.pin_memory() if not src.is_cuda and not src.is_pinned() else src
                    n = src.numel()
                    e[b, 0, :n].copy_(src, non_blocking=True)
                    if n < e.shape[-1]:
                        e[b, 0, n:].zero_()
                y = self.runner(cin, e)
            else:
                y = self.runner(cin)
            hop = y.shape[-1] // Tb
            q = pcm16(y) if to_pcm16 else None
            for b, i in enumerate(grp):
                n = lengths[i] * hop
                if to_pcm16:
                    hbuf = torch.empty(n, dtype=torch.int16).pin_memory()
                    hbuf.copy_(q[b, 0, :n], non_blocking=True)
                    pending.append((i, hbuf))
                else:
                    out[i] = y[b, :, :n].transpose(1, 0).clone()
        if pending:
            torch.cuda.current_stream().synchronize()
            for i, hbuf in pending:
                out[i] = hbuf.numpy()
        return out


def decoder_kind(model):
    """How ``Decoder`` feeds a generator: "pwg" (noise and mels), "style" (per-utterance inference), "units" (the
    discrete-symbol HiFi-GAN), "uhifigan" (mels and excitation) or "mel2wav" (mels)."""
    from . import models

    return ("pwg" if isinstance(model, models.ParallelWaveGANGenerator) else
            "style" if isinstance(model, models.StyleMelGANGenerator) else
            "units" if type(model) is models.DiscreteSymbolHiFiGANGenerator else
            "uhifigan" if isinstance(model, models.UHiFiGANGenerator) else "mel2wav")


def _excitation_rows(excitations, mels, idxs, hop):
    """The excitations of utterances ``idxs`` as {i: (T_i * hop,) float32 tensor}, each checked against the frame count
    of mels[i]"""
    if excitations is None:
        raise PwgbError("Decoder: the U-Net HiFi-GAN needs excitations=[...], one per utterance (features.excitation)")
    if len(excitations) != len(mels):
        raise PwgbError(f"Decoder: {len(excitations)} excitations for {len(mels)} utterances")
    rows = {}
    for i in idxs:
        x = excitations[i]
        e = x if isinstance(x, torch.Tensor) else torch.from_numpy(np.asarray(x, dtype=np.float32))
        e = e.to(torch.float32).reshape(-1)
        want = int(np.shape(mels[i])[0]) * hop
        if e.numel() != want:
            raise PwgbError(f"Decoder: excitation {i} has {e.numel()} samples, its {want // hop} frames need {want} (hop {hop})")
        rows[i] = e.contiguous()
    return rows


def _unit_rows(x, speakers):
    """One utterance of units: (T, 2) (symbol, speaker) or (T, 1) / (T,) symbols -> (T, K) int64 on the host, K = 2 with
    speakers, else 1 (DiscreteSymbolHiFiGANGenerator.inference's input)"""
    u = torch.as_tensor(np.asarray(x) if not isinstance(x, torch.Tensor) else x).cpu()
    if u.dim() == 1:
        u = u[:, None]
    if u.dim() != 2 or u.shape[1] not in (1, 2) or (speakers and u.shape[1] != 2):
        raise PwgbError(f"Decoder: units must be (T, 2) (symbol, speaker){' or (T, 1)' if not speakers else ''}, got {tuple(u.shape)}")
    u = u.to(torch.int64)
    return u if speakers else u[:, :1]


@torch.no_grad()
def decode_utterances(model, mels, rank=0, world=1, normalize_before=False, use_graphs=True):
    """Decode this rank's share (i mod world == rank) of ``mels`` (list of (T', C) tensors / arrays), every utterance
    bit-identical to ``model.inference`` of it alone.  Returns {index: waveform (T, out_channels) on the device}."""
    return Decoder(model, use_graphs=use_graphs, rank=rank, world=world).decode(mels, normalize_before=normalize_before, to_pcm16=False)
