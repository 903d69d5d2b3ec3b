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
with symbol 0 past its end (and its own speaker).  The discrete-symbol StyleMelGAN decodes units one utterance at a
time through ``inference``, like StyleMelGAN (its InstanceNorm takes statistics over the whole signal, so padding
would change every item): (T, 2) units, or (T, 1) units with ``speakers=[...]``.

The U-Net HiFi-GAN decodes mels with their excitations (bin/decode.py:156-230): ``decode(mels, excitations=...)``, one
(T', hop) or (T' * hop,) excitation per utterance, which crosses PCIe once from pinned memory into its batch slot and is
padded with zero samples where the mels get zero frames.  Mels and excitation are the static inputs of the graph.

The VQ-VAE converts waveforms (bin/decode.py's VQ-WAV2WAV branch): ``convert(waves, locals, globals)`` runs ``z =
model.encode(x); y = model.decode(z, l, g)`` per utterance and returns the converted waveform and the code indices.
With ``ragged=True`` the per-layer lengths of each batch (the encoder's ceil(L / s) chain and the decoder's frames) go
to the device, where every conv keeps each item zero past its own end and reflects at its own end
(``VQVAE.encode(x, lengths)`` / ``decode(..., lengths)``, DESIGN.md §3.16)."""
import ctypes as C

import numpy as np
import torch

from . import capi, ops, sharding
from .capi import PAD_REPLICATE, PAD_ZERO, PwgbError
from .layers import CausalConv1d


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
    if t is models.HiFiGANGenerator or t is models.DiscreteSymbolHiFiGANGenerator or t is models.VQVAE:
        return None
    reasons = {
        models.MelGANGenerator: "MelGAN pads its input by reflection at the signal's end (and multi-band MelGAN's PQMF "
                                "synthesis looks ahead), which a zero-padded batch cannot reproduce per item",
        models.ParallelWaveGANGenerator: "the fused WaveNet stack of Parallel WaveGAN has no per-item length mask",
        models.StyleMelGANGenerator: "StyleMelGAN's InstanceNorm takes statistics over the whole signal",
        models.DiscreteSymbolStyleMelGANGenerator: "StyleMelGAN's InstanceNorm takes statistics over the whole signal",
        models.UHiFiGANGenerator: "the U-Net HiFi-GAN's strided encoder and excitation input have no per-item length mask",
        models.DiscreteSymbolDurationGenerator: "the duration model's regulated length is only known after its predictor runs",
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
        if self.kind == "wav2wav":
            _check_wav2wav(model)
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

        def fwd_wav2wav(x, *a):  # waveforms, the model's locals and globals, then (ragged) the encoder's layer lengths
            k = 0
            l = g = None
            if hasattr(model, "local_embed"):
                l, k = a[k], k + 1
            if hasattr(model, "global_embed"):
                g, k = a[k], k + 1
            lens = list(a[k:])
            if not lens:
                idx = model.encode(x)
                return model.decode(idx, l, g), idx
            idx = model.codebook(model.encoder(x, lens)[-1])
            return model._decode(idx, l, g, lens[-1]), idx

        run = {"uhifigan": fwd_excitation, "wav2wav": fwd_wav2wav}.get(self.kind, fwd)
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
    def decode(self, mels, normalize_before=False, to_pcm16=True, noises=None, excitations=None, speakers=None):
        """mels: list of (T_i, C) arrays / tensors (units for the discrete-symbol generators).  Returns {index:
        waveform}: int16 numpy arrays of shape (samples,) (``to_pcm16``) or float32 device tensors (samples,
        out_channels).  ``noises`` (Parallel WaveGAN only): optional {index: (samples, 1)} noise for reproducibility
        (``inference(c, x)``).  ``excitations`` (the U-Net HiFi-GAN only, and required there): a list aligned with
        ``mels``, entry i (T_i, hop) or (T_i * hop,).  ``speakers`` (the discrete-symbol StyleMelGAN only): a list
        aligned with ``mels`` of speaker ids, which replace the units' speaker column as ``inference(c, g)`` does;
        without it every utterance is (T_i, 2) (symbol, speaker)."""
        m = self.model
        if self.kind == "wav2wav":
            raise PwgbError("Decoder: a VQ-VAE converts waveforms; use Decoder.convert(waves, locals, globals)")
        if speakers is not None and self.kind != "style_units":
            raise PwgbError(f"Decoder: speakers are an input of the discrete-symbol StyleMelGAN only, not of {type(m).__name__}")
        idxs = list(sharding.partition(len(mels), self.rank, self.world))
        exc = None
        if self.kind == "uhifigan":
            if normalize_before:
                raise PwgbError("Decoder: the U-Net HiFi-GAN's inference ignores normalize_before; normalise the mels "
                                "before decoding (normalize_before=False)")
            exc = _excitation_rows(excitations, mels, idxs, self.hop)
        elif excitations is not None:
            raise PwgbError(f"Decoder: excitations are an input of the U-Net HiFi-GAN only, not of {type(m).__name__}")
        if self.kind == "style_units":  # batch-1 inference, as the "style" kind, on units
            if normalize_before:
                raise PwgbError("Decoder: units are not normalised (normalize_before=False)")
            if noises is not None:
                raise PwgbError("Decoder: the discrete-symbol StyleMelGAN draws its noise in inference (style_melgan.py:588-595); "
                                "noises are an input of Parallel WaveGAN only")
            spk = _speaker_list(speakers, len(mels), idxs, m.num_spk_embs)
            out = {}
            for i in idxs:
                u = _unit_rows(mels[i], speakers=spk is None).to(self.dev)
                y = m.inference(u, g=None if spk is None else spk[i])
                out[i] = pcm16(y[:, 0]).cpu().numpy() if to_pcm16 else y
            return out
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


    @torch.no_grad()
    def convert(self, waves, locals=None, globals=None, to_pcm16=True):
        """VQ-VAE wav2wav (bin/decode.py's VQ-WAV2WAV branch): ``z = model.encode(x); y = model.decode(z, l, g)`` for
        every utterance of this rank's share.  waves: list of (T_i,) or (T_i, 1) arrays / tensors; ``locals`` (models
        with local conditioning, and required there): one (T'_i, num_local_embeds) array per utterance, T'_i = ceil(T_i
        / hop); ``globals`` (models with a global embedding, and required there): one speaker id per utterance.
        Returns {index: (waveform, indices)}: the waveform of T'_i * hop samples as int16 numpy (``to_pcm16``) or a
        float32 device tensor (T'_i * hop, 1), the indices a (T'_i,) int64 numpy array (the reference's ``text``)."""
        m = self.model
        if self.kind != "wav2wav":
            raise PwgbError(f"Decoder.convert: {type(m).__name__} is not a VQ-VAE; use Decoder.decode(mels)")
        if m.training:
            raise PwgbError("Decoder.convert: the model is in train mode; call model.eval() (dropout-free inference)")
        hop = m.hop
        idxs = list(sharding.partition(len(waves), self.rank, self.world))
        xs = {i: _wave_row(waves[i], i) for i in idxs}
        samples = {i: xs[i].numel() for i in idxs}
        frames = {i: -(-samples[i] // hop) for i in idxs}
        least = m.min_ragged_samples()
        short = [i for i in idxs if samples[i] < least]
        if short:
            raise PwgbError(f"Decoder.convert: utterances {short} hold fewer than {least} samples, which the reflect pads of "
                            f"encode / decode need")
        ls = _cond_rows(m, locals, len(waves), idxs, frames)
        gs = _speaker_ids(m, globals, len(waves), idxs)
        out, pending = {}, []
        for key, grp in self._groups(samples if self.exact and not self.ragged else frames, idxs):
            B = len(grp)
            T = key if self.exact and not self.ragged else key * hop  # padded samples
            Tf = -(-T // hop)
            x = torch.zeros((B, 1, T), device=self.dev, dtype=torch.float32)
            for b, i in enumerate(grp):
                x[b, 0, : samples[i]].copy_(_pinned(xs[i]), non_blocking=True)
            args = [x]
            if ls is not None:
                l = torch.zeros((B, ls[grp[0]].shape[1], Tf), dtype=torch.float32)
                for b, i in enumerate(grp):
                    l[b, :, : frames[i]] = ls[i].transpose(0, 1)
                args.append(l.pin_memory().to(self.dev, non_blocking=True))
            if gs is not None:
                args.append(torch.tensor([gs[i] for i in grp], dtype=torch.int64).pin_memory().to(self.dev, non_blocking=True))
            if self.ragged:
                lens = torch.stack(m.encoder.layer_lengths(torch.tensor([samples[i] for i in grp], dtype=torch.int32)))
                lens = lens.pin_memory().to(self.dev, non_blocking=True)
                args += list(lens.unbind(0))
            y, idx = self.runner(*args)
            q = pcm16(y) if to_pcm16 else None
            for b, i in enumerate(grp):
                n = frames[i] * hop
                ibuf = torch.empty(frames[i], dtype=torch.int64).pin_memory()
                ibuf.copy_(idx[b, : frames[i]], non_blocking=True)
                if to_pcm16:
                    hbuf = torch.empty(n, dtype=torch.int16).pin_memory()
                    hbuf.copy_(q[b, 0, :n], non_blocking=True)
                    pending.append((i, hbuf, ibuf))
                else:
                    pending.append((i, y[b, :, :n].transpose(1, 0).clone(), ibuf))
        torch.cuda.current_stream().synchronize()
        for i, w, ibuf in pending:
            out[i] = (w.numpy() if to_pcm16 else w, ibuf.numpy())
        return out


def decoder_kind(model):
    """How ``Decoder`` feeds a generator: "pwg" (noise and mels), "style" (per-utterance inference), "style_units"
    (per-utterance inference of the discrete-symbol StyleMelGAN on units), "units" (the discrete-symbol HiFi-GAN),
    "uhifigan" (mels and excitation), "wav2wav" (the VQ-VAE: waveforms, ``convert``) or "mel2wav" (mels)."""
    from . import models

    return ("pwg" if isinstance(model, models.ParallelWaveGANGenerator) else
            "style_units" if isinstance(model, models.DiscreteSymbolStyleMelGANGenerator) else
            "style" if isinstance(model, models.StyleMelGANGenerator) else
            "units" if type(model) is models.DiscreteSymbolHiFiGANGenerator else
            "uhifigan" if isinstance(model, models.UHiFiGANGenerator) else
            "wav2wav" if isinstance(model, models.VQVAE) else "mel2wav")


def _check_wav2wav(model):
    """The VQ-VAE configurations ``convert`` serves: one audio channel in and out through the MelGAN encoder / decoder"""
    from . import models

    if not isinstance(model.encoder, models.MelGANDiscriminator) or not isinstance(model.decoder, models.MelGANGenerator):
        raise PwgbError("Decoder: the VQ-VAE must have a MelGANDiscriminator encoder and a MelGANGenerator decoder")
    if isinstance(list(model.decoder.melgan)[0], CausalConv1d):
        raise PwgbError("Decoder: a causal VQ-VAE decoder (use_causal_conv=True) is not converted")
    if model.decoder.pqmf is not None or [q for q in model.decoder.melgan if isinstance(q, torch.nn.Conv1d)][-1].out_channels > 1:
        raise PwgbError("Decoder: out_channels > 1 (the reference's PQMF synthesis branch) is not converted")
    if model.in_channels != 1:
        raise PwgbError(f"Decoder: in_channels {model.in_channels}; convert takes one audio channel")


def _pinned(t):
    return t.pin_memory() if not t.is_cuda and not t.is_pinned() else t


def _wave_row(x, i):
    """one waveform, (T,) or (T, 1), as a (T,) float32 tensor on the host (or where it already is)"""
    w = x if isinstance(x, torch.Tensor) else torch.from_numpy(np.asarray(x, dtype=np.float32))
    if w.dim() == 2 and w.shape[1] == 1:
        w = w[:, 0]
    if w.dim() != 1:
        raise PwgbError(f"Decoder.convert: waveform {i} must be (T,) or (T, 1), got {tuple(w.shape)}")
    return w.to(torch.float32).contiguous()


def _cond_rows(model, locals, n, idxs, frames):
    """the local conditioning of utterances ``idxs`` as {i: (T'_i, C) float32 host tensor}, or None for a model without"""
    if not hasattr(model, "local_embed"):
        if locals is not None:
            raise PwgbError("Decoder.convert: the model has no local conditioning; locals must be None")
        return None
    if locals is None:
        raise PwgbError("Decoder.convert: the model has local conditioning; locals=[...] (T'_i, num_local_embeds) are required")
    if len(locals) != n:
        raise PwgbError(f"Decoder.convert: {len(locals)} local tracks for {n} utterances")
    C_in = model.local_embed.in_channels if model.local_embed is not None else None
    rows = {}
    for i in idxs:
        l = torch.as_tensor(np.asarray(locals[i], dtype=np.float32) if not isinstance(locals[i], torch.Tensor) else locals[i])
        l = l.to(torch.float32).cpu()
        if l.dim() != 2 or l.shape[0] != frames[i] or (C_in is not None and l.shape[1] != C_in):
            raise PwgbError(f"Decoder.convert: local track {i} is {tuple(l.shape)}; the encoder gives {frames[i]} frames "
                            f"(ceil(samples / hop)){f' of {C_in} channels' if C_in is not None else ''}")
        rows[i] = l
    return rows


def _speaker_ids(model, globals, n, idxs):
    """the target speaker of utterances ``idxs`` as {i: int}, or None for a model without a global embedding"""
    if not hasattr(model, "global_embed"):
        if globals is not None:
            raise PwgbError("Decoder.convert: the model has no global embedding; globals must be None")
        return None
    if globals is None:
        raise PwgbError("Decoder.convert: the model has a global embedding; globals=[...] (one speaker id per utterance) are required")
    return _speaker_list(globals, n, idxs, model.global_embed.num_embeddings, "Decoder.convert")


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


def _speaker_list(speakers, n, idxs, num_spk, who="Decoder"):
    """The speaker ids of utterances ``idxs`` as {i: int}, each checked against the table size, or None without
    ``speakers``"""
    if speakers is None:
        return None
    if len(speakers) != n:
        raise PwgbError(f"{who}: {len(speakers)} speaker ids for {n} utterances")
    ids = {i: int(np.asarray(speakers[i]).reshape(-1)[0]) if np.asarray(speakers[i]).size == 1 else None for i in idxs}
    bad = [i for i in idxs if ids[i] is None or not 0 <= ids[i] < num_spk]
    if bad:
        raise PwgbError(f"{who}: utterances {bad} need one speaker id in [0, {num_spk})")
    return ids


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
