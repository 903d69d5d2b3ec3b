"""Input pipeline on the GPU (SURVEY.md 8f-3): a device-resident corpus + the training collater.

``DeviceCorpus`` keeps every utterance of a training set in HBM (audio concatenated in one tensor, feature
matrices concatenated along frames); ``Collater`` mirrors ``parallel_wavegan.bin.train.Collater`` (train.py:646-925):
same constructor arguments, same filtering of short utterances, the SAME host RNG call sequence for the crop
positions (one ``np.random.randint(start_offset, length + end_offset)`` per kept item, train.py:739-744), so a given
``np.random.seed`` yields the reference's batch bit for bit; the gather itself is one kernel (``pwgb_collate_crop``)
and the noise ``z`` of the Parallel WaveGAN recipes is drawn on the device."""
import ctypes as C

import numpy as np
import torch

from . import capi
from .capi import PwgbError


class DeviceCorpus:
    """items: list of (audio (T,), feats (frames, C)) numpy arrays / tensors [mel2wav case], of
    (audio, feats, f0 (frames,), excitation (frames, E)) [UHiFiGAN recipes], or of audio arrays [audio-only case].
    ``hop_size`` applies ``Collater._adjust_length`` (train.py:868-893): audio shorter than ``frames * hop_size`` is
    edge-padded; any other mismatch is an error, like the reference's assert.  f0 is kept as a 1-channel feature
    matrix whose rows line up with the features', excitation flattened like audio (E samples per frame)."""

    def __init__(self, items, device, hop_size=None):
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise PwgbError("DeviceCorpus lives on a CUDA device (no CPU fallback)")
        auds, fts, self.x_start, self.c_start, self.x_len, self.c_len = [], [], [], [], [], []
        f0s, exs, self.e_start = [], [], []
        xo = co = eo = 0
        self.has_feats = len(items) > 0 and isinstance(items[0], (tuple, list))
        self.has_f0 = self.has_feats and len(items[0]) == 4
        self.excitation_width = 0
        for it in items:
            x, c = (it[0], it[1]) if self.has_feats else (it, None)
            if self.has_f0:
                f0 = np.asarray(it[2], dtype=np.float32).reshape(-1, 1)
                ex = np.asarray(it[3], dtype=np.float32)
                ex = ex.reshape(len(ex), -1)
                if len(f0) != len(c) or len(ex) != len(c):
                    raise PwgbError(f"f0 / excitation have {len(f0)} / {len(ex)} frames, features {len(c)}")
                if self.excitation_width and ex.shape[1] != self.excitation_width:
                    raise PwgbError("excitation frames of different widths")
                self.excitation_width = ex.shape[1]
                f0s.append(torch.from_numpy(f0))
                exs.append(torch.from_numpy(ex.reshape(-1)))
                self.e_start.append(eo)
                eo += ex.size
            x = np.asarray(x, dtype=np.float32).reshape(-1)
            if c is not None:
                c = np.asarray(c, dtype=np.float32)
                if hop_size is not None:
                    if len(x) < len(c) * hop_size:
                        x = np.pad(x, (0, len(c) * hop_size - len(x)), mode="edge")
                    if len(x) != len(c) * hop_size:
                        raise PwgbError(f"audio / feature length mismatch: {len(x)} != {len(c)} * {hop_size}")
                fts.append(torch.from_numpy(c))
                self.c_start.append(co)
                self.c_len.append(len(c))
                co += len(c)
            auds.append(torch.from_numpy(x))
            self.x_start.append(xo)
            self.x_len.append(len(x))
            xo += len(x)
        self.audio = torch.cat(auds).to(self.device) if auds else torch.empty(0, device=self.device)
        self.feats = torch.cat(fts).contiguous().to(self.device) if fts else None
        self.channels = self.feats.shape[1] if self.feats is not None else 0
        self.f0 = torch.cat(f0s).contiguous().to(self.device) if f0s else None
        self.excitation = torch.cat(exs).to(self.device) if exs else None

    def __len__(self):
        return len(self.x_start)


class Collater:
    """``Collater`` of bin/train.py:646-925 for the mel2wav and audio-only cases, on the device."""

    def __init__(self, batch_max_steps=20480, hop_size=256, aux_context_window=2, use_noise_input=False, use_aux_input=True,
                 use_f0_and_excitation=False, use_duration=False, pad_value=0):
        if hop_size is not None:
            if batch_max_steps % hop_size != 0:
                batch_max_steps += -(batch_max_steps % hop_size)
            assert batch_max_steps % hop_size == 0
            self.hop_size = hop_size
            self.batch_max_frames = batch_max_steps // hop_size
        self.batch_max_steps = batch_max_steps
        self.aux_context_window = aux_context_window
        self.use_noise_input = use_noise_input
        self.use_aux_input = use_aux_input
        self.use_f0_and_excitation = use_f0_and_excitation
        self.use_duration = use_duration
        self.pad_value = pad_value  # the duration collater pads codes with it: generator_params["num_embs"] (train.py:1321-1323)
        if use_duration and (not use_aux_input or use_noise_input):
            raise PwgbError("Collater(use_duration=True) needs use_aux_input=True and use_noise_input=False (train.py:691-695)")
        if not use_aux_input:
            assert not use_noise_input, "Not supported."
        if use_aux_input:
            self.start_offset = aux_context_window
            self.end_offset = -(self.batch_max_frames + aux_context_window)
            self.mel_threshold = self.batch_max_frames + 2 * aux_context_window
        else:
            self.start_offset = 0
            self.end_offset = -self.batch_max_steps
            self.audio_threshold = self.batch_max_steps
        self.generator = None  # optional torch.Generator (device) for the noise input

    def __call__(self, corpus, indices):
        """indices: the utterance ids of this batch (what the sampler yields).  Returns ``(inputs, y)`` exactly like
        the reference: inputs = (z, c) / (c,) [mel2wav] with c (B, C, frames + 2*ctx) and y (B, 1, T); with
        ``use_f0_and_excitation`` (train.py:758-797) f0 (B, 1, F) and excitation (B, 1, F * E) follow, cropped at the
        feature rows of c (F = frames + 2*ctx), each gathered by one more pwgb_collate_crop launch.  With ``use_duration``
        (train.py:768-783) it returns ``(c, y, ds)``: the cropped (F, C) symbol rows, truncated to int64, run-length encoded
        per item (torch.unique_consecutive(dim=0)); c (B, C, S) int64 padded with ``pad_value``, ds (B, S) int64 run
        lengths padded with 0.  pwgb_collate_runlength counts the runs at the crop offsets, the host reads the B counts
        to size S (one device-to-host copy), and a second pass writes codes and lengths."""
        dev = corpus.device
        if self.use_aux_input:
            if not corpus.has_feats:
                raise PwgbError("Collater(use_aux_input=True) needs a corpus with features")
            keep = [i for i in indices if corpus.c_len[i] > self.mel_threshold]  # train.py:727-729
            starts = np.array([np.random.randint(self.start_offset, corpus.c_len[i] + self.end_offset) for i in keep], dtype=np.int64)
            x_off = np.array([corpus.x_start[i] for i in keep], dtype=np.int64) + starts * self.hop_size
            c_off = np.array([corpus.c_start[i] for i in keep], dtype=np.int64) + starts - self.aux_context_window
            F = self.batch_max_frames + 2 * self.aux_context_window
        else:
            keep = [i for i in indices if corpus.x_len[i] >= self.audio_threshold]  # train.py:840-843
            starts = np.array([np.random.randint(self.start_offset, corpus.x_len[i] + self.end_offset) for i in keep], dtype=np.int64)
            x_off = np.array([corpus.x_start[i] for i in keep], dtype=np.int64) + starts
            c_off, F = None, 0
        B, T = len(keep), self.batch_max_steps
        y = torch.empty((B, 1, T), device=dev, dtype=torch.float32)
        xo = torch.from_numpy(x_off).pin_memory().to(dev, non_blocking=True)
        c = co = None
        if c_off is not None:
            co = torch.from_numpy(c_off).pin_memory().to(dev, non_blocking=True)
            if not self.use_duration:
                c = torch.empty((B, corpus.channels, F), device=dev, dtype=torch.float32)
        vp = C.c_void_p
        rc = capi.lib().pwgb_collate_crop(vp(corpus.audio.data_ptr()), vp(xo.data_ptr()), vp(corpus.feats.data_ptr()) if c is not None else None,
                                          vp(co.data_ptr()) if co is not None else None, vp(y.data_ptr()), vp(c.data_ptr()) if c is not None else None,
                                          B, T, corpus.channels, F, vp(torch.cuda.current_stream().cuda_stream))
        capi.check(rc, "pwgb_collate_crop")
        if self.use_aux_input and self.use_duration:
            return self._runlength(corpus, co, B, F, y)
        f0 = e = None
        if self.use_aux_input and self.use_f0_and_excitation:
            if not corpus.has_f0:
                raise PwgbError("Collater(use_f0_and_excitation=True) needs a corpus with f0 and excitation")
            E = corpus.excitation_width
            e_off = np.array([corpus.e_start[i] for i in keep], dtype=np.int64) + (starts - self.aux_context_window) * E
            eo = torch.from_numpy(e_off).pin_memory().to(dev, non_blocking=True)
            f0 = torch.empty((B, 1, F), device=dev, dtype=torch.float32)
            e = torch.empty((B, 1, F * E), device=dev, dtype=torch.float32)
            # excitation as the "audio" of the gather, f0 as a 1-channel feature matrix at the rows of c
            rc = capi.lib().pwgb_collate_crop(vp(corpus.excitation.data_ptr()), vp(eo.data_ptr()), vp(corpus.f0.data_ptr()),
                                              vp(co.data_ptr()), vp(e.data_ptr()), vp(f0.data_ptr()), B, F * E, 1, F,
                                              vp(torch.cuda.current_stream().cuda_stream))
            capi.check(rc, "pwgb_collate_crop")
        if not self.use_aux_input:
            return (None, None), y  # the reference returns (l_batch, g_batch) = (None, None) here (train.py:861-876)
        inputs = (c,)
        if self.use_noise_input:
            z = torch.randn(y.shape, device=dev, generator=self.generator)  # train.py:790-792, drawn on the device
            inputs = (z,) + inputs
        if f0 is not None:
            inputs = inputs + (f0, e)
        return inputs, y

    def _runlength(self, corpus, co, B, F, y):
        L, vp, st = capi.lib(), C.c_void_p, C.c_void_p(torch.cuda.current_stream().cuda_stream)
        Cc, dev = corpus.channels, corpus.device
        runs = torch.empty(B, device=dev, dtype=torch.int64)
        rc = L.pwgb_collate_runlength(vp(corpus.feats.data_ptr()), vp(co.data_ptr()) if B else None, B, Cc, F,
                                      vp(runs.data_ptr()) if B else None, None, None, 0, 0, st)
        capi.check(rc, "pwgb_collate_runlength")
        S = int(runs.cpu().max()) if B else 0  # sizes the padded batch: one device-to-host copy of B int64
        c = torch.empty((B, Cc, S), device=dev, dtype=torch.int64)
        ds = torch.empty((B, S), device=dev, dtype=torch.int64)
        rc = L.pwgb_collate_runlength(vp(corpus.feats.data_ptr()), vp(co.data_ptr()) if B else None, B, Cc, F, None,
                                      vp(c.data_ptr()) if c.numel() else None, vp(ds.data_ptr()) if ds.numel() else None, S,
                                      int(self.pad_value), st)
        capi.check(rc, "pwgb_collate_runlength")
        return c, y, ds
