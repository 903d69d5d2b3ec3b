"""Feature extraction on the GPU (SURVEY.md 8f-4): ``logmelfilterbank`` of bin/preprocess.py:26-89 on the fused STFT /
mel kernels of the loss path (pwgb_stft_amplitude_forward + pwgb_mel_project_forward), so that analysis-synthesis
(wav -> log-mel -> vocoder) never leaves the device.  Same signature, same (#frames, num_mels) output; the reference's
own test pins this function to ``MelSpectrogram`` at 6 decimals (test/test_mel_loss.py:16-46).  ``excitation`` is the
U-Net HiFi-GAN's sine excitation of bin/preprocess.py:420-440 on ``layers.SineGen``."""
import torch

from .capi import PwgbError
from .layers import SineGen
from .losses import MelSpectrogram

_CACHE = {}


def logmelfilterbank(audio, sampling_rate, fft_size=1024, hop_size=256, win_length=None, window="hann", num_mels=80, fmin=None,
                     fmax=None, eps=1e-10, log_base=10.0):
    """audio: (T,) or (B, T) float32 CUDA tensor -> (#frames, num_mels) or (B, #frames, num_mels) log-mel features."""
    if not isinstance(audio, torch.Tensor) or not audio.is_cuda:
        raise PwgbError("logmelfilterbank: expected a CUDA tensor (no CPU fallback; the reference's librosa path is the CPU implementation)")
    key = (sampling_rate, fft_size, hop_size, win_length, window, num_mels, fmin, fmax, eps, log_base, audio.device)
    ms = _CACHE.get(key)
    if ms is None:
        ms = MelSpectrogram(fs=sampling_rate, fft_size=fft_size, hop_size=hop_size, win_length=win_length, window=window,
                            num_mels=num_mels, fmin=fmin, fmax=fmax, eps=eps, log_base=log_base).to(audio.device)
        _CACHE[key] = ms
    x = audio.reshape(1, -1) if audio.dim() == 1 else audio
    with torch.no_grad():
        mel = ms(x.float().contiguous())  # (B, num_mels, frames)
    out = mel.transpose(1, 2).contiguous()
    return out[0] if audio.dim() == 1 else out


def excitation(f0, n_frames, sampling_rate, hop_size, generator=None):
    """bin/preprocess.py:420-440 on the device: f0 (#frames,) CUDA tensor as the dump holds it (log f0 on voiced frames,
    0 on unvoiced ones: preprocess.py:131 takes the log, and this function converts nothing) -> the dump's
    ``excitation`` (n_frames, hop_size).

    f0 is trimmed to ``n_frames`` or padded with its last value.  It is then extended to the sample rate as the
    reference does, ``reshape(1, 1, -1).repeat(1, hop, 1).reshape(1, -1, 1)``: that TILES the contour, so sample k reads
    f0[k mod n_frames] rather than frame k // hop.  Trained checkpoints saw this excitation, so it is reproduced.  The
    sine comes from ``SineGen(samp_rate=sampling_rate)`` with its defaults, its random draws from ``generator``.  (On a
    (#frames, 1) array shorter than the mels, the reference's ``np.pad(f0, (0, k), mode="edge")`` also widens the second
    axis; the one-dimensional edge pad here is what that line means.)"""
    if not isinstance(f0, torch.Tensor) or not f0.is_cuda:
        raise PwgbError("excitation: expected f0 as a CUDA tensor (no CPU fallback)")
    n_frames, hop_size = int(n_frames), int(hop_size)
    f0 = f0.reshape(-1).float()
    if n_frames <= 0 or hop_size <= 0 or f0.numel() == 0:
        raise PwgbError(f"excitation: need n_frames > 0, hop_size > 0 and a non-empty f0, got {n_frames}, {hop_size}, {f0.numel()}")
    if f0.numel() >= n_frames:
        f0 = f0[:n_frames]
    else:
        f0 = torch.cat([f0, f0[-1:].expand(n_frames - f0.numel())])
    extended = f0.reshape(1, 1, -1).repeat(1, hop_size, 1).reshape(1, -1, 1)
    sine_waves, _, _ = SineGen(samp_rate=sampling_rate)(extended, generator=generator)
    return sine_waves.reshape(-1)[: n_frames * hop_size].reshape(n_frames, hop_size)
