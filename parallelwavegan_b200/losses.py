"""Host-side mirror of ``parallel_wavegan.losses`` (class names, ctor kwargs, return values).

Forward values are produced by fused sm_90a kernels (``libpwgb.so``): the STFT losses
never materialise framed / complex / magnitude tensors, the GAN losses are deterministic
two-stage reductions.  Every loss returns 0-dim CUDA tensors like the reference.
Backward: the overlap-add of the STFT adjoint (``pwgb_stft_amplitude_backward``) scatters frames with fp32
atomicAdd, so waveform gradients of the STFT / mel losses differ run to run in the last bits (like cuFFT-based
torch.stft backward); everything else is fixed-order.
"""
import numpy as np
import torch

from . import ops
from .capi import PwgbError


# --------------------------------------------------------------------------
# losses/stft_loss.py
# --------------------------------------------------------------------------


def stft(x, fft_size, hop_size, win_length, window):
    """Magnitude spectrogram (B, #frames, fft_size // 2 + 1)  (losses/stft_loss.py:16-40).
    ``window`` is a device tensor (the reference passes the registered buffer)."""
    ax, _ = ops.stft_amplitude(x, None, fft_size, hop_size, win_length, window, 1e-7)
    return ax


def _stft_loss_terms(x_mag, y_mag):
    """[sc, mag] of losses/stft_loss.py:50-61, 71-82 on materialised magnitudes -- pwgb_stft_loss_terms."""
    import ctypes as C

    from . import capi

    if x_mag.shape != y_mag.shape:
        raise PwgbError("stft loss: magnitude shapes differ")
    if torch.is_grad_enabled() and (x_mag.requires_grad or y_mag.requires_grad):
        raise PwgbError("the standalone magnitude losses have no backward kernel; train through STFTLoss / MultiResolutionSTFTLoss")
    xm, ym = ops._dev(x_mag, "x_mag"), ops._dev(y_mag, "y_mag")
    out = torch.zeros(2, device=xm.device, dtype=torch.float32)
    sums = torch.empty(3, device=xm.device, dtype=torch.float64)
    ws = torch.empty(3 * 1024, device=xm.device, dtype=torch.float64)
    rc = capi.lib().pwgb_stft_loss_terms(ops._p(xm), ops._p(ym), xm.numel(), 1.0, 0, ops._p(out), ops._p(sums), ops._p(ws), 3 * 1024, ops._stream())
    capi.check(rc, "pwgb_stft_loss_terms")
    return out


class SpectralConvergenceLoss(torch.nn.Module):
    """losses/stft_loss.py:43-61 on precomputed magnitudes (B, #frames, #bins): ||y - x||_F / ||y||_F."""

    def forward(self, x_mag, y_mag):
        return _stft_loss_terms(x_mag, y_mag)[0]


class LogSTFTMagnitudeLoss(torch.nn.Module):
    """losses/stft_loss.py:64-82 on precomputed magnitudes: mean |log y - log x|."""

    def forward(self, x_mag, y_mag):
        return _stft_loss_terms(x_mag, y_mag)[1]


class STFTLoss(torch.nn.Module):
    """losses/stft_loss.py:85-118."""

    def __init__(self, fft_size=1024, shift_size=120, win_length=600, window="hann_window"):
        super().__init__()
        self.fft_size = fft_size
        self.shift_size = shift_size
        self.win_length = win_length
        self.spectral_convergence_loss = SpectralConvergenceLoss()
        self.log_stft_magnitude_loss = LogSTFTMagnitudeLoss()
        self.register_buffer("window", getattr(torch, window)(win_length))

    def forward(self, x, y):
        return _mr_stft_loss([self], x, y)


def _check_target(y):
    if torch.is_grad_enabled() and y.requires_grad:
        raise PwgbError("spectral losses differentiate the generated signal only: the target must not require grad "
                        "(detach it)")


def _mr_stft_loss(resolutions, x, y):
    """[STFTLoss] -> (sc, mag): the fused no-grad kernels, or MrStftLossFn when x requires grad."""
    _check_target(y)
    if torch.is_grad_enabled() and x.requires_grad:
        from .autograd import MrStftLossFn

        if x.dim() == 3:
            x = x.reshape(-1, x.size(2))
            y = y.reshape(-1, y.size(2))
        out = MrStftLossFn.apply(x.contiguous(), y.contiguous(), [f.fft_size for f in resolutions],
                                 [f.shift_size for f in resolutions], [f.win_length for f in resolutions],
                                 *[f.window for f in resolutions])
        return out[0], out[1]
    out = ops.mr_stft_loss(x, y, [f.fft_size for f in resolutions], [f.shift_size for f in resolutions],
                           [f.win_length for f in resolutions], [f.window for f in resolutions])
    return out[0], out[1]


class MultiResolutionSTFTLoss(torch.nn.Module):
    """losses/stft_loss.py:121-170: one fused launch per resolution + one final reduction."""

    def __init__(self, fft_sizes=[1024, 2048, 512], hop_sizes=[120, 240, 50], win_lengths=[600, 1200, 240], window="hann_window"):
        super().__init__()
        assert len(fft_sizes) == len(hop_sizes) == len(win_lengths)
        self.stft_losses = torch.nn.ModuleList()
        for fs, ss, wl in zip(fft_sizes, hop_sizes, win_lengths):
            self.stft_losses += [STFTLoss(fs, ss, wl, window)]

    def forward(self, x, y):
        """x, y: (B, T) or (B, #subband, T) -> (sc_loss, mag_loss)."""
        return _mr_stft_loss(self.stft_losses, x, y)


# --------------------------------------------------------------------------
# losses/mel_loss.py
# --------------------------------------------------------------------------


def slaney_mel_basis(sr, n_fft, n_mels, fmin, fmax):
    """``librosa.filters.mel(sr=, n_fft=, n_mels=, fmin=, fmax=)`` (htk=False, norm="slaney"),
    which the reference calls at losses/mel_loss.py:52-58.  librosa is an un-vendored dependency;
    this is its published algorithm: Slaney mel scale, triangular filters, area normalisation."""

    def hz_to_mel(f):
        f = np.asarray(f, dtype=np.float64)
        f_sp, min_log_hz = 200.0 / 3, 1000.0
        min_log_mel, logstep = min_log_hz / f_sp, np.log(6.4) / 27.0
        return np.where(f >= min_log_hz, min_log_mel + np.log(np.maximum(f, 1e-10) / min_log_hz) / logstep, f / f_sp)

    def mel_to_hz(m):
        m = np.asarray(m, dtype=np.float64)
        f_sp, min_log_hz = 200.0 / 3, 1000.0
        min_log_mel, logstep = min_log_hz / f_sp, np.log(6.4) / 27.0
        return np.where(m >= min_log_mel, min_log_hz * np.exp(logstep * (m - min_log_mel)), f_sp * m)

    n_bins = 1 + n_fft // 2
    fftfreqs = np.linspace(0, sr / 2.0, n_bins)
    mel_f = mel_to_hz(np.linspace(hz_to_mel(fmin), hz_to_mel(fmax), n_mels + 2))
    fdiff = np.diff(mel_f)
    ramps = mel_f[:, None] - fftfreqs[None, :]
    weights = np.zeros((n_mels, n_bins))
    for i in range(n_mels):
        weights[i] = np.maximum(0, np.minimum(-ramps[i] / fdiff[i], ramps[i + 2] / fdiff[i + 1]))
    weights *= (2.0 / (mel_f[2 : n_mels + 2] - mel_f[:n_mels]))[:, None]
    return weights.astype(np.float32)


class MelSpectrogram(torch.nn.Module):
    """losses/mel_loss.py:15-110."""

    def __init__(self, fs=22050, fft_size=1024, hop_size=256, win_length=None, window="hann", num_mels=80, fmin=80,
                 fmax=7600, center=True, normalized=False, onesided=True, eps=1e-10, log_base=10.0):
        super().__init__()
        if not center or normalized or not onesided:
            raise PwgbError("MelSpectrogram: only center=True, normalized=False, onesided=True has an sm_90a kernel")
        self.fft_size = fft_size
        self.win_length = fft_size if win_length is None else win_length
        self.hop_size = hop_size
        self.center, self.normalized, self.onesided = center, normalized, onesided
        if window is not None and not hasattr(torch, f"{window}_window"):
            raise ValueError(f"{window} window is not implemented")
        self.window = window
        self.eps = eps
        fmin = 0 if fmin is None else fmin
        fmax = fs / 2 if fmax is None else fmax
        melmat = slaney_mel_basis(fs, fft_size, num_mels, fmin, fmax)
        self.register_buffer("melmat", torch.from_numpy(melmat.T.copy()).float())
        self.log_base = log_base
        if log_base is None:
            self._log_scale = 1.0
        elif log_base == 2.0:
            self._log_scale = 1.0 / np.log(2.0)
        elif log_base == 10.0:
            self._log_scale = 1.0 / np.log(10.0)
        else:
            raise ValueError(f"log_base: {log_base} is not supported.")

    def _window(self, x):
        if self.window is None:
            return torch.ones(self.win_length, dtype=x.dtype, device=x.device)
        return getattr(torch, f"{self.window}_window")(self.win_length, dtype=x.dtype, device=x.device)

    def forward(self, x):
        """(B, T) or (B, 1, T) -> (B, #mels, #frames)."""
        if x.dim() == 3:
            x = x.reshape(-1, x.size(2))
        ax, _ = ops.stft_amplitude(x, None, self.fft_size, self.hop_size, self.win_length, self._window(x), self.eps)
        mel, _ = ops.mel_project(ax, None, self.melmat, self.eps, self._log_scale, want_mel=True)
        return mel


class MelSpectrogramLoss(torch.nn.Module):
    """losses/mel_loss.py:113-165: both signals share one FFT per frame; L1 fused into the projection."""

    def __init__(self, fs=22050, fft_size=1024, hop_size=256, win_length=None, window="hann", num_mels=80, fmin=80,
                 fmax=7600, center=True, normalized=False, onesided=True, eps=1e-10, log_base=10.0):
        super().__init__()
        self.mel_spectrogram = MelSpectrogram(fs=fs, fft_size=fft_size, hop_size=hop_size, win_length=win_length,
                                              window=window, num_mels=num_mels, fmin=fmin, fmax=fmax, center=center,
                                              normalized=normalized, onesided=onesided, eps=eps, log_base=log_base)

    def forward(self, y_hat, y):
        m = self.mel_spectrogram
        _check_target(y)
        if y_hat.dim() == 3:
            y_hat = y_hat.reshape(-1, y_hat.size(2))
            y = y.reshape(-1, y.size(2))
        if torch.is_grad_enabled() and y_hat.requires_grad:
            from .autograd import MelLossFn

            return MelLossFn.apply(y_hat.contiguous(), y.contiguous(), m.melmat, m._window(y_hat), m.fft_size, m.hop_size,
                                   m.win_length, m.eps, m._log_scale)[0]
        ax, ay = ops.stft_amplitude(y_hat, y, m.fft_size, m.hop_size, m.win_length, m._window(y_hat), m.eps)
        _, loss = ops.mel_project(ax, ay, m.melmat, m.eps, m._log_scale, want_mel=False, want_loss=True)
        return loss[0]


# --------------------------------------------------------------------------
# losses/adversarial_loss.py, losses/feat_match_loss.py
# --------------------------------------------------------------------------


def _last(o):
    return o[-1] if isinstance(o, (tuple, list)) else o


class GeneratorAdversarialLoss(torch.nn.Module):
    """losses/adversarial_loss.py:12-58."""

    def __init__(self, average_by_discriminators=True, loss_type="mse"):
        super().__init__()
        self.average_by_discriminators = average_by_discriminators
        assert loss_type in ["mse", "hinge"], f"{loss_type} is not supported."
        self.loss_type = loss_type

    def _term(self, x, weight, out, first):
        if self.loss_type == "mse":
            return ops.reduce_mean("mse_const", x, c=1.0, weight=weight, out=out, accumulate=not first)
        return ops.reduce_mean("linear", x, s=-1.0, weight=weight, out=out, accumulate=not first)

    def forward(self, outputs):
        if isinstance(outputs, (tuple, list)):
            n = len(outputs)
            w = 1.0 / n if self.average_by_discriminators else 1.0
            out = None
            for i, o in enumerate(outputs):
                out = self._term(_last(o), w, out, i == 0)
            return out[0]
        return self._term(outputs, 1.0, None, True)[0]


class DiscriminatorAdversarialLoss(torch.nn.Module):
    """losses/adversarial_loss.py:61-123."""

    def __init__(self, average_by_discriminators=True, loss_type="mse"):
        super().__init__()
        self.average_by_discriminators = average_by_discriminators
        assert loss_type in ["mse", "hinge"], f"{loss_type} is not supported."
        self.loss_type = loss_type

    def _real(self, x, w, out, first):
        if self.loss_type == "mse":
            return ops.reduce_mean("mse_const", x, c=1.0, weight=w, out=out, accumulate=not first)
        return ops.reduce_mean("hinge", x, c=1.0, s=1.0, weight=w, out=out, accumulate=not first)

    def _fake(self, x, w, out, first):
        if self.loss_type == "mse":
            return ops.reduce_mean("mse_const", x, c=0.0, weight=w, out=out, accumulate=not first)
        return ops.reduce_mean("hinge", x, c=1.0, s=-1.0, weight=w, out=out, accumulate=not first)

    def forward(self, outputs_hat, outputs):
        if isinstance(outputs, (tuple, list)):
            n = len(outputs)
            w = 1.0 / n if self.average_by_discriminators else 1.0
            real = fake = None
            for i, (oh, o) in enumerate(zip(outputs_hat, outputs)):
                real = self._real(_last(o), w, real, i == 0)
                fake = self._fake(_last(oh), w, fake, i == 0)
            return real[0], fake[0]
        return self._real(outputs, 1.0, None, True)[0], self._fake(outputs_hat, 1.0, None, True)[0]


class FeatureMatchLoss(torch.nn.Module):
    """losses/feat_match_loss.py:12-54."""

    def __init__(self, average_by_layers=True, average_by_discriminators=True, include_final_outputs=False):
        super().__init__()
        self.average_by_layers = average_by_layers
        self.average_by_discriminators = average_by_discriminators
        self.include_final_outputs = include_final_outputs

    def forward(self, feats_hat, feats):
        nd = len(feats)
        wd = 1.0 / nd if self.average_by_discriminators else 1.0
        out = None
        first = True
        for fh, f in zip(feats_hat, feats):
            if not self.include_final_outputs:
                fh, f = fh[:-1], f[:-1]
            wl = 1.0 / len(f) if self.average_by_layers else 1.0
            for a, b in zip(fh, f):
                out = ops.reduce_mean("l1", a, b.detach(), weight=wd * wl, out=out, accumulate=not first)
                first = False
        return out[0]


# --------------------------------------------------------------------------
# losses/duration_prediction_loss.py
# --------------------------------------------------------------------------
class DurationPredictorLoss(torch.nn.Module):
    """losses/duration_prediction_loss.py:15-52: MSELoss between the log-domain prediction and log(targets + offset)
    over all (B, T), padding included (pwgb_duration_loss_forward)."""

    def __init__(self, offset=1.0, reduction="mean"):
        super().__init__()
        if reduction != "mean":
            raise PwgbError(f"DurationPredictorLoss(reduction={reduction!r}) has no sm_90a kernel (mean only)")
        self.offset = offset

    def forward(self, outputs, targets):
        return ops.duration_loss(outputs, targets, self.offset)[0]


# --------------------------------------------------------------------------
# criterion["mse"] of the VQ-VAE recipes (bin/train.py:1384-1451, 210-211)
# --------------------------------------------------------------------------
class MSELoss(torch.nn.Module):
    """torch.nn.MSELoss() (mean reduction) between two tensors of the same size -- pwgb_reduce_mean_forward mode 4,
    with gradients to both operands."""

    def forward(self, x, y):
        if x.shape != y.shape:
            raise PwgbError(f"MSELoss: shapes {tuple(x.shape)} and {tuple(y.shape)} differ")
        return ops.reduce_mean("mse", x, y)[0]
