"""The float64 STFT oracle and the per-frame error bound the STFT kernels are held to (tests/test_gpu_spectral_exact.py).

``oracle/ref_ops.stft_power`` computes in its input's dtype, so on float64 inputs it is an exact reference of the fp32
kernels.  Here it is pinned to ``torch.stft`` in float64, and ``helpers.stft_frame_bound`` is shown to be sharp: the
framing mistakes a kernel can make (window off by one sample, replicate instead of reflect padding, a frame missing) all
exceed it by 100x or more, at every geometry of the matrix."""
import warnings

import pytest
import torch
import torch.nn.functional as F

from helpers import SPECTRAL_GEOMS, stft_frame_bound
from oracle import ref_ops, synth


def _signal(B, T, seed, scale=0.3):
    return synth.randn((B, T), seed, scale).double()  # fp32 values: the fp32 kernels see exactly these inputs


def _amp(p, eps=1e-7):
    return torch.sqrt(torch.clamp(p, min=eps))


def _worst_ratio(a, a64, bound):
    """max over (row, frame) of ||a - a64||_2 over the bins / the frame's bound."""
    return float(((a.double() - a64).norm(dim=-1) / bound).max())


@pytest.mark.parametrize("window", ["hann", None])
@pytest.mark.parametrize("n,hop,win,T", SPECTRAL_GEOMS)
def test_float64_oracle_matches_torch_stft(n, hop, win, T, window):
    x = _signal(3, T, 40 + n)
    w = torch.hann_window(win, dtype=torch.float64) if window == "hann" else None
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")  # torch.stft warns when no window is given
        s = torch.stft(x, n, hop, win, window=w, center=True, pad_mode="reflect", return_complex=True)
    p_ref = (s.real**2 + s.imag**2).transpose(1, 2)
    p = ref_ops.stft_power(x, n, hop, win, window)
    assert p.dtype == torch.float64 and p.shape == p_ref.shape == (3, 1 + T // hop, n // 2 + 1)
    assert float((p - p_ref).norm() / p_ref.norm()) < 1e-12
    # the framing itself, window included: the windowed frames carry the same energy as the spectrum (Parseval)
    fr = ref_ops.windowed_frames(x, n, hop, win, window)
    e_spec = 2 * p.sum(-1) - p[..., 0] - p[..., -1]
    assert torch.allclose(n * fr.pow(2).sum(-1), e_spec, rtol=1e-12, atol=0)


def test_float32_oracle_unchanged_by_dtype_following():
    """fp32 inputs still go through an fp32 rFFT with the window rounded to fp32 (the golden-vector parity path)."""
    x = _signal(2, 4096, 7).float()
    p = ref_ops.stft_power(x, 1024, 120, 600)
    assert p.dtype == torch.float32
    w = torch.zeros(1024, dtype=torch.float64)
    w[212:812] = ref_ops.hann_window(600)
    fr = ref_ops.windowed_frames(x, 1024, 120, 600)
    assert torch.equal(fr[0, 10], x[0, 10 * 120 - 512 : 10 * 120 + 512] * w.float())


def _mutant_frames(x, n, hop, win, pad_mode="reflect", shift=0, drop_last=False):
    """Windowed frames as a kernel with one framing mistake would form them."""
    pad = n // 2
    xp = F.pad(x.unsqueeze(1), (pad, pad), mode=pad_mode).squeeze(1)
    frames = 1 + x.shape[1] // hop
    idx = torch.arange(n).unsqueeze(0) + hop * torch.arange(frames).unsqueeze(1)
    w = torch.zeros(n + 1, dtype=torch.float64)
    left = (n - win) // 2
    w[left + shift : left + shift + win] = ref_ops.hann_window(win)
    fr = xp[:, idx] * w[:n]
    if drop_last:
        fr[:, -1] = 0.0  # the last frame never computed: its output stays zero
    return fr


@pytest.mark.parametrize("n,hop,win,T", SPECTRAL_GEOMS)
def test_frame_bound_is_sharp(n, hop, win, T):
    x, y = _signal(3, T, 10 + n), _signal(3, T, 20 + n)
    bound = stft_frame_bound(x, y, n, hop, win)
    a64 = _amp(ref_ops.stft_power(x, n, hop, win))
    assert torch.equal(_mutant_frames(x, n, hop, win), ref_ops.windowed_frames(x, n, hop, win))

    def mutant(**kw):
        return _amp(torch.fft.rfft(_mutant_frames(x, n, hop, win, **kw), dim=-1).abs() ** 2)

    ratios = {
        "window shifted by one sample": _worst_ratio(mutant(shift=1), a64, bound),
        "replicate padding": _worst_ratio(mutant(pad_mode="replicate"), a64, bound),
        "last frame dropped": _worst_ratio(mutant(drop_last=True), a64, bound),
    }
    for name, r in ratios.items():
        assert r >= 100.0, (name, r)
    # an fp32 FFT of the same frames (pocketfft, not the kernel's radix-2) stays inside the bound
    a32 = _amp(ref_ops.stft_power(x.float(), n, hop, win).double())
    assert _worst_ratio(a32, a64, stft_frame_bound(x, None, n, hop, win)) < 1.0
