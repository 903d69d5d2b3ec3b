"""GPU: the STFT and mel loss kernels (csrc/stft.cu) and their adjoints against the float64 oracle.

``oracle/ref_ops`` computes the STFT, the MR-STFT loss and the mel loss in float64 when given float64 inputs, so every
kernel output here is compared with an exact value of the same operation:
* amplitudes, per frame, within ``helpers.stft_frame_bound`` (the forward error of an fp32 radix-2 FFT, kappa = 1),
  x alone and x sharing its FFT with y, at the geometries of ``helpers.SPECTRAL_GEOMS``;
* MR-STFT and mel loss values within 2e-5 relative (log-mel within 1e-4 in natural-log units), the fused no-grad path and
  the autograd path within 1e-6 of each other, repeated calls bit-identical;
* waveform gradients within ``helpers.conditioning_tolerances`` of float64 autograd, over the whole signal and, each on
  its own, over its first and last n/2 samples, where the adjoint folds back through the reflect padding.
The signals include a 1000:1 level ratio between the two signals of the pair transform and a row with a stretch of
exact zeros (the clamps of the forward and the clamp mask of the adjoint)."""
import math

import pytest
import torch

from helpers import SPECTRAL_GEOMS, conditioning_tolerances, rel_l2, stft_frame_bound
from oracle import ref_ops, synth

pytestmark = pytest.mark.gpu

EPS = 1e-7  # stft_loss.py clamp
KINDS = ["matched", "x1000", "y1000", "zeros", "same"]
GRAD_KINDS = ["matched", "x1000", "y1000", "zeros"]  # x == y: sign(log ym - log xm) is rounding noise in any fp32 pair

MR_SETS = {
    "default": ([1024, 2048, 512], [120, 240, 50], [600, 1200, 240]),
    "kss_melgan_v3": ([2048, 4096, 1024], [240, 480, 100], [1200, 2400, 480]),  # egs/kss/voc1/conf/melgan.v3.yaml
    "small": ([64, 128, 256], [16, 32, 64], [64, 128, 256]),
}

MEL_CONFIGS = {
    "v1": dict(fs=22050, fft_size=1024, hop_size=256, fmin=0, fmax=11025, log_base=None),
    "default": dict(),
    "24k": dict(fs=24000, fft_size=2048, hop_size=300, win_length=1200, fmin=0, fmax=12000),
    "n512_40": dict(fft_size=512, hop_size=128, num_mels=40),
    "n256_empty": dict(fs=22050, fft_size=256, hop_size=64, num_mels=80, fmin=80, fmax=7600),
    "no_window": dict(window=None),
    "log2": dict(log_base=2.0),
}
MEL_DEFAULTS = dict(fs=22050, fft_size=1024, hop_size=256, win_length=None, window="hann", num_mels=80, fmin=80, fmax=7600,
                    eps=1e-10, log_base=10.0)


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    import __graft_entry__

    __graft_entry__.build()
    return torch.device("cuda:0")


def _signals(kind, B, T, n, seed):
    """(x, y) fp32 on the CPU.  x1000 / y1000: one signal at 1000x the level of the other; zeros: row 0 of x holds a
    stretch of exact zeros longer than a frame (the whole row when T is that short); same: y is x."""
    x = synth.randn((B, T), seed, 0.3)
    y = synth.randn((B, T), seed + 1, 0.3)
    if kind == "x1000":
        y = y * 1e-3
    elif kind == "y1000":
        x = x * 1e-3
    elif kind == "zeros":  # 2n samples hold a whole frame's window at every geometry of the matrix (hop <= 2n - win)
        L = min(T, 2 * n)
        s = (T - L) // 2
        x[0, s : s + L] = 0.0
        # then n samples at 1e-7: frames whose bins sit below both clamps without being exactly zero, so a clamp mask
        # that let them through would show (exact zeros give X = 0 and no gradient either way)
        q = min(n, T - s - L)
        x[0, s + L : s + L + q] *= 1e-7 / 0.3
    elif kind == "same":
        y = x.clone()
    return x, y


# ---------------------------------------------------------------------------------------------------- amplitudes
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("n,hop,win,T", SPECTRAL_GEOMS)
def test_stft_amplitude_within_fft_bound(dev, n, hop, win, T, B, kind):
    """||a - a64|| per frame <= log2(n) 2^-24 sqrt(n) (||w x_f|| + ||w y_f||), x alone and x paired with y."""
    from parallelwavegan_b200 import ops

    x, y = _signals(kind, B, T, n, 1000 + n + B)
    x64, y64 = x.double(), y.double()
    w = torch.hann_window(win)  # the oracle multiplies by the same fp32 values: near its ends it is 1e-3 off Hann
    # exact |STFT|, clamped from below at the amplitude the kernel's fp32 clamp produces, sqrtf(fp32(1e-7)): in quiet
    # frames the rounding of that constant is larger than the FFT bound
    clamp32 = float(torch.tensor(EPS, dtype=torch.float32).sqrt())
    ax64 = ref_ops.stft_power(x64, n, hop, win, w).sqrt().clamp(min=clamp32)
    ay64 = ref_ops.stft_power(y64, n, hop, win, w).sqrt().clamp(min=clamp32)
    worst = {}
    a, none = ops.stft_amplitude(x.to(dev), None, n, hop, win, w.to(dev), EPS)
    assert none is None and a.shape == ax64.shape
    b_alone = stft_frame_bound(x64, None, n, hop, win)
    assert bool((b_alone[0] == 0).any()) == (kind == "zeros")  # the zero stretch silences whole frames of x
    worst["x alone"] = _kappa(a, ax64, b_alone)
    ax, ay = ops.stft_amplitude(x.to(dev), y.to(dev), n, hop, win, w.to(dev), EPS)
    b_pair = stft_frame_bound(x64, y64, n, hop, win)
    worst["x paired"] = _kappa(ax, ax64, b_pair)
    worst["y paired"] = _kappa(ay, ay64, b_pair)
    print(f"[kappa] n={n} hop={hop} win={win} T={T} B={B} {kind}: " + " ".join(f"{k}={v:.3f}" for k, v in worst.items()))
    for k, v in worst.items():
        assert v <= 1.0, (k, v)


def _kappa(a, a64, bound):
    """Worst ratio of a frame's amplitude error to its bound.  A frame whose windowed input is all zeros has bound 0:
    every bin must be exactly the fp32 clamp value there."""
    a = a.cpu()
    silent = bound == 0
    if bool(silent.any()):
        assert torch.equal(a[silent].double(), a64[silent])
    err = (a.double() - a64).norm(dim=-1)
    return float((err[~silent] / bound[~silent]).max()) if bool((~silent).any()) else 0.0


# ---------------------------------------------------------------------------------------------------- MR-STFT value
def _mr(dev, name):
    from parallelwavegan_b200 import losses

    return losses.MultiResolutionSTFTLoss(*MR_SETS[name]).to(dev)


def _mr64(mr, x, y):
    """The float64 MR-STFT loss with the module's own (fp32) windows."""
    fs, hs, wls = (list(v) for v in zip(*[(s.fft_size, s.shift_size, s.win_length) for s in mr.stft_losses]))
    return ref_ops.mr_stft_loss(x, y, fs, hs, wls, [s.window for s in mr.stft_losses])


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("name", list(MR_SETS))
def test_mr_stft_value_both_paths(dev, name, kind):
    fs, hs, wls = MR_SETS[name]
    x, y = _signals(kind, 3, 9000, max(fs), 2000 + len(name))
    mr = _mr(dev, name)
    sc64, mag64 = _mr64(mr, x.double(), y.double())
    xd, yd = x.to(dev), y.to(dev)
    with torch.no_grad():
        sc0, mag0 = mr(xd, yd)
        sc1, mag1 = mr(xd, yd)
    assert torch.equal(sc0, sc1) and torch.equal(mag0, mag1)
    xg = xd.clone().requires_grad_(True)
    scg, magg = mr(xg, yd)
    assert scg.requires_grad and magg.requires_grad
    scg2, magg2 = mr(xg, yd)
    assert torch.equal(scg, scg2) and torch.equal(magg, magg2)
    if kind == "same":
        for v in (sc0, mag0, scg, magg):
            assert float(v) < 1e-6
        return
    for v, r in ((sc0, sc64), (mag0, mag64), (scg, sc64), (magg, mag64)):
        assert abs(float(v) - float(r)) <= 2e-5 * abs(float(r)), (float(v), float(r))
    for a, b in ((sc0, scg), (mag0, magg)):
        assert abs(float(a) - float(b)) <= 1e-6 * abs(float(b)), (float(a), float(b))


def test_mr_stft_subband_input(dev):
    """(B, C, T) input: every subband is a row of its own, on both paths and in the gradient."""
    x, y = _signals("matched", 6, 2048, 256, 2100)
    x, y = x.view(2, 3, -1), y.view(2, 3, -1)
    mr = _mr(dev, "small")
    sc64, mag64 = _mr64(mr, x.double(), y.double())
    with torch.no_grad():
        sc, mag = mr(x.to(dev), y.to(dev))
    xg = x.to(dev).requires_grad_(True)
    scg, magg = mr(xg, y.to(dev))
    (scg + magg).backward()
    for v, r in ((sc, sc64), (mag, mag64), (scg, sc64), (magg, mag64)):
        assert abs(float(v) - float(r)) <= 2e-5 * abs(float(r))
    assert xg.grad.shape == x.shape
    y64 = y.double()

    def grad_fn(lv):
        xr = lv["x"].clone().requires_grad_(True)
        (g,) = torch.autograd.grad(sum(_mr64(mr, xr, y64)), xr)
        return _split(g, 128)

    _check_grad(xg.grad.cpu().double(), grad_fn, x.double(), 128, "subband (2, 3, T)")


# ---------------------------------------------------------------------------------------------------- MR-STFT gradient
def _check_grad(dg, grad_fn, x64, h, label):
    """dg: the kernel's dx; grad_fn: float64 autograd -> {"all", "head", "tail"} with head / tail the first / last
    h samples of every row.  Each is held to its own conditioning tolerance (rel_eps 1e-6, floor 2e-5)."""
    base, tol, obs = conditioning_tolerances(grad_fn, {"x": x64}, rel_eps=1e-6, floor=2e-5)
    got = {"all": dg, "head": dg[..., :h], "tail": dg[..., -h:]}
    errs = {k: rel_l2(got[k], base[k]) for k in base}
    print(f"[grad] {label}: " + " ".join(f"{k}={errs[k]:.2e}/{tol[k]:.2e}" for k in errs))
    for k in errs:
        assert errs[k] <= tol[k], (k, errs[k], tol[k], obs[k])


def _split(g, h):
    return {"all": g, "head": g[..., :h], "tail": g[..., -h:]}


TERMS = {"sc": lambda sc, mag: sc, "mag": lambda sc, mag: mag, "sc+mag": lambda sc, mag: sc + mag}


@pytest.mark.parametrize("term", list(TERMS))
@pytest.mark.parametrize("kind", GRAD_KINDS)
@pytest.mark.parametrize("name", list(MR_SETS))
def test_mr_stft_gradient(dev, name, kind, term):
    fs, hs, wls = MR_SETS[name]
    x, y = _signals(kind, 3, 9000, max(fs), 3000 + len(name))
    h = max(fs) // 2
    f = TERMS[term]
    mr = _mr(dev, name)
    xg = x.to(dev).requires_grad_(True)
    f(*mr(xg, y.to(dev))).backward()
    y64 = y.double()

    def grad_fn(lv):
        xr = lv["x"].clone().requires_grad_(True)
        (g,) = torch.autograd.grad(f(*_mr64(mr, xr, y64)), xr)
        return _split(g, h)

    _check_grad(xg.grad.cpu().double(), grad_fn, x.double(), h, f"{name} {kind} {term}")


def test_single_resolution_stft_loss_gradient(dev):
    """STFTLoss on its own differentiates x (it used to return a loss detached from x)."""
    from parallelwavegan_b200 import losses

    x, y = _signals("matched", 2, 4000, 1024, 3100)
    st = losses.STFTLoss(1024, 120, 600).to(dev)
    xg = x.to(dev).requires_grad_(True)
    sc, mag = st(xg, y.to(dev))
    (sc + mag).backward()
    y64 = y.double()

    def grad_fn(lv):
        xr = lv["x"].clone().requires_grad_(True)
        (g,) = torch.autograd.grad(sum(ref_ops.mr_stft_loss(xr, y64, (1024,), (120,), (600,), [st.window])), xr)
        return _split(g, 512)

    _check_grad(xg.grad.cpu().double(), grad_fn, x.double(), 512, "STFTLoss")


# ---------------------------------------------------------------------------------------------------- mel
def _mel_kw(name):
    return dict(MEL_DEFAULTS, **MEL_CONFIGS[name])


def _mel_ref_kw(kw, ms, dev):
    """Oracle kwargs for a MelSpectrogram ``ms``, with the fp32 window it computes on the device."""
    return dict(fft_size=ms.fft_size, hop_size=ms.hop_size, win_length=ms.win_length, eps=kw["eps"],
                log_base=kw["log_base"], window=ms._window(torch.empty(0, device=dev)))


def _melmat64(m):
    return m.melmat.detach().cpu().double()  # the kernel's fp32 bank, exactly


def test_mel_bank_with_empty_filters():
    """22050 Hz, n = 256, 80 mels over 80-7600 Hz: the bins are 86 Hz apart, so the narrowest low filters catch no bin."""
    from parallelwavegan_b200 import losses

    bank = losses.slaney_mel_basis(22050, 256, 80, 80, 7600)
    assert int((abs(bank).sum(1) == 0).sum()) == 4


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("name", list(MEL_CONFIGS))
def test_mel_value_both_paths(dev, name, kind):
    from parallelwavegan_b200 import losses

    kw = _mel_kw(name)
    x, y = _signals(kind, 3, 8193, kw["fft_size"], 4000 + len(name))
    ms = losses.MelSpectrogram(**kw).to(dev)
    ml = losses.MelSpectrogramLoss(**kw).to(dev)
    mm = _melmat64(ms)
    rkw = _mel_ref_kw(kw, ms, dev)
    ln_base = 1.0 if kw["log_base"] is None else math.log(kw["log_base"])
    xd, yd = x.to(dev), y.to(dev)
    with torch.no_grad():
        m0, m1 = ms(xd), ms(xd)
        l0, l1 = ml(xd, yd), ml(xd, yd)
    assert torch.equal(m0, m1) and torch.equal(l0, l1)
    m64 = ref_ops.mel_spectrogram(x.double(), mm, **rkw)
    assert m0.shape == m64.shape
    assert float((m0.cpu().double() - m64).abs().max()) * ln_base <= 1e-4
    xg = xd.clone().requires_grad_(True)
    lg, lg2 = ml(xg, yd), ml(xg, yd)
    assert lg.requires_grad and torch.equal(lg, lg2)
    if kind == "same":
        assert float(l0) < 1e-6 and float(lg) < 1e-6
        return
    l64 = float(ref_ops.mel_loss(x.double(), y.double(), mm, **rkw))
    for v in (l0, lg):
        assert abs(float(v) - l64) <= 2e-5 * l64, (float(v), l64)
    assert abs(float(l0) - float(lg)) <= 1e-6 * l64


@pytest.mark.parametrize("kind", GRAD_KINDS)
@pytest.mark.parametrize("name", list(MEL_CONFIGS))
def test_mel_gradient(dev, name, kind):
    from parallelwavegan_b200 import losses

    kw = _mel_kw(name)
    n = kw["fft_size"]
    x, y = _signals(kind, 3, 8193, n, 5000 + len(name))
    ml = losses.MelSpectrogramLoss(**kw).to(dev)
    mm = _melmat64(ml.mel_spectrogram)
    rkw = _mel_ref_kw(kw, ml.mel_spectrogram, dev)
    xg = x.to(dev).requires_grad_(True)
    ml(xg, y.to(dev)).backward()
    y64 = y.double()

    def grad_fn(lv):
        xr = lv["x"].clone().requires_grad_(True)
        (g,) = torch.autograd.grad(ref_ops.mel_loss(xr, y64, mm, **rkw), xr)
        return _split(g, n // 2)

    _check_grad(xg.grad.cpu().double(), grad_fn, x.double(), n // 2, f"mel {name} {kind}")


# ---------------------------------------------------------------------------------------------------- errors
def _both_paths(dev, loss, x, y):
    """The no-grad (fused) call and the autograd call of one loss module."""
    from parallelwavegan_b200.capi import PwgbError

    with pytest.raises(PwgbError):
        with torch.no_grad():
            loss(x.to(dev), y.to(dev))
    with pytest.raises(PwgbError):
        loss(x.to(dev).requires_grad_(True), y.to(dev))


def test_errors_length_at_half_fft(dev):
    """T = n/2 leaves no sample for the reflect padding to mirror; torch.stft rejects it too."""
    from parallelwavegan_b200 import losses

    x, y = _signals("matched", 2, 512, 1024, 6000)
    with pytest.raises(RuntimeError):
        torch.stft(x, 1024, 120, 600, window=torch.hann_window(600), center=True, pad_mode="reflect", return_complex=True)
    _both_paths(dev, losses.MultiResolutionSTFTLoss([1024], [120], [600]).to(dev), x, y)
    _both_paths(dev, losses.MelSpectrogramLoss(fft_size=1024, hop_size=256).to(dev), x, y)
    x, y = _signals("matched", 2, 513, 1024, 6001)  # the shortest admitted length runs
    with torch.no_grad():
        losses.MultiResolutionSTFTLoss([1024], [120], [600]).to(dev)(x.to(dev), y.to(dev))


def test_errors_non_power_of_two_fft(dev):
    """The MB-MelGAN subband resolutions (egs/*/voc1/conf/multi_band_melgan.*.yaml) have no radix-2 FFT."""
    from parallelwavegan_b200 import losses

    x, y = _signals("matched", 4, 4096, 683, 6100)
    _both_paths(dev, losses.MultiResolutionSTFTLoss([384, 683, 171], [30, 60, 10], [150, 300, 60]).to(dev), x, y)
    _both_paths(dev, losses.MelSpectrogramLoss(fft_size=384, hop_size=96).to(dev), x, y)


def test_errors_target_requires_grad(dev):
    """Both losses differentiate the generated signal only; a target that requires grad is refused, not dropped."""
    from parallelwavegan_b200 import losses
    from parallelwavegan_b200.capi import PwgbError

    x, y = _signals("matched", 2, 4096, 1024, 6200)
    for loss in (losses.MultiResolutionSTFTLoss().to(dev), losses.MelSpectrogramLoss().to(dev)):
        yg = y.to(dev).requires_grad_(True)
        for xx in (x.to(dev), x.to(dev).requires_grad_(True)):
            with pytest.raises(PwgbError):
                loss(xx, yg)
        with torch.no_grad():  # no graph, nothing to drop
            loss(x.to(dev), yg)
