"""numpy restatement of the reference's SineGen (layers/sine.py, flag_for_pulse=False) and of the excitation block of
bin/preprocess.py:420-440 (TEST INFRASTRUCTURE).

Every elementwise step is the reference's fp32 operation in its order; the two prefix sums accumulate in float64 and
round each output to float32, which is what CPU ``torch.cumsum`` does on float32.  The random draws are arguments:
``rand_ini`` (B, dim) uniform, column 0 ignored as the reference zeroes it, and ``n`` (B, T, dim) standard normal.
Also the seeded f0 contours and draws of the fixtures whose samples ``tests/golden/sine_*.npz`` does not store."""
import numpy as np

F32 = np.float32


def sine_gen(f0, harmonic_num, samp_rate, sine_amp=0.1, noise_std=0.003, voiced_threshold=0, rand_ini=None, n=None):
    """f0 (B, T) float32 at the sample rate -> dict(phase, sine_waves, uv, noise): phase (B, T, dim) is the argument of
    sin, uv (B, T, 1), the others (B, T, dim)."""
    f0 = np.asarray(f0, dtype=F32)
    dim = harmonic_num + 1
    f0h = np.empty(f0.shape + (dim,), dtype=F32)
    f0h[..., 0] = f0
    for h in range(1, dim):
        f0h[..., h] = f0 * F32(h + 1)
    rad = np.remainder(f0h / F32(samp_rate), F32(1))
    ini = np.array(rand_ini, dtype=F32, copy=True)
    ini[:, 0] = 0
    rad[:, 0, :] = rad[:, 0, :] + ini
    s1 = np.cumsum(rad.astype(np.float64), axis=1).astype(F32)
    tmp = np.remainder(s1, F32(1))
    shift = np.zeros_like(rad)
    shift[:, 1:, :] = np.where(tmp[:, 1:, :] - tmp[:, :-1, :] < 0, F32(-1), F32(-0.0))
    s2 = np.cumsum((rad + shift).astype(np.float64), axis=1).astype(F32)
    phase = (s2 * F32(2)) * F32(np.pi)
    sine = np.sin(phase) * F32(sine_amp)
    uv = (f0[..., None] > F32(voiced_threshold)).astype(F32)
    amp = uv * F32(noise_std) + (F32(1) - uv) * F32(sine_amp) / F32(3)
    noise = amp * np.asarray(n, dtype=F32)
    return dict(phase=phase, sine_waves=sine * uv + noise, uv=uv, noise=noise)


def extend_f0(f0, n_frames, hop_size):
    """bin/preprocess.py:425-434: f0 trimmed or edge-padded to n_frames, then tiled to the sample rate by
    reshape(1, 1, -1).repeat(1, hop, 1).reshape(1, -1, 1) -- sample k reads f0[k mod n_frames].  Returns (1, n_frames * hop)."""
    f0 = np.asarray(f0, dtype=F32).reshape(-1)
    f0 = f0[:n_frames] if len(f0) >= n_frames else np.pad(f0, (0, n_frames - len(f0)), mode="edge")
    return np.tile(f0, hop_size)[None, :]


def excitation(f0, n_frames, sampling_rate, hop_size, rand_ini, n):
    """bin/preprocess.py:420-440 with SineGen(samp_rate=sampling_rate) defaults: -> (n_frames, hop_size)"""
    y = sine_gen(extend_f0(f0, n_frames, hop_size), 0, sampling_rate, rand_ini=rand_ini, n=n)["sine_waves"]
    return y.reshape(-1)[: n_frames * hop_size].reshape(n_frames, hop_size)


def f0_contour(T, seed, low=80.0, high=400.0, log=False, below_threshold=False):
    """A float32 f0 track of T samples in Hz: voiced runs gliding within [low, high], unvoiced runs of 0; ``log``: log f0
    on voiced samples and 0 elsewhere, as the dumps hold it; ``below_threshold``: some runs of 0.5-5 Hz, voiced only
    for voiced_threshold 0."""
    rng = np.random.default_rng(seed)
    f0 = np.zeros(T, dtype=np.float64)
    t = 0
    voiced = bool(rng.integers(0, 2))
    while t < T:
        run = int(rng.integers(1, max(2, min(T, 4000))))
        if voiced:
            a, b = rng.uniform(low, high, 2)
            f0[t : t + run] = np.linspace(a, b, run)[: T - t]
        elif below_threshold and rng.integers(0, 2):
            f0[t : t + run] = rng.uniform(0.5, 5.0, min(run, T - t))
        t += run
        voiced = not voiced
    f0 = f0.astype(F32)
    if log:
        nz = f0 != 0
        f0[nz] = np.log(f0[nz])
    return f0


def long_case_inputs(meta):
    """(f0 (B, T), rand_ini (B, dim), n (B, T, dim)) of a fixture that stores seeds instead of samples: the f0 rows from
    ``f0_contour(T, seed + b)``, the draws as the reference made them after ``torch.manual_seed(seed)`` (torch.rand for
    rand_ini, then randn_like for n)."""
    import torch

    B, T, dim, seed = meta["B"], meta["T"], meta["harmonic_num"] + 1, meta["seed"]
    f0 = np.stack([f0_contour(T, seed + b, **meta["contour"]) for b in range(B)])
    torch.manual_seed(seed)
    rand_ini = torch.rand(B, dim).numpy()
    n = torch.randn(B, T, dim).numpy()
    return f0, rand_ini, n
