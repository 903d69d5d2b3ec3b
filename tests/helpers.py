"""Shared helpers for parity tests (tolerances are stated here once)."""
import json
import math
import os

import numpy as np
import torch

from oracle import ref_ops, synth
from oracle.ref_ops import fold_weight_norm

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")

# north_star: "outputs match the reference PyTorch forward ... to <= 1e-3 rel fp32"
REL_TOL = 1e-3
# oracle-vs-reference on the same CPU ATen ops: only summation-order noise is allowed
ORACLE_TOL = 2e-5


def rel_l2(a, b):
    a = torch.as_tensor(a).double().reshape(-1)
    b = torch.as_tensor(b).double().reshape(-1)
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def max_abs_over_peak(a, b):
    a = torch.as_tensor(a).double()
    b = torch.as_tensor(b).double()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def load_golden(name):
    z = np.load(os.path.join(GOLD, name + ".npz"), allow_pickle=False)
    meta = json.loads(str(z["meta"]))
    arrays = {k: torch.from_numpy(z[k]) for k in z.files if k != "meta"}
    return meta, arrays


def golden_weights(meta):
    """Regenerate the synthetic checkpoint of a fixture (raw, with weight_g/weight_v)
    and verify the checksum recorded when the reference produced the golden output."""
    sd = synth.synth_state_dict([(k, tuple(s)) for k, s in meta["spec"]], meta["seed"], meta["gain"])
    cs = synth.checksum(sd)
    assert abs(cs - meta["checksum"]) <= 1e-9 * abs(meta["checksum"]), "synthetic weights drifted from the fixture"
    return sd


def golden_effective_weights(meta):
    return fold_weight_norm(golden_weights(meta))


def flatten_outs(outs):
    """(nested) list of feature maps -> [(name, tensor)] with the naming of oracle/make_golden.summarize."""
    flat = []
    if isinstance(outs, torch.Tensor):
        outs = [outs]
    for i, o in enumerate(outs):
        if isinstance(o, (list, tuple)):
            for j, t in enumerate(o):
                flat.append((f"o{i}_{j}", t))
        else:
            flat.append((f"o{i}", o))
    return flat


def check_fingerprint(outs, meta, g, tol):
    """Compare feature maps with the golden fingerprint (shape, sum / L2 norm in float64, head, tail)."""
    flat = flatten_outs(outs)
    assert [(n, list(t.shape)) for n, t in flat] == [(n, list(s)) for n, s in meta["shapes"]]
    for n, t in flat:
        t = t.detach().cpu()
        v = t.reshape(-1).double()
        ssum, snorm = float(g[n + "_stat"][0]), float(g[n + "_stat"][1])
        assert abs(float(v.norm()) - snorm) <= tol * snorm, (n, float(v.norm()), snorm)
        assert abs(float(v.sum()) - ssum) <= tol * max(snorm * v.numel() ** 0.5, 1e-12), (n, float(v.sum()), ssum)
        assert rel_l2(t.reshape(-1)[:96], g[n + "_head"]) < tol, n
        assert rel_l2(t.reshape(-1)[-96:], g[n + "_tail"]) < tol, n


# STFT geometries (n_fft, hop, win_length, T) where framing and FFT kernels go wrong: the shortest admitted T = n/2 + 1,
# odd n - win, hops that do not divide T or exceed n, fewer bins than a warp (n = 16) and the largest n (4096).
SPECTRAL_GEOMS = [
    (16, 4, 16, 9),
    (32, 7, 25, 100),
    (64, 80, 41, 300),
    (512, 50, 240, 2000),
    (1024, 120, 600, 8192),
    (1024, 256, 1024, 8192),
    (2048, 300, 1200, 8193),
    (4096, 480, 2400, 9000),
]


def stft_frame_bound(x, y, n_fft, hop, win_length, window="hann", kappa=1.0):
    """Per-frame bound on the fp32 STFT amplitude error: over the bins of frame f,
    ||a - a64||_2 <= kappa * log2(n) * 2^-24 * sqrt(n) * (||w x_f||_2 + ||w y_f||_2),
    the forward error of a radix-2 FFT of length n on z = w (x + i y).  ``y`` is the signal that shares x's FFT
    (None when x runs alone): in the pair transform each signal's rounding error scales with both energies.
    x, y: (B, T) -> (B, frames) float64."""

    def energy(s):
        return ref_ops.windowed_frames(s.double(), n_fft, hop, win_length, window).norm(dim=-1)

    e = energy(x) + (energy(y) if y is not None else 0.0)
    return kappa * math.log2(n_fft) * 2.0**-24 * math.sqrt(n_fft) * e


def conditioning_tolerances(grad_fn, leaves, rel_eps=1e-6, k=4.0, floor=1e-3, seed=1234):
    """Per-tensor tolerance for gradient parity that follows the CONDITIONING of the computation instead of a
    hand-picked constant.  ``grad_fn(leaves) -> {name: grad}`` runs the CPU oracle with torch autograd.  It is run
    twice: on ``leaves`` and on ``leaves * (1 + rel_eps * N(0,1))`` -- a perturbation of the size of fp32 input rounding.
    Whatever change that produces in a gradient tensor (LeakyReLU / clamp masks flipping, log of small magnitudes ...)
    is a change ANY fp32 implementation with a different rounding order may show; the tolerance is
    ``max(floor, k * observed relative change)``.  Returns (baseline grads, {name: tol}, {name: observed change})."""
    base = grad_fn(leaves)
    g = torch.Generator().manual_seed(seed)
    pert = {n: (t.detach() * (1.0 + rel_eps * torch.randn(t.shape, generator=g))) for n, t in leaves.items()}
    moved = grad_fn(pert)
    tol, obs = {}, {}
    for n, gb in base.items():
        d = rel_l2(moved[n], gb)
        obs[n] = d
        tol[n] = max(floor, k * d)
    return base, tol, obs
