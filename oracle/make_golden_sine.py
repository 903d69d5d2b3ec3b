#!/usr/bin/env python
"""Golden vectors of the reference's SineGen and of the excitation block of bin/preprocess.py (TEST INFRASTRUCTURE), run
against the REAL reference in the build container (needs ``/root/reference``); writes ``tests/golden/sine_*.npz``.

    python oracle/make_golden_sine.py

``layers/sine.py`` is imported by path (it needs only torch and numpy).  The random draws come from torch's CPU
generator seeded with the fixture's seed; ``torch.rand``, ``torch.randn_like`` and ``torch.sin`` are wrapped during the
call, so each fixture stores the draws the reference made (``rand_ini`` before it zeroes column 0, ``n``) and the
fp32 argument of ``sin`` (``phase``), besides ``sine_waves``, ``uv`` and ``noise``.  The long fixtures store every
STRIDE-th sample of the outputs and rebuild their inputs from seeds (``oracle.ref_sine.long_case_inputs``)."""
import importlib.util
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import ref_sine  # noqa: E402
from oracle.make_golden import save  # noqa: E402

REF_SINE = "/root/reference/parallel_wavegan/layers/sine.py"
STRIDE = 16
# (name, B, T, harmonic_num, voiced_threshold, contour kwargs, stored in full)
CASES = [
    ("sine_len1", 2, 1, 2, 0, dict(), True),
    ("sine_hz_h0", 2, 2047, 0, 0, dict(below_threshold=True), True),  # one block minus one sample
    ("sine_log_h0", 2, 2048, 0, 0, dict(log=True), True),  # one block, log f0 as dumped
    ("sine_hz_h2_thr5", 2, 2049, 2, 5, dict(below_threshold=True), True),  # one block plus one
    ("sine_log_h2_thr5", 2, 6000, 2, 5, dict(log=True), True),  # log f0 under a threshold of 5: some "voiced" rows off
    ("sine_long_h0", 2, 100003, 0, 0, dict(low=60.0, high=900.0), False),
    ("sine_long_h2_log", 1, 100003, 2, 0, dict(log=True), False),
]
# egs/opencpop/voc1/conf/uhifigan.v1.yaml: 24 kHz, hop 300, win 1200
OPENCPOP = dict(sampling_rate=24000, hop_size=300, win_length=1200)


def _sine_module():
    spec = importlib.util.spec_from_file_location("reference_sine", REF_SINE)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def run_recorded(gen, f0, seed):
    """gen(f0) under torch.manual_seed(seed), recording the draws and the argument of torch.sin"""
    rec = {}
    rand, randn_like, sin = torch.rand, torch.randn_like, torch.sin

    def _rand(*a, **k):
        r = rand(*a, **k)
        rec["rand_ini"] = r.clone()
        return r

    def _randn_like(*a, **k):
        r = randn_like(*a, **k)
        rec["n"] = r.clone()
        return r

    def _sin(x, *a, **k):
        rec["phase"] = x.clone()
        return sin(x, *a, **k)

    torch.manual_seed(seed)
    torch.rand, torch.randn_like, torch.sin = _rand, _randn_like, _sin
    try:
        out = gen(f0)
    finally:
        torch.rand, torch.randn_like, torch.sin = rand, randn_like, sin
    return out, rec


def main():
    mod = _sine_module()
    for k, (name, B, T, hn, thr, contour, full) in enumerate(CASES):
        seed = 300 + 17 * k
        meta = dict(B=B, T=T, harmonic_num=hn, voiced_threshold=thr, samp_rate=24000, sine_amp=0.1, noise_std=0.003,
                    seed=seed, contour=contour, stride=None if full else STRIDE)
        f0 = np.stack([ref_sine.f0_contour(T, seed + b, **contour) for b in range(B)])
        gen = mod.SineGen(samp_rate=24000, harmonic_num=hn, voiced_threshold=thr)
        (sine, uv, noise), rec = run_recorded(gen, torch.from_numpy(f0)[..., None], seed)
        outs = dict(phase=rec["phase"], sine_waves=sine, uv=uv, noise=noise)
        if full:
            save(name, meta, f0=f0, rand_ini=rec["rand_ini"], n=rec["n"], **outs)
        else:
            f0_, ini_, n_ = ref_sine.long_case_inputs(meta)
            assert np.array_equal(f0_, f0) and np.array_equal(ini_, rec["rand_ini"].numpy()) and np.array_equal(n_, rec["n"].numpy())
            save(name, meta, **{k_: v[:, ::STRIDE] for k_, v in outs.items()})

    # the dump's excitation of one opencpop utterance: log f0 two frames longer than the mels (trimmed), as dumped
    n_frames, hop, sr = 60, OPENCPOP["hop_size"], OPENCPOP["sampling_rate"]
    seed = 400
    f0 = ref_sine.f0_contour(n_frames + 2, seed, low=120.0, high=700.0, log=True)
    extractor = mod.SineGen(samp_rate=sr)

    def preprocess_block(f0_):
        # bin/preprocess.py:425-440, with f0 one-dimensional
        f0_ = f0_[:n_frames] if len(f0_) > n_frames else np.pad(f0_, (0, n_frames - len(f0_)), mode="edge")
        extended_f0 = torch.from_numpy(f0_).reshape(1, 1, -1).repeat(1, hop, 1).reshape(1, -1, 1)
        sine_waves, _, _ = extractor(extended_f0)
        excitation = sine_waves.squeeze(0).squeeze(-1).cpu().numpy()
        return excitation[: n_frames * hop].reshape(-1, hop)

    exc, rec = run_recorded(preprocess_block, f0, seed)
    meta = dict(OPENCPOP, n_frames=n_frames, seed=seed)
    save("sine_opencpop_excitation", meta, f0=f0, rand_ini=rec["rand_ini"], n=rec["n"], phase=rec["phase"], excitation=exc)


if __name__ == "__main__":
    main()
