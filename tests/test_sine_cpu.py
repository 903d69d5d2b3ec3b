"""SineGen and the U-Net HiFi-GAN decoder without a GPU: the numpy restatement ``oracle/ref_sine.py`` against the
reference's goldens (the phase, uv and noise bit for bit, the sine within 2 fp32 ulp x sine_amp), the refusals of
``layers.SineGen`` / ``ops.sine_gen``, the decoder's host logic for excitations, and the codegen of ``sine.cu``."""
import json
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from oracle import ref_sine

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
SINE_CASES = ["sine_len1", "sine_hz_h0", "sine_log_h0", "sine_hz_h2_thr5", "sine_log_h2_thr5", "sine_long_h0", "sine_long_h2_log"]
EPS = float(np.finfo(np.float32).eps)


def _golden(name):
    z = np.load(os.path.join(GOLD, name + ".npz"), allow_pickle=False)
    return json.loads(str(z["meta"])), {k: z[k] for k in z.files if k != "meta"}


def sine_inputs(meta, g):
    """(f0 (B, T), rand_ini (B, dim), n (B, T, dim)) of a SineGen fixture, stored or rebuilt from its seeds"""
    if meta["stride"]:
        return ref_sine.long_case_inputs(meta)
    return g["f0"], g["rand_ini"], g["n"]


@pytest.mark.parametrize("name", SINE_CASES)
def test_ref_sine_matches_reference(name):
    meta, g = _golden(name)
    f0, rand_ini, n = sine_inputs(meta, g)
    r = ref_sine.sine_gen(f0, meta["harmonic_num"], meta["samp_rate"], meta["sine_amp"], meta["noise_std"], meta["voiced_threshold"],
                          rand_ini, n)
    s = meta["stride"] or 1
    for k in ("phase", "uv", "noise"):
        assert np.array_equal(r[k][:, ::s].view(np.uint32), g[k].view(np.uint32)), k
    assert np.abs(r["sine_waves"][:, ::s] - g["sine_waves"]).max() <= 2 * EPS * meta["sine_amp"]
    if name == "sine_hz_h2_thr5":  # the threshold case has samples 0 < f0 <= 5 that uv turns off
        f0_ = np.asarray(f0)
        assert ((f0_ > 0) & (f0_ <= 5)).any() and (g["uv"][..., 0][(f0_ > 0) & (f0_ <= 5)] == 0).all()


def test_ref_excitation_matches_preprocess():
    meta, g = _golden("sine_opencpop_excitation")
    assert len(g["f0"]) > meta["n_frames"]  # the dump's f0 is trimmed to the mels
    e = ref_sine.excitation(g["f0"], meta["n_frames"], meta["sampling_rate"], meta["hop_size"], g["rand_ini"], g["n"])
    assert e.shape == (meta["n_frames"], meta["hop_size"])
    assert np.abs(e - g["excitation"]).max() <= 2 * EPS * 0.1
    # the extension tiles the contour: sample k reads f0[k mod n_frames]
    ext = ref_sine.extend_f0(g["f0"], meta["n_frames"], meta["hop_size"])[0]
    k = np.arange(ext.size)
    assert np.array_equal(ext, g["f0"][: meta["n_frames"]][k % meta["n_frames"]])


def test_sinegen_refusals():
    from parallelwavegan_b200 import layers, ops
    from parallelwavegan_b200.capi import PwgbError

    with pytest.raises(PwgbError, match="flag_for_pulse"):
        layers.SineGen(24000, flag_for_pulse=True)
    g = layers.SineGen(24000, harmonic_num=2)
    assert (g.dim, g.sampling_rate, g.sine_amp, g.noise_std, g.voiced_threshold) == (3, 24000, 0.1, 0.003, 0)
    with pytest.raises(PwgbError, match="no CPU fallback"):
        g(torch.zeros(1, 8, 1))
    with pytest.raises(PwgbError, match=r"\(B, T, 1\)"):
        g(torch.zeros(1, 8))
    with pytest.raises(PwgbError, match="no CPU fallback"):
        ops.sine_gen(torch.zeros(1, 8), 0, 24000, 0.1, 0.003, 0, torch.zeros(1, 1), torch.zeros(1, 8, 1))


# ------------------------------------------------------------------ decoder host logic

SMALL_U = dict(in_channels=8, channels=8, downsample_scales=[2, 2], downsample_kernel_sizes=[4, 4], upsample_scales=[2, 2],
               upsample_kernel_sizes=[4, 4], resblock_kernel_sizes=[3], resblock_dilations=[[1]])


def test_decoder_kind_routing():
    from parallelwavegan_b200 import decode, models

    assert decode.decoder_kind(models.UHiFiGANGenerator(**SMALL_U)) == "uhifigan"
    assert decode.decoder_kind(models.HiFiGANGenerator(channels=32)) == "mel2wav"
    assert decode.decoder_kind(models.MelGANGenerator()) == "mel2wav"
    assert decode.decoder_kind(models.ParallelWaveGANGenerator(layers=3, stacks=1)) == "pwg"
    assert decode.decoder_kind(models.StyleMelGANGenerator()) == "style"


def _bare(kind, hop=4, rank=0, world=1):
    from parallelwavegan_b200 import decode, models

    d = object.__new__(decode.Decoder)
    d.kind, d.hop, d.rank, d.world = kind, hop, rank, world
    d.model = models.UHiFiGANGenerator(**SMALL_U) if kind == "uhifigan" else models.HiFiGANGenerator(channels=32)
    return d


def test_decoder_excitation_checks():
    from parallelwavegan_b200 import decode
    from parallelwavegan_b200.capi import PwgbError

    mels = [np.zeros((3, 8), np.float32), np.zeros((5, 8), np.float32)]
    good = [np.zeros((3, 4), np.float32), torch.zeros(20)]
    with pytest.raises(PwgbError, match="needs excitations"):
        _bare("uhifigan").decode(mels)
    with pytest.raises(PwgbError, match="2 utterances"):
        _bare("uhifigan").decode(mels, excitations=good[:1])
    with pytest.raises(PwgbError, match="excitation 1 has 19 samples"):
        _bare("uhifigan").decode(mels, excitations=[good[0], torch.zeros(19)])
    with pytest.raises(PwgbError, match="normalize_before"):
        _bare("uhifigan").decode(mels, normalize_before=True, excitations=good)
    with pytest.raises(PwgbError, match="U-Net HiFi-GAN only"):
        _bare("mel2wav").decode(mels, excitations=good)
    # (T', hop) and (T' * hop,) are both accepted; only this rank's utterances are checked
    rows = decode._excitation_rows(good, mels, [0, 1], 4)
    assert {i: tuple(r.shape) for i, r in rows.items()} == {0: (12,), 1: (20,)}
    assert list(decode._excitation_rows([good[0], torch.zeros(19)], mels, [0], 4)) == [0]


# ------------------------------------------------------------------ codegen

def _nvcc():
    cand = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    return cand if os.path.isfile(cand) and os.access(cand, os.X_OK) else None


def test_sine_kernels_compile_without_spills(tmp_path):
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not found")
    csrc = os.path.join(ROOT, "parallelwavegan_b200", "csrc")
    cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-I", os.path.join(ROOT, "include"), "-I", csrc,
           "-Xptxas", "-v", "-c", os.path.join(csrc, "sine.cu"), "-o", str(tmp_path / "sine.o")]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout[-4000:]
    props = {}
    for m in re.finditer(r"Function properties for (\S*sine_\w*kernel\S*)\s*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                         r"(\d+) bytes spill loads", r.stdout):
        props[m.group(1)] = tuple(int(g) for g in m.group(2, 3, 4))
    assert len(props) == 4, sorted(props)  # the three chunk passes and the scan
    assert not {k: v for k, v in props.items() if any(v)}, props
