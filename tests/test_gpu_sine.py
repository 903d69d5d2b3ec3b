"""SineGen on the GPU (pwgb_sine_gen_forward): against the reference's goldens with the reference's draws injected (the
phase, uv and noise bit for bit, the sine within 2 fp32 ulp x sine_amp: sinf against the CPU's sin), batches of distinct
rows against each row alone across the chunk edges, determinism, a seeded generator, and ``features.excitation``
against the excitation of bin/preprocess.py."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import ref_sine

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
SINE_CASES = ["sine_len1", "sine_hz_h0", "sine_log_h0", "sine_hz_h2_thr5", "sine_log_h2_thr5", "sine_long_h0", "sine_long_h2_log"]
EPS = float(np.finfo(np.float32).eps)
CHUNK = 2048  # samples per block of sine.cu (kChunk)


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    import __graft_entry__

    __graft_entry__.build()
    return torch.device("cuda:0")


def _golden(name):
    z = np.load(os.path.join(GOLD, name + ".npz"), allow_pickle=False)
    return json.loads(str(z["meta"])), {k: z[k] for k in z.files if k != "meta"}


def _run(dev, f0, hn, sr, amp, std, thr, rand_ini, n):
    from parallelwavegan_b200 import ops

    t = lambda a: torch.as_tensor(np.ascontiguousarray(a), dtype=torch.float32).to(dev)  # noqa: E731
    sine, uv, noise, phase = ops.sine_gen(t(f0), hn, sr, amp, std, thr, t(rand_ini), t(n), phase=True)
    return dict(sine_waves=sine.cpu().numpy(), uv=uv.cpu().numpy(), noise=noise.cpu().numpy(), phase=phase.cpu().numpy())


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


@pytest.mark.parametrize("name", SINE_CASES)
def test_sine_gen_matches_reference(dev, name):
    meta, g = _golden(name)
    f0, rand_ini, n = ref_sine.long_case_inputs(meta) if meta["stride"] else (g["f0"], g["rand_ini"], g["n"])
    r = _run(dev, f0, meta["harmonic_num"], meta["samp_rate"], meta["sine_amp"], meta["noise_std"], meta["voiced_threshold"], rand_ini, n)
    s = meta["stride"] or 1
    for k in ("phase", "uv", "noise"):
        got = r[k][:, ::s]
        bad = np.flatnonzero(_bits(got) != _bits(g[k]))
        assert bad.size == 0, (k, bad.size, bad[:5])
    assert np.abs(r["sine_waves"][:, ::s] - g["sine_waves"]).max() <= 2 * EPS * meta["sine_amp"]
    if meta["stride"]:  # every sample against the numpy restatement, which the CPU tests pin to the reference
        ref = ref_sine.sine_gen(f0, meta["harmonic_num"], meta["samp_rate"], meta["sine_amp"], meta["noise_std"],
                                meta["voiced_threshold"], rand_ini, n)
        for k in ("phase", "uv", "noise"):
            assert np.array_equal(_bits(r[k]), _bits(ref[k])), k
        assert np.abs(r["sine_waves"] - ref["sine_waves"]).max() <= 2 * EPS * meta["sine_amp"]


@pytest.mark.parametrize("T", [1, CHUNK - 1, CHUNK, CHUNK + 1, 7 * CHUNK + 913])
@pytest.mark.parametrize("hn", [0, 2])
def test_batch_equals_rows_alone(dev, T, hn):
    """16 distinct rows (Hz with sub-threshold runs, log f0) in one launch = each row alone = the numpy restatement"""
    B = 16
    f0 = np.stack([ref_sine.f0_contour(T, 1000 + b, log=b % 2 == 1, below_threshold=b % 4 == 0) for b in range(B)])
    rng = np.random.default_rng(T * 10 + hn)
    rand_ini = rng.random((B, hn + 1), dtype=np.float32)
    n = rng.standard_normal((B, T, hn + 1), dtype=np.float32)
    args = (hn, 24000, 0.1, 0.003, 1.0)
    batch = _run(dev, f0, *args, rand_ini, n)
    again = _run(dev, f0, *args, rand_ini, n)
    ref = ref_sine.sine_gen(f0, hn, 24000, 0.1, 0.003, 1.0, rand_ini, n)
    for b in range(B):
        alone = _run(dev, f0[b : b + 1], *args, rand_ini[b : b + 1], n[b : b + 1])
        for k in alone:
            assert np.array_equal(_bits(batch[k][b : b + 1]), _bits(alone[k])), (b, k)
    for k in batch:
        assert np.array_equal(_bits(batch[k]), _bits(again[k])), k
    for k in ("phase", "uv", "noise"):
        assert np.array_equal(_bits(batch[k]), _bits(ref[k])), k


def test_sinegen_module_and_generator(dev):
    from parallelwavegan_b200 import layers

    gen = layers.SineGen(24000, harmonic_num=1)
    f0 = torch.from_numpy(np.stack([ref_sine.f0_contour(5000, 7), ref_sine.f0_contour(5000, 8)])[..., None]).to(dev)
    outs = [gen(f0, generator=torch.Generator(device=dev).manual_seed(3)) for _ in range(2)]
    sine, uv, noise = outs[0]
    assert tuple(sine.shape) == (2, 5000, 2) and tuple(uv.shape) == (2, 5000, 1) and tuple(noise.shape) == (2, 5000, 2)
    assert all(torch.equal(a, b) for a, b in zip(*outs))
    other = gen(f0, generator=torch.Generator(device=dev).manual_seed(4))
    assert not torch.equal(other[2], noise)
    # injected draws give the numpy restatement's phase-exact result
    g = torch.Generator(device=dev).manual_seed(5)
    rand_ini = torch.rand(2, 2, device=dev, generator=g)
    n = torch.randn(2, 5000, 2, device=dev, generator=g)
    sine, uv, noise = gen(f0, rand_ini=rand_ini, noise=n)
    ref = ref_sine.sine_gen(f0[..., 0].cpu().numpy(), 1, 24000, rand_ini=rand_ini.cpu().numpy(), n=n.cpu().numpy())
    assert np.array_equal(_bits(noise.cpu().numpy()), _bits(ref["noise"]))
    assert np.abs(sine.cpu().numpy() - ref["sine_waves"]).max() <= 2 * EPS * 0.1
    assert not sine.requires_grad


def test_excitation_matches_preprocess(dev, monkeypatch):
    """features.excitation with the reference's draws in place of its own"""
    from parallelwavegan_b200 import features

    meta, g = _golden("sine_opencpop_excitation")
    rand, randn = torch.rand, torch.randn
    monkeypatch.setattr(torch, "rand", lambda *a, **k: torch.from_numpy(g["rand_ini"]).to(dev))
    monkeypatch.setattr(torch, "randn", lambda *a, **k: torch.from_numpy(g["n"]).to(dev))
    e = features.excitation(torch.from_numpy(g["f0"]).to(dev), meta["n_frames"], meta["sampling_rate"], meta["hop_size"])
    monkeypatch.setattr(torch, "rand", rand)
    monkeypatch.setattr(torch, "randn", randn)
    assert tuple(e.shape) == (meta["n_frames"], meta["hop_size"]) and e.is_cuda
    assert np.abs(e.cpu().numpy() - g["excitation"]).max() <= 2 * EPS * 0.1
    # a seeded generator reproduces; a short f0 is edge-padded
    a = features.excitation(torch.from_numpy(g["f0"][:50]).to(dev), 60, 24000, 300, generator=torch.Generator(device=dev).manual_seed(1))
    b = features.excitation(torch.from_numpy(np.pad(g["f0"][:50], (0, 10), mode="edge")).to(dev), 60, 24000, 300,
                            generator=torch.Generator(device=dev).manual_seed(1))
    assert torch.equal(a, b)
