"""The references of oracle/philox.py and oracle/edge_exact.py checked on the CPU, before tests/test_gpu_edge_exact.py
holds the dropout, nearest-code search, PCM16 and feature-prep kernels to them bit for bit:

- Philox4x32-10 reproduces the Random123 known-answer vectors, and the vectorised generator agrees with a scalar
  restatement of dropout.cu's round (key bumped after every round) over random counters and keys;
- the dropout stream lays elements out as dropout.cu defines it (group e / 4, word e % 4, both counter and key words);
- the VQ argmin follows torch.min on the reference's distances (ties, NaN), and the grid data is exact;
- PCM16 and prep_features agree with independent restatements (Python's round, torch's pad and arithmetic)."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import edge_exact as E
from oracle import philox as PX
from oracle import ref_vqvae

f32 = np.float32


# ---------------------------------------------------------------------------------------------------- Philox
@pytest.mark.parametrize("ctr,key,want", [
    ((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
    ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
    ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0), (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1)),
])
def test_philox_known_answers(ctr, key, want):
    got = PX.philox4x32_10(*ctr, *key)
    assert tuple(int(w) for w in got) == want, " ".join(f"{int(w):08x}" for w in got)


def _philox_scalar(c, k):
    """dropout.cu's philox4x32_10 in Python integers: ten rounds, the key bumped after each"""
    c, k = list(c), list(k)
    for _ in range(10):
        p0, p1 = PX.M0 * c[0], PX.M1 * c[2]
        c = [((p1 >> 32) ^ c[1] ^ k[0]) & PX.MASK32, p1 & PX.MASK32, ((p0 >> 32) ^ c[3] ^ k[1]) & PX.MASK32, p0 & PX.MASK32]
        k = [(k[0] + PX.W0) & PX.MASK32, (k[1] + PX.W1) & PX.MASK32]
    return tuple(c)


def test_philox_vectorised_matches_scalar_rounds():
    rng = np.random.default_rng(1)
    c = rng.integers(0, 2**32, size=(4, 64), dtype=np.uint64)
    k = rng.integers(0, 2**32, size=(2, 64), dtype=np.uint64)
    got = np.stack(PX.philox4x32_10(*c, *k))
    for i in range(64):
        assert tuple(int(v) for v in got[:, i]) == _philox_scalar([int(v) for v in c[:, i]], [int(v) for v in k[:, i]])


@pytest.mark.parametrize("seed,offset", [(0, 0), (2**32 - 1, 1), (2**32, 2**32 + 5), (2**63 - 2, 0), (0x1234_5678_9ABC_DEF1, 2**32 + 5)])
def test_dropout_stream_layout(seed, offset):
    """element e: word e % 4 of the call at counter (e / 4 low, e / 4 high, offset low, offset high), key (seed low,
    seed high), its top 24 bits over 2^24"""
    n = 23
    u = PX.uniforms(n, seed, offset)
    assert u.dtype == f32
    for e in range(n):
        g = e // 4
        w = _philox_scalar([g & PX.MASK32, g >> 32, offset & PX.MASK32, offset >> 32], [seed & PX.MASK32, seed >> 32])[e % 4]
        assert float(u[e]) == (w >> 8) / 2.0**24
    # every word of the counter and key matters
    assert not np.array_equal(u, PX.uniforms(n, seed ^ (1 << 40), offset))
    assert not np.array_equal(u, PX.uniforms(n, seed ^ 1, offset))
    assert not np.array_equal(u, PX.uniforms(n, seed, offset ^ (1 << 40)))
    assert not np.array_equal(u, PX.uniforms(n, seed, offset ^ 1))


def test_dropout_stream_high_group_word():
    """the counter's second word is the high half of the group index: element 4 * 2^32 uses counter (0, 1, ...)"""
    g = 2**32
    words = PX.philox4x32_10(g & PX.MASK32, g >> 32, 0, 0, 7, 0)
    assert tuple(int(w) for w in words) == _philox_scalar([0, 1, 0, 0], [7, 0])
    assert tuple(int(w) for w in words) != _philox_scalar([0, 0, 0, 0], [7, 0])


def test_dropout_reference_rules():
    x = np.array([1.5, -0.0, np.inf, -np.inf, np.nan, 3.0, -2.0, 0.0] * 64, f32)
    seed = 99
    y0 = PX.dropout(x, 0.0, seed)
    assert np.array_equal(y0.view(np.uint32)[~np.isnan(x)], x.view(np.uint32)[~np.isnan(x)]) and np.isnan(y0[np.isnan(x)]).all()
    y1 = PX.dropout(x, 1.0, seed)
    assert np.array_equal(y1.view(np.uint32), np.zeros(x.size, np.uint32))  # all +0.0, no NaN from inf * 0
    p = f32(0.3)
    y = PX.dropout(x, p, seed)
    keep = PX.uniforms(x.size, seed, 0) >= p
    assert 0 < keep.sum() < x.size
    assert np.array_equal(y[~keep].view(np.uint32), np.zeros((~keep).sum(), np.uint32))
    scale = f32(1) / (f32(1) - p)
    assert scale.dtype == f32 and PX.scale_of(p) == scale and float(scale) != 1 / (1 - float(p))  # the fp32 quotient
    with np.errstate(invalid="ignore"):
        want = x[keep] * scale
    assert np.array_equal(y[keep], want, equal_nan=True)
    assert np.signbit(y[keep & (x == 0) & np.signbit(x)]).all()  # a kept -0.0 stays -0.0


def test_dropout_u_boundary_is_kept():
    """p equal to some element's u keeps that element (u >= p), and the fp32 p of the C ABI is what is compared"""
    u = PX.uniforms(4097, 5, 1)
    j = int(np.argmin(np.abs(u - 0.5)))
    keep = PX.keep_mask(4097, u[j], 5, 1)
    assert keep[j] and not (u[~keep] >= u[j]).any()
    assert float(f32(0.1)) != 0.1 and PX.keep_mask(4097, 0.1, 5, 1).sum() == (u >= f32(0.1)).sum()


# ---------------------------------------------------------------------------------------------------- VQ argmin
@pytest.mark.parametrize("D,K", [(1, 1000), (3, 33), (100, 31), (768, 40)])
def test_vq_reference_matches_torch_min(D, K):
    """on grid data (D = 1 and 3 are full of ties) the exact float64 argmin is torch.min over the reference's fp32
    distances, and those distances are exact"""
    rng = np.random.default_rng(D + K)
    z, cb = E.vq_grid(rng, (2, D, 37)), E.vq_grid(rng, (K, D))
    cb[K - 1] = cb[0]
    want = E.vq_argmin(z, cb)
    d = ref_vqvae.distances(torch.from_numpy(z), torch.from_numpy(cb))
    assert np.array_equal(d.double().numpy().reshape(2, 37, K), E.vq_distances(z, cb))
    assert np.array_equal(want.reshape(-1), d.min(1)[1].numpy())
    assert np.array_equal(want, E.argmin_first(E.vq_distances(z, cb)))


def test_vq_reference_nan_and_inf_follow_torch_min():
    rng = np.random.default_rng(4)
    z, cb = E.vq_grid(rng, (2, 8, 40)), E.vq_grid(rng, (40, 8))
    cb[5, 2], cb[17, 0] = np.inf, -np.inf
    z[0, 1, 3], z[1, 4, 7], z[1, 6, 9] = np.inf, -np.inf, np.nan
    d = ref_vqvae.distances(torch.from_numpy(z), torch.from_numpy(cb))
    assert bool(torch.isnan(d).any()) and bool(torch.isinf(d).any())
    assert np.array_equal(E.argmin_first(d.numpy()), d.min(1)[1].numpy())
    dd = np.array([[3.0, np.nan, 1.0, np.nan], [2.0, 1.0, 1.0, 5.0], [np.inf, np.inf, np.inf, np.inf]])
    assert E.argmin_first(dd).tolist() == [1, 1, 0] == torch.from_numpy(dd).min(1)[1].tolist()


def test_vq_exactness_precondition():
    rng = np.random.default_rng(0)
    E.require_vq_exact(E.vq_grid(rng, (1, 768, 4)), E.vq_grid(rng, (3, 768)))
    with pytest.raises(AssertionError):
        E.require_vq_exact(E.vq_grid(rng, (1, 4, 4)) + f32(0.5), E.vq_grid(rng, (3, 4)))
    with pytest.raises(AssertionError):
        E.require_vq_exact(np.full((1, 768, 1), 100, f32), np.full((3, 768), 100, f32))


# ---------------------------------------------------------------------------------------------------- PCM16
def _pcm16_scalar(y):
    with np.errstate(over="ignore", invalid="ignore"):
        p = float(f32(y) * f32(32767.0))
    if math.isnan(p):
        return 0
    if math.isinf(p):
        return 32767 if p > 0 else -32768
    return max(-32768, min(32767, round(p)))  # Python's round: half to even


def test_pcm16_reference_rule():
    ys = np.concatenate([E.pcm16_specials(), E.pcm16_ties(), np.random.default_rng(2).uniform(-1.3, 1.3, 500).astype(f32)])
    got = E.pcm16(ys)
    assert got.dtype == np.int16
    assert got.tolist() == [_pcm16_scalar(y) for y in ys]
    assert int(E.pcm16(np.array([np.nan], f32))[0]) == 0


def test_pcm16_ties_are_ties():
    t = E.pcm16_ties()
    prod = (t * f32(32767.0)).astype(np.float64)
    assert np.array_equal(prod - np.floor(prod), np.full(t.size, 0.5))
    k = np.floor(np.abs(prod)).astype(np.int64)
    assert {0, 1} <= set((k % 2).tolist()) and (t > 0).any() and (t < 0).any()
    q = E.pcm16(t).astype(np.int64)
    assert (q % 2 == 0).all()  # half to even: neither truncation nor half away from zero
    assert not np.array_equal(q, np.trunc(prod).astype(np.int64)) and not np.array_equal(q, (np.sign(prod) * np.floor(np.abs(prod) + 0.5)).astype(np.int64))


# ---------------------------------------------------------------------------------------------------- prep_features
@pytest.mark.parametrize("C,T,pad_left,t_out", [(1, 1, 0, 1), (33, 31, 2, 60), (80, 33, 40, 50), (513, 200, 1, 150)])
@pytest.mark.parametrize("norm", [False, True])
@pytest.mark.parametrize("replicate", [False, True])
def test_prep_features_reference_matches_torch(C, T, pad_left, t_out, norm, replicate):
    rng = np.random.default_rng(C + T)
    c = (rng.standard_normal((T, C)) * 3).astype(f32)
    mean = rng.standard_normal(C).astype(f32) if norm else None
    scale = rng.uniform(0.3, 3.0, C).astype(f32) if norm else None
    got = E.prep_features(c, t_out, pad_left, mean, scale, replicate)
    x = torch.from_numpy(c).t()[None]  # (1, C, T)
    if replicate:
        xp = F.pad(x, (pad_left, max(0, t_out - T - pad_left)), mode="replicate")[0, :, :t_out]
        if norm:
            xp = (xp - torch.from_numpy(mean)[:, None]) / torch.from_numpy(scale)[:, None]
    else:
        if norm:
            x = (x - torch.from_numpy(mean)[None, :, None]) / torch.from_numpy(scale)[None, :, None]
        xp = F.pad(x, (pad_left, max(0, t_out - T - pad_left)))[0, :, :t_out]
    assert got.shape == (C, t_out) and got.dtype == f32
    assert np.array_equal(got.view(np.uint32), xp.contiguous().numpy().view(np.uint32))


def test_prep_features_reference_edges():
    c = np.array([[1.0, 2.0], [3.0, 4.0]], f32)
    mean, scale = np.array([1.0, 4.0], f32), np.array([0.0, 3.0], f32)
    z = E.prep_features(c, 5, 1, mean, scale, replicate=False)
    assert np.array_equal(z[:, [0, 3, 4]].view(np.uint32), np.zeros((2, 3), np.uint32))  # padding: +0.0, not normalised
    assert np.isnan(z[0, 1]) and z[0, 2] == np.inf  # (1 - 1) / 0 and (3 - 1) / 0
    assert z[1, 1] == f32(-2.0) / f32(3.0) and z[1, 2] == 0.0
    r = E.prep_features(c, 5, 1, mean, scale, replicate=True)
    assert np.isnan(r[0, :2]).all() and (r[0, 2:] == np.inf).all() and (r[1, 2:] == 0).all()
