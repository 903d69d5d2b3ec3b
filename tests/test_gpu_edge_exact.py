"""Dropout, the VQ nearest-code search, PCM16 and feature prep held bit for bit to independent references
(oracle/philox.py, oracle/edge_exact.py; tests/test_philox_cpu.py checks those on the CPU).

- dropout.cu: the mask and result of every element against a numpy Philox4x32-10, over lengths at the edges of the
  float4 groups and of one pass of the capped grid, misaligned pointers (the scalar path), seeds and offsets that use
  both words, p at 0, 1, their neighbours and exactly some element's u; non-finite inputs; the backward's mask;
- vq.cu: on integer grid data every fp32 distance is exact, so the index must be the float64 argmin with ties to the
  lowest index -- across D on both sides of the 48 KiB shared-memory opt-in and at the 768 maximum, K and T around the
  32-code chunk and 32-frame tile, planted ties in each place the search merges candidates, and the guard that keeps
  the zero-padded code slots of the last chunk out;
- decode.cu: PCM16 at rounding ties, saturation, non-finite values and the grid-stride tail; prep_features across
  channel tiles, both edge modes, t_out past the padded signal and inexact or zero scales.
Output buffers start as NaN with a guard zone after them, so an unwritten or overwritten element shows."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import edge_exact as E
from oracle import philox as PX
from oracle import ref_vqvae

pytestmark = pytest.mark.gpu
f32 = np.float32
DROP_PASS = 132 * 16 * 256 * 4  # elements one pass of the capped dropout grid covers
PCM_PASS = 1184 * 256  # elements one pass of the capped PCM16 grid covers
GUARD = 16


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    import __graft_entry__

    __graft_entry__.build()
    return torch.device("cuda:0")


def _same(what, got, ref):
    """bit-equal arrays, except that any NaN equals any NaN (the GPU does not keep NaN payloads)"""
    got, ref = np.asarray(got), np.asarray(ref)
    assert got.shape == ref.shape and got.dtype == ref.dtype, (what, got.shape, got.dtype, ref.shape, ref.dtype)
    if got.dtype == f32:
        gn, rn = np.isnan(got), np.isnan(ref)
        bad = (gn != rn) | (~gn & (got.view(np.uint32) != ref.view(np.uint32)))
    else:
        bad = got != ref
    if bad.any():
        i = tuple(np.argwhere(bad)[0])
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.size} elements differ, first at {list(i)}: got {got[i]!r}, want {ref[i]!r}")


def _lib():
    from parallelwavegan_b200 import capi, ops

    return capi, capi.lib(), ops._stream()


# ---------------------------------------------------------------------------------------------------- dropout
def _special_input(n, seed):
    """normal values with -0.0, +-inf and NaN planted at the start, the end and at random places"""
    rng = np.random.default_rng(seed)
    x = rng.standard_normal(n).astype(f32)
    sp = np.array([-0.0, np.inf, -np.inf, np.nan, 0.0], f32)
    for pos in (np.arange(min(n, 5)), np.arange(max(0, n - 5), n), rng.integers(0, n, size=min(n, 40))):
        x[pos] = sp[np.arange(pos.size) % sp.size]
    return x


def _dropout(x, p, seed, offset, dev, sx=0, sy=0, backward=False):
    """pwgb_dropout_forward / _backward of the flat x with x and y placed sx / sy elements past a 16-byte boundary"""
    capi, L, stream = _lib()
    n = x.size
    xb = torch.full((n + sx + GUARD,), float("nan"), device=dev)
    xb[sx:sx + n] = torch.from_numpy(x).to(dev)
    yb = torch.full((n + sy + GUARD,), float("nan"), device=dev)
    assert xb.data_ptr() % 16 == 0 and yb.data_ptr() % 16 == 0
    fn = L.pwgb_dropout_backward if backward else L.pwgb_dropout_forward
    rc = fn(C.c_void_p(xb.data_ptr() + 4 * sx), C.c_void_p(yb.data_ptr() + 4 * sy), n, float(p), int(seed), int(offset), stream)
    capi.check(rc, "dropout")
    y = yb.cpu().numpy()
    assert np.isnan(y[:sy]).all() and np.isnan(y[sy + n:]).all(), "dropout wrote outside its n elements"
    return y[sy:sy + n]


@pytest.mark.parametrize("n", [1, 2, 3, 4, 5, 4097, DROP_PASS, DROP_PASS + 1, 5_000_011])
def test_dropout_lengths_and_alignment(dev, n):
    """the float4 path (both pointers aligned) and the scalar path (either one off by 1-3 elements) write the same
    reference values, across the partial last group and the second pass of the grid-stride loop"""
    seed, offset, p = 0x1234_5678_9ABC_DEF1, 2**32 + 5, 0.1
    x = _special_input(n, n)
    gy = np.random.default_rng(n + 1).standard_normal(n).astype(f32)
    u = PX.uniforms(n, seed, offset)
    want, want_g = PX.dropout(x, p, seed, u=u), PX.dropout(gy, p, seed, u=u)
    for sx, sy in ((0, 0), (1, 0), (0, 3), (2, 1)):
        _same(f"forward n={n} shift=({sx},{sy})", _dropout(x, p, seed, offset, dev, sx, sy), want)
        _same(f"backward n={n} shift=({sx},{sy})", _dropout(gy, p, seed, offset, dev, sx, sy, backward=True), want_g)


SEEDS = [0, 2**32 - 1, 2**32, 2**63 - 2, 0xA5A5_0001_0F0F_7777]
OFFSETS = [0, 1, 2**32 + 5]


@pytest.mark.parametrize("seed", SEEDS)
def test_dropout_seeds_offsets_and_p(dev, seed):
    """every word of the seed and offset, p at its edges and at exactly one element's u (u == p is kept); p == 1
    drops everything, inf and NaN included, to +0.0"""
    n = 4099
    x = _special_input(n, 7)
    gy = np.random.default_rng(8).standard_normal(n).astype(f32)
    for offset in OFFSETS:
        u = PX.uniforms(n, seed, offset)
        j = int(np.argmin(np.abs(u - f32(0.37))))
        x[j] = 1.25  # a finite, non-zero element sits on the boundary
        ps = [0.0, 2.0**-24, 0.1, 0.5, 1.0 - 2.0**-24, 1.0, float(u[j])]
        for p in ps:
            want = PX.dropout(x, p, seed, u=u)
            got = _dropout(x, p, seed, offset, dev, 0, 0)
            _same(f"seed={seed} offset={offset} p={p}", got, want)
            if p == float(u[j]):
                assert got[j] == f32(1.25) * PX.scale_of(p), "the element with u == p must be kept"
            if p == 1.0:
                assert np.array_equal(got.view(np.uint32), np.zeros(n, np.uint32))
            if p == 0.0:
                _same("p = 0 is the identity", got, x)
        p = 0.5
        _same(f"backward seed={seed} offset={offset}", _dropout(gy, p, seed, offset, dev, 0, 1, backward=True), PX.dropout(gy, p, seed, u=u))


def test_dropout_refuses_bad_p(dev):
    capi, L, stream = _lib()
    x = torch.ones(64, device=dev)
    y = torch.full((64,), float("nan"), device=dev)
    for fn in (L.pwgb_dropout_forward, L.pwgb_dropout_backward):
        for p in (-2.0**-24, -0.5, 1.0 + 2.0**-23, 2.0, float("nan")):
            capi.reset_launch_count()
            assert fn(C.c_void_p(x.data_ptr()), C.c_void_p(y.data_ptr()), 64, p, 1, 0, stream) == -1, p
            assert capi.launch_count() == 0
            assert "p = " in L.pwgb_last_error().decode()
    assert bool(torch.isnan(y).all())


@pytest.mark.parametrize("s", [0, 11])
def test_dropout_model_level_seed_replay(dev, s):
    """ops.dropout draws its seed from torch's CPU generator: after torch.manual_seed(s) the forward, the
    DropoutFn backward and the no-grad path equal the reference with the replayed seed at offset 0"""
    from parallelwavegan_b200 import ops

    p = 0.3
    x = _special_input(2 * 48 * 97, 3 + s).reshape(2, 48, 97)
    gy = np.random.default_rng(s).standard_normal(x.shape).astype(f32)
    torch.manual_seed(s)
    seed = int(torch.randint(0, 2**63 - 1, (), dtype=torch.int64))
    want, want_g = PX.dropout(x, p, seed).reshape(x.shape), PX.dropout(gy, p, seed).reshape(x.shape)
    torch.manual_seed(s)
    xt = torch.from_numpy(x).to(dev).requires_grad_(True)
    y = ops.dropout(xt, p, True)
    y.backward(torch.from_numpy(gy).to(dev))
    _same("forward", y.detach().cpu().numpy(), want)
    _same("backward", xt.grad.cpu().numpy(), want_g)
    torch.manual_seed(s)
    with torch.no_grad():
        _same("no_grad forward", ops.dropout(torch.from_numpy(x).to(dev), p, True).cpu().numpy(), want)


# ---------------------------------------------------------------------------------------------------- VQ search
def _cb(cb, dev):
    """the codebook on the device in a buffer with 32 spare zero rows after it, so that a gather of a wrongly chosen
    padded slot reads defined memory and shows as a wrong index"""
    K, D = cb.shape
    buf = torch.zeros((K + 32, D), device=dev)
    buf[:K] = torch.from_numpy(cb).to(dev)
    return buf[:K]


def _vq(z, cb, dev, **kw):
    from parallelwavegan_b200 import ops

    idx, zq, dc = ops.vq_raw(torch.from_numpy(z).to(dev), _cb(cb, dev), **kw)
    return idx.cpu().numpy(), zq.cpu().numpy() if zq is not None else None, dc.cpu().numpy() if dc is not None else None


def _gathered(cb, idx):
    return np.ascontiguousarray(cb[idx].transpose(0, 2, 1))  # (B, D, T)


@pytest.mark.parametrize("D", [1, 3, 100, 192, 193, 768])
def test_vq_search_grid_shapes(dev, D):
    """D on both sides of the 48 KiB opt-in and the maximum; K and T around the 32-code chunk and the 32-frame tile.
    D = 1 and 3 are full of natural ties.  D = 192 fills exactly 48 KiB of dynamic shared memory, which with the
    kernel's static arrays needs the opt-in (the launch once failed there)"""
    rng = np.random.default_rng(D)
    for K in (1, 31, 32, 33, 1000):
        cb = E.vq_grid(rng, (K, D))
        for T in (1, 31, 32, 33, 100):
            for B in (1, 3):
                z = E.vq_grid(rng, (B, D, T))
                want = E.vq_argmin(z, cb)
                idx, zq, _ = _vq(z, cb, dev, z_q=True, dec=False)
                _same(f"D={D} K={K} T={T} B={B} index", idx, want)
                _same(f"D={D} K={K} T={T} B={B} z_q", zq, _gathered(cb, want))


# tie sets: each frame is a copy of the code at min(S), planted at every index of S.  The search gives thread (q, lane)
# codes k0 + 4 q + j (j < 4) of each 32-code chunk and merges the 8 warps' bests in warp order at the end
TIE_SETS = [
    (40, 41, 43),  # one thread (chunk 1, q 2), three j
    (70, 93),  # one chunk, warps 1 and 7
    (28, 32),  # chunk 0 warp 7 against chunk 1 warp 0: the lower index merges after the higher one
    (100, 500, 777),  # later chunks
    (993, 998),  # the last, partial chunk (992 .. 999 of K = 1000)
    (200, 997),  # an early code and a code of the partial chunk
    (0, 31, 999),  # the first code, the last of chunk 0 and the last code
    (6, 3 * 32 + 6, 5 * 32 + 6, 30 * 32 + 6),  # the same (q, j) slot of four chunks
]


@pytest.mark.parametrize("D", [5, 193])
def test_vq_search_planted_ties(dev, D):
    K, B, T = 1000, 2, 45
    rng = np.random.default_rng(D + 17)
    cb = E.vq_grid(rng, (K, D))
    z = E.vq_grid(rng, (B, D, T))
    frames = {}
    for i, S in enumerate(TIE_SETS):
        for s in S:
            cb[s] = cb[S[0]]
        for b, t in ((0, 3 * i), (1, T - 1 - 2 * i), (i % 2, 31 + i % 3)):  # both items, across the 32-frame tile edge
            z[b, :, t] = cb[S[0]]
            frames[(b, t)] = S[0]
    want = E.vq_argmin(z, cb)
    for (b, t), k in frames.items():
        assert want[b, t] == k
    idx, zq, _ = _vq(z, cb, dev)
    _same(f"D={D} planted ties", idx, want)
    _same(f"D={D} z_q", zq, _gathered(cb, want))


@pytest.mark.parametrize("D", [3, 193])
@pytest.mark.parametrize("K", [1, 31, 33, 1000])
def test_vq_search_ignores_padded_code_slots(dev, D, K):
    """every real code is far from every frame and the last chunk's padded slots are zero codes, nearer than any
    real code: the index stays below K"""
    rng = np.random.default_rng(K * D)
    cb = (rng.choice([-1.0, 1.0], size=(K, D)) * rng.integers(5, 7, size=(K, D))).astype(f32)
    z = E.vq_grid(rng, (2, D, 40), -1, 1)
    want = E.vq_argmin(z, cb)
    assert (E.vq_distances(z, cb).min(-1) > (z.astype(np.float64) ** 2).sum(1)).all()  # a zero code would win
    idx, _, _ = _vq(z, cb, dev, z_q=False, dec=False)
    assert (idx >= 0).all() and (idx < K).all()
    _same(f"D={D} K={K}", idx, want)


def test_vq_search_largest_batch(dev):
    rng = np.random.default_rng(65535)
    cb = E.vq_grid(rng, (33, 3))
    z = E.vq_grid(rng, (65535, 3, 1))
    idx, zq, _ = _vq(z, cb, dev)
    want = E.vq_argmin(z, cb)
    _same("B=65535 index", idx, want)
    _same("B=65535 z_q", zq, _gathered(cb, want))


def test_vq_search_non_finite_follows_torch_min(dev):
    """an inf code component and +-inf frames: the fp32 distances have inf and NaN, and the index is torch.min's over
    the reference's distances (the first NaN, else the lowest index of the minimum)"""
    rng = np.random.default_rng(4)
    D, K, B, T = 8, 40, 2, 40
    z, cb = E.vq_grid(rng, (B, D, T)), E.vq_grid(rng, (K, D))
    cb[5, 2], cb[17, 0] = np.inf, -np.inf
    z[0, 1, 3], z[1, 4, 7], z[0, 0, 33] = np.inf, -np.inf, np.inf
    z[1, 2, 12] = 0.0  # code 5's inf meets a zero: NaN
    d = ref_vqvae.distances(torch.from_numpy(z), torch.from_numpy(cb))
    want = d.min(1)[1].numpy().reshape(B, T)
    assert np.array_equal(want, E.argmin_first(d.numpy()).reshape(B, T))
    assert bool(torch.isnan(d).any()) and bool(torch.isinf(d).any())
    idx, _, _ = _vq(z, cb, dev, z_q=False, dec=False)
    _same("non-finite", idx, want)


def test_vq_assembly_gathers_exactly(dev):
    rng = np.random.default_rng(9)
    D, K, B, T, Cl, Cg, ng = 100, 33, 3, 70, 5, 4, 3
    cb, z = E.vq_grid(rng, (K, D)), E.vq_grid(rng, (B, D, T))
    l = rng.standard_normal((B, Cl, T)).astype(f32)
    gt = rng.standard_normal((ng, Cg)).astype(f32)
    g = np.array([2, 0, 1], np.int64)
    from parallelwavegan_b200 import ops

    idx, zq, dc = ops.vq_raw(torch.from_numpy(z).to(dev), _cb(cb, dev), l=torch.from_numpy(l).to(dev),
                             global_table=torch.from_numpy(gt).to(dev), g=torch.from_numpy(g).to(dev))
    want = E.vq_argmin(z, cb)
    _same("index", idx.cpu().numpy(), want)
    _same("z_q", zq.cpu().numpy(), _gathered(cb, want))
    _same("dec", dc.cpu().numpy(), np.concatenate([_gathered(cb, want), l, np.repeat(gt[g][:, :, None], T, 2)], 1))


def test_vq_refuses_before_launch(dev):
    from parallelwavegan_b200 import capi, ops
    from parallelwavegan_b200.capi import PwgbError

    for z, cb, what in ((torch.zeros(1, 769, 4, device=dev), torch.zeros(3, 769, device=dev), "embed_dim 769 > 768"),
                        (torch.zeros(65536, 2, 1, device=dev), torch.zeros(3, 2, device=dev), "batch 65536 > 65535")):
        capi.reset_launch_count()
        with pytest.raises(PwgbError, match=what):
            ops.vq_raw(z, cb)
        B, _, T = z.shape
        frame, end = torch.zeros(B, dtype=torch.int32, device=dev), torch.full((B,), T, dtype=torch.int32, device=dev)
        with pytest.raises(PwgbError, match=what):
            ops.vq_stream(z, cb, (frame, end, 1, 0))
        assert capi.launch_count() == 0


def test_vq_stream_launch_at_max_dim(dev):
    """pwgb_vq_stream_forward at D = 768: the search of the whole-signal launch inside each item's signal, index -1
    and +0.0 columns outside it"""
    from parallelwavegan_b200 import ops

    rng = np.random.default_rng(768)
    D, K, B, T, look = 768, 100, 3, 70, 4
    cb, z = E.vq_grid(rng, (K, D)), E.vq_grid(rng, (B, D, T))
    cb[99] = cb[3]
    z[0, :, 20] = cb[3]
    frame, end = np.array([0, 10, 5], np.int32), np.array([50, 80, 3], np.int32)
    pos = frame[:, None] - look + np.arange(T)[None, :]
    inside = (pos >= 0) & (pos < end[:, None])
    assert inside.any() and (~inside).any()
    dec = torch.full((B, D, T), float("nan"), device=dev)
    idx, dec = ops.vq_stream(torch.from_numpy(z).to(dev), _cb(cb, dev),
                             (torch.from_numpy(frame).to(dev), torch.from_numpy(end).to(dev), 1, look), dec=dec)
    want = E.vq_argmin(z, cb)
    _same("stream index", idx.cpu().numpy(), np.where(inside, want, -1))
    _same("stream dec", dec.cpu().numpy(), np.where(inside[:, None, :], _gathered(cb, want), f32(0.0)))


# ---------------------------------------------------------------------------------------------------- PCM16
@pytest.mark.parametrize("n", [1, PCM_PASS + 1, 4_000_037])
def test_pcm16_bit_exact(dev, n):
    """ties of both parities and signs, +-1 and their neighbours, overrange, +-inf, subnormals and NaN, placed at the
    start, the end (the grid-stride tail) and at random among uniform values"""
    from parallelwavegan_b200 import decode

    rng = np.random.default_rng(n)
    sp = np.concatenate([E.pcm16_specials(), E.pcm16_ties(8, n)])
    y = rng.uniform(-1.1, 1.1, n).astype(f32)
    if n == 1:
        cases = [y] + [sp[i:i + 1] for i in range(sp.size)]
    else:
        y[:sp.size], y[n - sp.size:] = sp, sp[::-1]
        y[rng.integers(0, n, size=4 * sp.size)] = np.tile(sp, 4)
        cases = [y]
    for v in cases:
        _same(f"pcm16 n={n}", decode.pcm16(torch.from_numpy(v).to(dev)).cpu().numpy(), E.pcm16(v))
    if n == 1:
        assert int(decode.pcm16(torch.tensor([float("nan")], device=dev)).item()) == 0


def test_pcm16_writes_only_n(dev):
    capi, L, stream = _lib()
    n = PCM_PASS + 3
    y = torch.from_numpy(np.random.default_rng(0).uniform(-1, 1, n).astype(f32)).to(dev)
    out = torch.full((n + GUARD,), -7, dtype=torch.int16, device=dev)
    capi.check(L.pwgb_pcm16_forward(C.c_void_p(y.data_ptr()), C.c_void_p(out.data_ptr()), n, stream), "pcm16")
    o = out.cpu().numpy()
    _same("pcm16", o[:n], E.pcm16(y.cpu().numpy()))
    assert (o[n:] == -7).all()


# ---------------------------------------------------------------------------------------------------- prep_features
@pytest.mark.parametrize("Cn", [1, 31, 32, 33, 80, 513])
def test_prep_features_bit_exact(dev, Cn):
    """normalisation with inexact quotients and zero scales (+-inf, NaN), zero and replicate edges, t_out below and past
    the padded signal; padded zero frames stay +0.0"""
    from parallelwavegan_b200 import decode

    rng = np.random.default_rng(Cn)
    mean = rng.standard_normal(Cn).astype(f32)
    scale = rng.uniform(0.3, 3.0, Cn).astype(f32)
    scale[3::7] = 0.0
    for T in (1, 31, 33, 200):
        c = (rng.standard_normal((T, Cn)) * 3).astype(f32)
        c[::5, 3::7] = mean[3::7]  # (mean - mean) / 0: NaN
        c[0, ::4] = -0.0
        cd = torch.from_numpy(c).to(dev)
        for pad_left in (0, 1, 2, 40):
            for t_out in sorted({max(1, T + pad_left - 3), T + pad_left, T + pad_left + 37}):
                for norm in (False, True):
                    for replicate in (False, True):
                        buf = torch.full((Cn * t_out + GUARD,), float("nan"), device=dev)
                        out = buf[:Cn * t_out].view(Cn, t_out)
                        decode.prep_features(cd, out, torch.from_numpy(mean).to(dev) if norm else None,
                                             torch.from_numpy(scale).to(dev) if norm else None, pad_left=pad_left, replicate=replicate)
                        b = buf.cpu().numpy()
                        what = f"C={Cn} T={T} pad_left={pad_left} t_out={t_out} norm={norm} replicate={replicate}"
                        _same(what, b[:Cn * t_out].reshape(Cn, t_out),
                              E.prep_features(c, t_out, pad_left, mean if norm else None, scale if norm else None, replicate))
                        assert np.isnan(b[Cn * t_out:]).all(), what
