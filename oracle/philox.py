"""numpy Philox4x32-10 and the dropout of csrc/dropout.cu, written from its definition, for bit-exact comparison.

Philox4x32-10 (Salmon, Moraes, Dror, Shaw: "Parallel random numbers: as easy as 1, 2, 3", SC 2011; the Random123
library's philox4x32_R with R = 10): a 128-bit counter (c0, c1, c2, c3) and a 64-bit key (k0, k1).  One round is

    hi0:lo0 = M0 * c0,  hi1:lo1 = M1 * c2  (32 x 32 -> 64-bit products)
    (c0, c1, c2, c3) <- (hi1 ^ c1 ^ k0, lo1, hi0 ^ c3 ^ k1, lo0)

and the key is bumped by the Weyl constants (W0, W1) between rounds.  Vectorised over counters: every argument may be
an array and they broadcast.

The dropout of element e of a tensor (dropout.cu): word e % 4 of philox4x32_10(counter = (g, g >> 32, offset,
offset >> 32) with g = e / 4, key = (seed, seed >> 32)) gives u = (word >> 8) * 2^-24, a 24-bit uniform in [0, 1)
that fp32 holds exactly.  The element is kept when u >= p and then becomes x * scale with scale = fp32(1 / (1 - p))
computed in fp32; a dropped element is +0.0.  p is an fp32 value (the C ABI takes a float).

numpy only; no CUDA, no torch.  CPU only."""
import numpy as np

M0, M1 = 0xD2511F53, 0xCD9E8D57
W0, W1 = 0x9E3779B9, 0xBB67AE85
MASK32 = 0xFFFFFFFF
F32 = np.float32


def _u32(v):
    return np.asarray(v, dtype=np.uint64) & np.uint64(MASK32)


def philox4x32_10(c0, c1, c2, c3, k0, k1, rounds=10):
    """the four output words (uint32 arrays, broadcast shape) of Philox4x32-R for counter (c0..c3) and key (k0, k1)"""
    c0, c1, c2, c3, k0, k1 = (_u32(v) for v in (c0, c1, c2, c3, k0, k1))
    c0, c1, c2, c3, k0, k1 = np.broadcast_arrays(c0, c1, c2, c3, k0, k1)
    m0, m1, w0, w1, m32, s32 = (np.uint64(v) for v in (M0, M1, W0, W1, MASK32, 32))
    for r in range(rounds):
        if r:
            k0 = (k0 + w0) & m32
            k1 = (k1 + w1) & m32
        p0 = m0 * c0  # < 2^64: exact in uint64
        p1 = m1 * c2
        c0, c1, c2, c3 = (p1 >> s32) ^ c1 ^ k0, p1 & m32, (p0 >> s32) ^ c3 ^ k1, p0 & m32
    return tuple(v.astype(np.uint32) for v in (c0, c1, c2, c3))


def uniforms(n, seed, offset):
    """u of elements 0 .. n-1 (fp32, exact multiples of 2^-24 in [0, 1)) for the dropout stream (seed, offset)"""
    seed, offset = int(seed), int(offset)
    assert 0 <= seed < 2**64 and 0 <= offset < 2**64
    g = np.arange((n + 3) // 4, dtype=np.uint64)
    words = philox4x32_10(g & np.uint64(MASK32), g >> np.uint64(32), offset & MASK32, offset >> 32, seed & MASK32, seed >> 32)
    w = np.stack(words, axis=1).reshape(-1)[:n]
    return ((w >> np.uint32(8)).astype(np.float64) * 2.0**-24).astype(F32)


def scale_of(p):
    """fp32(1) / (fp32(1) - fp32(p)) in fp32: +inf at p == 1"""
    with np.errstate(divide="ignore"):
        return F32(1) / (F32(1) - F32(p))


def keep_mask(n, p, seed, offset):
    return uniforms(n, seed, offset) >= F32(p)


def dropout(x, p, seed, offset=0, u=None):
    """dropout.cu's forward (and, on a gradient, its backward) of the flat fp32 array x"""
    x = np.asarray(x, dtype=F32).reshape(-1)
    if u is None:
        u = uniforms(x.size, seed, offset)
    keep = u >= F32(p)
    with np.errstate(invalid="ignore", over="ignore"):
        kept = x * scale_of(p)
    return np.where(keep, kept, F32(0.0)).astype(F32)
