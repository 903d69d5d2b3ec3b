"""Exact references for three small kernels that sit on every decoded file and on VQ-VAE training: the nearest-code
search of vq.cu, the PCM16 quantisation and the feature preparation of decode.cu.  Each returns what the kernel must
produce bit for bit on the data the GPU tests use.

* ``vq_argmin``: the index of the nearest code from float64 distances, with torch.min's order (the first NaN wins,
  otherwise the smallest distance, ties to the lowest index).  On integer data in [-GRID, GRID] with D <= 768 every
  fp32 product, partial sum and the distance fmaf(-2, dot, |c|^2 + |x|^2) of the kernel is an integer below 2^24, so
  the kernel's fp32 distances equal these float64 ones and its index must equal this argmin.
* ``pcm16``: fp32(y) * 32767 in fp32, rounded half to even, NaN -> 0, saturated to [-32768, 32767].
* ``prep_features``: out[ch, u] = (c[u - pad_left, ch] - mean[ch]) / scale[ch] in fp32, in that order; frames outside
  [0, T) are +0.0 (zero edge, not normalised) or the edge frame, normalised (replicate edge).

numpy only; no CUDA.  CPU only."""
import numpy as np

F32 = np.float32
GRID = 6  # |value| of the VQ grid data


def vq_grid(rng, shape, lo=-GRID, hi=GRID):
    return rng.integers(lo, hi + 1, size=shape).astype(F32)


def require_vq_exact(z_e, codebook):
    """the precondition of bit-exact search: integer data whose squared norms and dots stay below 2^24"""
    z, c = np.asarray(z_e, np.float64), np.asarray(codebook, np.float64)
    assert np.array_equal(z, np.round(z)) and np.array_equal(c, np.round(c)), "VQ exactness: non-integer data"
    top = float(np.abs(z).max(initial=0.0)) ** 2 * c.shape[1] + float(np.abs(c).max(initial=0.0)) ** 2 * c.shape[1]
    assert 3 * top < 2**24, "VQ exactness: sums can exceed 2^24"


def vq_distances(z_e, codebook):
    """(B, T, K) float64 distances |c|^2 + |x|^2 - 2 x.c of z_e (B, D, T) to every code of codebook (K, D)"""
    x = np.asarray(z_e, np.float64).transpose(0, 2, 1)
    c = np.asarray(codebook, np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        return (c * c).sum(1)[None, None, :] + (x * x).sum(2)[:, :, None] - 2.0 * (x @ c.T)


def argmin_first(d, axis=-1):
    """torch.min's index along axis: the first NaN if there is one, else the lowest index of the smallest value"""
    d = np.moveaxis(np.asarray(d, np.float64), axis, -1)
    nan = np.isnan(d)
    k = np.where(nan, -np.inf, d).argmin(-1)  # np.argmin returns the first of equal minima
    return np.where(nan.any(-1), nan.argmax(-1), k)


def vq_argmin(z_e, codebook):
    """(B, T) int64 nearest-code indices of the grid data z_e (B, D, T) in codebook (K, D)"""
    require_vq_exact(z_e, codebook)
    return argmin_first(vq_distances(z_e, codebook)).astype(np.int64)


def pcm16(y):
    """decode.cu's PCM16 rule on the fp32 array y"""
    with np.errstate(invalid="ignore", over="ignore"):
        v = np.rint(np.asarray(y, F32) * F32(32767.0))  # one fp32 product; rint rounds half to even
    v = np.where(np.isnan(v), 0.0, v)
    return np.clip(v, -32768.0, 32767.0).astype(np.int16)


def pcm16_ties(count=4, seed=0):
    """fp32 values y in (-1, 1) whose fp32 product with 32767 is exactly k + 1/2: `count` each of even and odd k, both
    signs -- where round-half-to-even, round-half-away and truncation all differ"""
    rng = np.random.default_rng(seed)
    found = {0: [], 1: []}
    while min(len(v) for v in found.values()) < count:
        k = int(rng.integers(0, 32767))
        target = k + 0.5
        y0 = F32(target / 32767.0)
        for y in (np.nextafter(y0, F32(-1)), y0, np.nextafter(y0, F32(2))):
            if float(F32(y) * F32(32767.0)) == target and len(found[k & 1]) < count:
                found[k & 1].append(F32(y))
                break
    out = np.array(found[0] + found[1], F32)
    return np.concatenate([out, -out])


def pcm16_specials():
    """the values where a float -> int16 conversion goes wrong: signed zeros, +-1 and their neighbours, overrange,
    infinities, subnormals and NaN"""
    one = F32(1.0)
    v = [0.0, -0.0, 1.0, -1.0, np.nextafter(one, F32(2)), np.nextafter(one, F32(0)), -np.nextafter(one, F32(2)),
         -np.nextafter(one, F32(0)), 1.5, -1.5, 2.0, -2.0, 1e30, -1e30, np.inf, -np.inf, np.nan, -np.nan,
         np.finfo(F32).tiny, -np.finfo(F32).tiny, 1e-45, -1e-45, 0.5 / 32767, -0.5 / 32767, 1.5 / 32767, -1.5 / 32767,
         32767.5 / 32767, -32768.5 / 32767, -32767.5 / 32767, np.finfo(F32).max, -np.finfo(F32).max]
    return np.array(v, F32)


def prep_features(c, t_out, pad_left=0, mean=None, scale=None, replicate=False):
    """decode.cu's prep_features_kernel: c (T, C) fp32 -> (C, t_out) fp32"""
    c = np.asarray(c, F32)
    T, _ = c.shape
    src = np.arange(t_out) - pad_left
    inside = (src >= 0) & (src < T)
    rows = c[np.clip(src, 0, T - 1)]
    if mean is not None:
        with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
            rows = (rows - np.asarray(mean, F32)[None, :]) / np.asarray(scale, F32)[None, :]
    if not replicate:
        rows = np.where(inside[:, None], rows, F32(0.0))
    return np.ascontiguousarray(rows.T.astype(F32))
