"""Exact fp64 emulation of the bf16x3 tensor-core convolutions, and data on which their fp32 result is unique.

The tensor-core kernels split every fp32 operand v into bf16 parts, hi = RN_bf16(v) and lo = RN_bf16(v - hi), and
accumulate x_hi*w_hi + x_lo*w_hi + x_hi*w_lo in fp32 (the lo*lo product is dropped).  In general the fp32 result depends
on the order of the accumulation.  It does not when every product and every partial sum is an integer multiple of one
power of two g (the grid) and smaller than 2^24 g: then each fp32 addition is exact.  On such data there is exactly one
correct fp32 output, which a kernel must reproduce bit for bit whatever order it sums in.

- ``grid_values`` draws such data: v = s * (h + l * 2^-10), h and l small integers, l = 0 whenever h = 0, s a power of
  two.  RN_bf16(v) = s*h and the remainder s*l*2^-10 is exactly bf16, so hi + lo == v.
- ``conv1d``, ``conv_transpose1d``, ``conv1d_wgrad`` and ``resblock_pair`` emulate the kernels in fp64 (exact: the
  products have at most 16 significant bits and the sums stay far below 2^53 g) and apply the epilogue in the kernels'
  order.  Each returns the fp32 result and an ``Exactness`` record.
- ``Exactness.ok`` is the guard: per output element, the sum of the magnitudes of every term that reaches it (products,
  bias, residual, previous output) must stay below 2^22 g, where g is the grid of everything that is summed.  That
  leaves two bits of margin below fp32's 24.  Without the l = 0 rule a value whose hi part is zero has its hi part at the
  lo scale, the grid collapses by 2^10, and the guard fails.

CPU only; the GPU tests compare the kernels' outputs with these results by ``torch.equal``.
"""
import math
from dataclasses import dataclass

import numpy as np
import torch
import torch.nn.functional as F

LO_SCALE = 2.0 ** -10  # the lo part of a grid value, relative to its scale
EXACT_BITS = 22        # the guard: every partial sum below 2^22 grid steps (fp32 has 24)


def split(t):
    """bf16 hi / lo parts of fp32 ``t`` as fp32 tensors: hi = RN_bf16(t), lo = RN_bf16(t - hi), round to nearest even
    (``__floats2bfloat162_rn`` in ``split8`` / ``split2``)."""
    t = t.float()
    hi = t.to(torch.bfloat16).float()
    lo = (t - hi).to(torch.bfloat16).float()  # t - hi is exact in fp32
    return hi, lo


def lrelu(t, slope):
    """the kernels' LeakyReLU in fp32: v > 0 ? v : v * slope"""
    t = t.float()
    return t if slope == 1.0 else torch.where(t > 0, t, t * slope)


def grid(*ts):
    """The largest power of two that divides every value of the tensors (inf when all are zero)."""
    v = np.concatenate([torch.as_tensor(t).double().reshape(-1).numpy() for t in ts if t is not None] or [np.zeros(0)])
    v = np.abs(v[v != 0])
    if v.size == 0:
        return math.inf
    m, e = np.frexp(v)  # v = m * 2^e, 0.5 <= m < 1
    n = np.ldexp(m, 53).astype(np.int64)  # the 53-bit significand as an integer
    low = np.log2((n & -n).astype(np.float64)).astype(np.int64)  # its lowest set bit
    return math.ldexp(1.0, int((e.astype(np.int64) - 53 + low).min()))


def grid_values(shape, gen, scale=1.0, hmax=1, zero_frac=0.0, lo=True, lo_without_hi=False):
    """fp32 values s * (h + l * 2^-10): h uniform in [-hmax, hmax], set to 0 with probability ``zero_frac`` on top;
    l uniform in {-1, 0, 1} (0 when ``lo`` is False), and l = 0 wherever h = 0 unless ``lo_without_hi`` (which breaks
    the rule, for testing the guard).  ``scale`` must be a power of two."""
    assert math.frexp(scale)[0] == 0.5, "scale must be a power of two"
    h = torch.randint(-hmax, hmax + 1, shape, generator=gen, dtype=torch.int64)
    if zero_frac > 0:
        h[torch.rand(shape, generator=gen) < zero_frac] = 0
    l = torch.randint(-1, 2, shape, generator=gen, dtype=torch.int64) if lo else torch.zeros(shape, dtype=torch.int64)
    if not lo_without_hi:
        l[h == 0] = 0
    return (scale * (h.double() + LO_SCALE * l.double())).float()


@dataclass
class Exactness:
    """Guard of one emulated op: ``bound`` = max over output elements of the summed magnitudes of everything that reaches
    it, ``g`` = the grid they share (both fp64 scalars)."""

    bound: float
    g: float

    @property
    def bits(self):
        return math.log2(self.bound / self.g) if self.bound > 0 else -math.inf

    @property
    def ok(self):
        return self.bound < math.ldexp(self.g, EXACT_BITS)

    def check(self, what="op"):
        assert self.ok, f"{what}: data are not exact in fp32 (sum of magnitudes 2^{self.bits:.2f} grid steps >= 2^{EXACT_BITS})"

    def __and__(self, other):
        """the record of a chain of ops: ok only when both are"""
        return self if self.bits >= other.bits else other


def _term_grid(ah, al, bh, bl):
    """grid of the three products ah*bh, al*bh, ah*bl (al*bl is not computed by the tensor cores)"""
    gah, gal, gbh, gbl = grid(ah), grid(al), grid(bh), grid(bl)
    return min(gah * gbh, gal * gbh, gah * gbl)


def _pad(x, left, right, mode):
    if mode in ("zero", "zeros"):
        return F.pad(x, (left, right))
    return F.pad(x, (left, right), mode=mode)


def _epilogue(acc, bound, g, bias, post_act, post_slope, residual, out_scale, prev):
    """(act(acc + bias) + residual) * out_scale [+ prev] in fp64, in the kernels' order, and its exactness record"""
    v = acc.clone()
    if bias is not None:
        v = v + bias.double().reshape(1, -1, *([1] * (v.dim() - 2)))
        bound = bound + bias.double().abs().reshape(1, -1, *([1] * (v.dim() - 2)))
        g = min(g, grid(bias))
    if post_act == "lrelu":
        v = torch.where(v > 0, v, v * post_slope)
        g = g * min(1.0, post_slope)
    elif post_act not in (None, "none"):
        raise ValueError(f"post_act {post_act!r} is not exact")
    if residual is not None:
        v = v + residual.double()
        bound = bound + residual.double().abs()
        g = min(g, grid(residual))
    v = v * out_scale
    g = g * min(1.0, out_scale)
    if prev is not None:
        v = v + prev.double()
        bound = bound + prev.double().abs()
        g = min(g, grid(prev))
    ex = Exactness(float(bound.max()) if bound.numel() else 0.0, g)
    return v.float(), ex


def conv1d_acc(x, w, *, stride=1, padding=(0, 0), dilation=1, groups=1, pad_mode="zero", pre_slope=1.0, lolo=False):
    """fp64 accumulator of the bf16x3 conv: sum of x_hi w_hi + x_lo w_hi + x_hi w_lo over (channel, tap) of
    lrelu(x, pre_slope) padded by ``padding`` = (left, right) in ``pad_mode`` (zero / reflect / replicate).
    ``lolo`` adds the x_lo w_lo term the tensor cores drop (then the result is the fp64 conv of the fp32 operands).
    Returns (acc, per-element sum of the magnitudes of the terms, their grid)."""
    xh, xl = split(lrelu(x, pre_slope))
    wh, wl = split(w)
    pl, pr = padding
    xh, xl = (_pad(t.double(), pl, pr, pad_mode) for t in (xh, xl))
    wh, wl = wh.double(), wl.double()
    kw = dict(stride=stride, dilation=dilation, groups=groups)
    acc = F.conv1d(xh, wh, **kw) + F.conv1d(xl, wh, **kw) + F.conv1d(xh, wl, **kw)
    if lolo:
        acc = acc + F.conv1d(xl, wl, **kw)
    # |x_hi w_hi| + |x_lo w_hi| + |x_hi w_lo| <= (|x_hi| + |x_lo|)(|w_hi| + |w_lo|): one conv of magnitudes
    bound = F.conv1d(xh.abs() + xl.abs(), wh.abs() + wl.abs(), **kw)
    return acc, bound, _term_grid(xh, xl, wh, wl)


def conv1d(x, w, bias=None, *, stride=1, padding=(0, 0), dilation=1, groups=1, pad_mode="zero", pre_slope=1.0,
           post_act=None, post_slope=1.0, residual=None, out_scale=1.0, prev=None):
    """The stride-1 tensor-core conv (and the strided one after space-to-depth):
    y = [prev +] out_scale * (act(conv_bf16x3(lrelu(x)) + bias) + residual).  Returns (y fp32, Exactness)."""
    if isinstance(padding, int):
        padding = (padding, padding)
    acc, bound, g = conv1d_acc(x, w, stride=stride, padding=padding, dilation=dilation, groups=groups, pad_mode=pad_mode,
                               pre_slope=pre_slope)
    return _epilogue(acc, bound, g, bias, post_act, post_slope, residual, out_scale, prev)


def conv_transpose1d(x, w, bias=None, *, stride, padding=0, output_padding=0, pre_slope=1.0):
    """ConvTranspose1d (w: (cin, cout, k)) on lrelu(x) with bf16x3 products, + bias.  Returns (y fp32, Exactness)."""
    xh, xl = (t.double() for t in split(lrelu(x, pre_slope)))
    wh, wl = (t.double() for t in split(w))
    kw = dict(stride=stride, padding=padding, output_padding=output_padding)
    acc = F.conv_transpose1d(xh, wh, **kw) + F.conv_transpose1d(xl, wh, **kw) + F.conv_transpose1d(xh, wl, **kw)
    bound = F.conv_transpose1d(xh.abs() + xl.abs(), wh.abs() + wl.abs(), **kw)
    return _epilogue(acc, bound, _term_grid(xh, xl, wh, wl), bias, None, 1.0, None, 1.0, None)


def conv1d_wgrad(x, gy, kernel, *, pad_left=0, dilation=1, groups=1, x_slope=1.0, g_slope=1.0):
    """Weight gradient of a stride-1 zero-padded conv: dw[co, ci, k] = sum_{b,t} gy'[b, co, t] x'[b, ci, t + k*D - pad]
    with gy' = lrelu(gy, g_slope), x' = lrelu(x, x_slope) and bf16x3 products gy_hi x_hi + gy_lo x_hi + gy_hi x_lo.
    Returns (dw fp32 (cout, cin / groups, kernel), Exactness)."""
    gh, gl = (t.double() for t in split(lrelu(gy, g_slope)))
    xh, xl = (t.double() for t in split(lrelu(x, x_slope)))
    B, cout, t_out = gy.shape
    cin = x.shape[1]
    need = t_out + (kernel - 1) * dilation  # rows of x read, from -pad_left on
    right = need - pad_left - x.shape[2]
    xh, xl = (F.pad(t, (pad_left, max(right, 0)))[..., :need] for t in (xh, xl))

    def wg(a, b):
        return torch.nn.grad.conv1d_weight(a, (cout, cin // groups, kernel), b, dilation=dilation, groups=groups)

    acc = wg(xh, gh) + wg(xh, gl) + wg(xl, gh)
    bound = wg(xh.abs() + xl.abs(), gh.abs() + gl.abs())
    return _epilogue(acc, bound, _term_grid(gh, gl, xh, xl), None, None, 1.0, None, 1.0, None)


def resblock_pair(x, w1, b1, w2, b2, *, kernel_size, dilation, slope, out_scale=1.0, prev=None):
    """One HiFi-GAN ResBlock conv pair: h = conv_{k,d}(lrelu(x)) + b1 (exact in fp32 by its own guard), then
    y = [prev +] out_scale * (conv_{k,1}(lrelu(h)) + b2 + x), conv2 on split(lrelu(h)).  Returns (y, Exactness of both)."""
    k, d = kernel_size, dilation
    h, ex1 = conv1d(x, w1, b1, padding=(k - 1) // 2 * d, dilation=d, pre_slope=slope)
    y, ex2 = conv1d(h, w2, b2, padding=(k - 1) // 2, pre_slope=slope, residual=x, out_scale=out_scale, prev=prev)
    return y, ex1 & ex2
